"""Compile the reference's OWN ray-caster kernels for sm_90a into oracle/_ref/ (git-ignored).

TEST INFRASTRUCTURE.  third_lib/dvr and third_lib/dvxlr are torch C++/CUDA extensions made
of two files each; they are compiled from where they lie under /root/reference by this
recipe, never copied into the repo.  They do not build unmodified against torch 2.11
(`AT_DISPATCH_FLOATING_TYPES(x.type(), ...)` needs a ScalarType; `x.type().is_cuda()` is
gone), so the recipe applies a mechanical two-token patch to a *temporary* copy:
    .type().is_cuda()  ->  .is_cuda()
    X.type(),          ->  X.scalar_type(),     (inside AT_DISPATCH_FLOATING_TYPES only)
No arithmetic is touched.  Outputs: oracle/_ref/ref_{dvr,dvxlr,dvxlr_v2}.so.

The products can only *run* on a GPU box.  They serve as (1) a second oracle there
(tests/test_ref_cuda_gpu.py, tools/make_golden_dvr.py) and (2) the same-box GPU baseline.
/root/reference does not exist on the GPU box: build here, the .so files travel.
"""
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = "/root/reference/third_lib"
TARGETS = {
    "ref_dvr": ("dvr", ["dvr.cpp", "dvr.cu"]),
    "ref_dvxlr": ("dvxlr", ["dvxlr.cpp", "dvxlr.cu"]),
    "ref_dvxlr_v2": ("dvxlr", ["dvxlr_v2.cpp", "dvxlr_v2.cu"]),
}
# dvr.cu launches 1024-thread blocks (dvr.cu:345,651); uncapped, its render kernels need
# > 64 registers/thread, and 1024 x 65+ exceeds the 64K-register file: every launch fails
# with cudaErrorLaunchOutOfResources.  A register cap is the build flag that makes the
# unmodified kernel launchable; it changes no arithmetic.
EXTRA_FLAGS = {"ref_dvr": ["-maxrregcount=64"]}


def _patch(text):
    text = text.replace(".type().is_cuda()", ".is_cuda()")
    text = re.sub(r"AT_DISPATCH_FLOATING_TYPES\((\w+)\.type\(\)", r"AT_DISPATCH_FLOATING_TYPES(\1.scalar_type()", text)
    return text


KNN_SRC = "/root/reference/third_lib/chamfer_dist/chamferdist/chamferdist"


def build_knn_cpu(force=False):
    """The reference's CPU KNN (chamferdist ext.cpp + knn_cpu.cpp, built WITHOUT `WITH_CUDA`) compiled
    unmodified from where it lies -> oracle/_ref/ref_knn_cpu.so.  It runs on any host, so it pins the
    NN oracle here and can serve as a `kind: "reference"` CPU baseline."""
    if not os.path.isdir(KNN_SRC):
        return None
    out = so_path("ref_knn_cpu")
    if os.path.exists(out) and not force:
        return out
    from torch.utils import cpp_extension
    os.makedirs(OUT, exist_ok=True)
    bdir = tempfile.mkdtemp(prefix="ref_knn_build_")
    try:
        cpp_extension.load(name="ref_knn_cpu", sources=[os.path.join(KNN_SRC, "ext.cpp"), os.path.join(KNN_SRC, "knn_cpu.cpp")],
                           extra_include_paths=[KNN_SRC], build_directory=bdir, verbose=False, is_python_module=False)
        shutil.copy(os.path.join(bdir, "ref_knn_cpu.so"), out)
    finally:
        shutil.rmtree(bdir, ignore_errors=True)
    return out


def so_path(name):
    return os.path.join(OUT, name + ".so")


def _cuda_flags(name):
    return ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"] + EXTRA_FLAGS.get(name, [])


def _stamp_path(name):
    return so_path(name) + ".flags"


def is_current(name):
    """The .so exists and, for the CUDA targets, was built with today's flags (architecture included): a
    library left from a build for another GPU is rebuilt rather than loaded."""
    if not os.path.exists(so_path(name)):
        return False
    if name not in TARGETS:
        return True
    try:
        with open(_stamp_path(name)) as fh:
            return fh.read().strip() == " ".join(_cuda_flags(name))
    except OSError:
        return False


def _build_one(name, force=False):
    sub, files = TARGETS[name]
    if is_current(name) and not force:
        return so_path(name)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", "2")
    from torch.utils import cpp_extension
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix=f"{name}_src_")
    bdir = tempfile.mkdtemp(prefix=f"{name}_build_")
    try:
        srcs = []
        for f in files:
            with open(os.path.join(REF, sub, f)) as fh:
                text = _patch(fh.read())
            dst = os.path.join(tmp, f)
            with open(dst, "w") as fh:
                fh.write(text)
            srcs.append(dst)
        cpp_extension.load(
            name=name, sources=srcs, build_directory=bdir, verbose=False,
            extra_cuda_cflags=_cuda_flags(name),
            is_python_module=False)
        shutil.copy(os.path.join(bdir, name + ".so"), so_path(name))
        with open(_stamp_path(name), "w") as fh:
            fh.write(" ".join(_cuda_flags(name)))
        return so_path(name)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.rmtree(bdir, ignore_errors=True)


def build(names=None, force=False, parallel=True):
    """Build the missing reference extensions (each ~4 min of ptxas on the MAX_D local arrays); the
    targets are independent, so they are compiled in parallel child processes."""
    if not os.path.isdir(REF):
        return {}        # GPU box: use the prebuilt files
    import subprocess
    os.makedirs(OUT, exist_ok=True)
    want = [n for n in list(TARGETS) + ["ref_knn_cpu"] if not names or n in names]
    todo = [n for n in want if force or not is_current(n)]
    if parallel and len(todo) > 1:
        procs = [(n, subprocess.Popen([sys.executable, os.path.abspath(__file__), "--one", n] + (["--force"] if force else []),
                                      stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)) for n in todo]
        for n, p in procs:
            _, err = p.communicate()
            if p.returncode != 0:
                raise RuntimeError(f"building {n} failed:\n{err[-2000:]}")
    else:
        for n in todo:
            build_knn_cpu(force) if n == "ref_knn_cpu" else _build_one(n, force)
    return {n: so_path(n) for n in want if os.path.exists(so_path(n))}


def load(name):
    """Import a prebuilt reference extension (needs a CUDA-capable torch at call time)."""
    import importlib.util

    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    path = so_path(name)
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not built (run `python oracle/build_ref.py` where /root/reference exists)")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    argv = [a for a in sys.argv[1:] if not a.startswith("--")]
    force = "--force" in sys.argv
    if "--one" in sys.argv:
        print(build_knn_cpu(force) if argv[0] == "ref_knn_cpu" else _build_one(argv[0], force))
    else:
        print(build(names=argv or None, force=force))
