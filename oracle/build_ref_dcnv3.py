"""Compile the reference's OWN DCNv3 extension (InternImage's ops_dcnv3) for sm_90a into oracle/_ref/ref_dcnv3.so.

TEST INFRASTRUCTURE, the DCNv3 companion of oracle/build_ref.py (same output directory, same `load`).  The sources
(`src/vision.cpp`, `src/cuda/dcnv3_cuda.cu`, `src/cpu/dcnv3_cpu.cpp` and the headers next to them) are read from the
reference checkout and compiled from a temporary patched copy, never copied into the repo.  They do not build
unmodified against torch 2.x; the patch is mechanical and touches no arithmetic:
    .type().is_cuda()                              ->  .is_cuda()
    AT_DISPATCH_FLOATING_TYPES_AND_HALF(X.type()   ->  AT_DISPATCH_FLOATING_TYPES_AND_HALF(X.scalar_type()
    #include <THC/THCAtomics.cuh>                  ->  #include <ATen/cuda/Atomic.cuh>
`-DWITH_CUDA` goes to both the C++ and the nvcc flags, with `src/` on the include path.  The product runs on a GPU
box only: there it is a second oracle (tests/test_dcnv3_gpu.py) and the baseline of tools/bench_dcnv3.py.
"""
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))

from oracle import build_ref  # noqa: E402

NAME = "ref_dcnv3"
SRC = "/root/reference/projects/mmdet3d_plugin/bevformer/backbones/ops_dcnv3/src"
SOURCES = ["vision.cpp", "cuda/dcnv3_cuda.cu", "cpu/dcnv3_cpu.cpp"]
CUDA_FLAGS = ["-DWITH_CUDA", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"]


def _patch(text):
    text = text.replace(".type().is_cuda()", ".is_cuda()")
    text = re.sub(r"AT_DISPATCH_FLOATING_TYPES_AND_HALF\((\s*)(\w+)\.type\(\)",
                  r"AT_DISPATCH_FLOATING_TYPES_AND_HALF(\1\2.scalar_type()", text)
    return text.replace("#include <THC/THCAtomics.cuh>", "#include <ATen/cuda/Atomic.cuh>")


def _stamp():
    return build_ref.so_path(NAME) + ".flags"


def is_current():
    try:
        with open(_stamp()) as fh:
            return os.path.exists(build_ref.so_path(NAME)) and fh.read().strip() == " ".join(CUDA_FLAGS)
    except OSError:
        return False


def build(force=False):
    """Build oracle/_ref/ref_dcnv3.so where the reference checkout exists (about 5 minutes of nvcc); returns its
    path, or None without a checkout."""
    if not os.path.isdir(SRC):
        return None
    if is_current() and not force:
        return build_ref.so_path(NAME)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils import cpp_extension
    os.makedirs(build_ref.OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix=f"{NAME}_src_")
    bdir = tempfile.mkdtemp(prefix=f"{NAME}_build_")
    try:
        for root, _, files in os.walk(SRC):
            for f in files:
                if f.endswith((".cpp", ".cu", ".h", ".cuh")):
                    rel = os.path.relpath(os.path.join(root, f), SRC)
                    os.makedirs(os.path.dirname(os.path.join(tmp, rel)), exist_ok=True)
                    with open(os.path.join(SRC, rel)) as fh:
                        text = _patch(fh.read())
                    with open(os.path.join(tmp, rel), "w") as fh:
                        fh.write(text)
        cpp_extension.load(name=NAME, sources=[os.path.join(tmp, s) for s in SOURCES], extra_include_paths=[tmp],
                           extra_cflags=["-DWITH_CUDA"], extra_cuda_cflags=CUDA_FLAGS, build_directory=bdir,
                           verbose=False, is_python_module=False)
        shutil.copy(os.path.join(bdir, NAME + ".so"), build_ref.so_path(NAME))
        with open(_stamp(), "w") as fh:
            fh.write(" ".join(CUDA_FLAGS))
        return build_ref.so_path(NAME)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.rmtree(bdir, ignore_errors=True)


def load():
    """The prebuilt module (dcnv3_forward / dcnv3_backward); FileNotFoundError when it was not built."""
    return build_ref.load(NAME)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
