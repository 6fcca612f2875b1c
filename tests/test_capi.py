"""The C-ABI library builds, loads on a GPU-less host and exports every symbol that
include/vidar_b200.h declares (no compute calls here)."""
import ctypes
import os
import re
import subprocess

from vidar_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_is_built_and_loads():
    build.build()
    L = _lib.lib()
    assert b"sm_90a" in L.vidar_version()
    assert L.vidar_last_error() == b""
    assert L.vidar_launch_count() == 0 or L.vidar_launch_count() > 0


def test_every_declared_symbol_is_exported():
    build.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    with open(_lib.HEADER) as fh:
        src = re.sub(r"/\*.*?\*/", "", fh.read(), flags=re.S)
    names = re.findall(r"\b(vidar_\w+)\s*\(", src)
    assert len(names) >= 12
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/vidar_b200.h but not exported"
    # and the typed view used by the Python layer covers the int-returning entry points
    typed = {n for n, _ in _lib.declared_symbols()}
    assert {"vidar_msda_forward", "vidar_msda_backward", "vidar_dvr_render"} <= typed


def test_library_has_no_torch_dependency_and_is_sm90a():
    build.build()
    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "torch" not in out and "c10" not in out
    sass = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass


def test_bad_arguments_are_reported_not_crashed():
    L = _lib.lib()
    rc = L.vidar_msda_forward(None, None, None, None, None, None, 1, 1, 1, 32, 1, 1, 1, 64, None)
    assert rc == 1
    assert b"null pointer" in L.vidar_last_error()
    try:
        _lib.check(rc)
    except RuntimeError as e:
        assert "null pointer" in str(e)
    else:
        raise AssertionError("check() must raise")


def test_argument_validation_of_the_fused_entry_points():
    """Shape contracts of the fused ops are checked before anything touches the device, so they can be
    exercised on a GPU-less host: every call below must return VIDAR_E_INVALID with a message."""
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    # the LatentRendering core on an empty cell range: a missing check would return success, not launch
    lr = (1, 16, 4, 4, 8, 0.5)                      # bs, D, Hb, Wb, grid_num, grid_step
    lr_g = (1, 16, 1, 4, 4, 8, 0.5, 1e-3)           # bs, D, G, Hb, Wb, grid_num, grid_step, eps
    cases = [
        (L.vidar_latent_prob_forward, (X, X, N) + lr + (1, 0, 0, N), b"null pointer"),
        (L.vidar_latent_pool_forward, (X, X, X, N) + lr_g + (0, 0, N), b"null pointer"),
        (L.vidar_latent_pool_backward, (X, X, X, N, X, X, X) + lr_g + (0, 0, N), b"null pointer"),
        (L.vidar_latent_pool_backward, (X, X, N, X, X, X, X) + lr_g + (0, 0, N), b"null pointer"),
        (L.vidar_latent_prob_backward, (X, N, X, X) + lr + (1, 0, 0, N), b"null pointer"),
        (L.vidar_latent_proj_in_forward, (N, N, N, N, N, N, N, 10, 64, 16, 16, N), b"embed_dims must be 128 or 256"),
        (L.vidar_latent_proj_in_backward, (N,) * 10 + (10, 256, 20, 16, N), b"pred_height + rank"),
        (L.vidar_latent_proj_out_forward, (N, N, N, N, N, 10, 256, 24, 8, N), b"embed_dims / pred_height"),
        (L.vidar_latent_proj_out_backward, (N,) * 9 + (10, 256, 8, 8, N), b"rank"),
        (L.vidar_latent_proj_in_forward, (N, N, N, N, N, N, N, 10, 256, 16, 16, N), b"null pointer"),
        (L.vidar_msda_sca_forward, (N,) * 7 + (1, 10, 8, 32, 1, 5, 4, 4, N), b"null pointer"),
        (L.vidar_ray_gumbel_forward, (N,) * 8 + (5, 1, 4, 4, 4, 0, 1.0, N), b"bad sizes"),
        (L.vidar_ray_gumbel_backward, (N,) * 9 + (5, 1, 4, 4, 4, 8, 1.0, N), b"null pointer"),
    ]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, rc)
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())
    # zero rows is a valid no-op
    assert L.vidar_latent_proj_out_forward(N, N, N, N, N, 0, 256, 16, 16, N) == 0
    assert L.vidar_ray_gumbel_forward(*((N,) * 8 + (0, 1, 4, 4, 4, 8, 1.0, N))) == 0


def test_argument_validation_of_the_round2_entry_points():
    """Row-indirect MSDA (BEV-slot) ops, the visible-list compaction and the tensor-core Linear: size contracts are
    rejected with a message before any launch.  Pointers are only compared with NULL on these paths, so a dummy
    non-null address stands in for device memory (every call here fails validation; nothing is launched)."""
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    rows_fwd = lambda **k: (X, X, X, X, X, k.get("idx", X), X, X, k.get("slots", X), k.get("bs", 1), k.get("ncl", 6),
                            k.get("cam0", 0), 100, 8, k.get("C", 32), 4, k.get("rows", 50), k.get("Qd", 50), 8,
                            k.get("S", 1), k.get("lo", 0), k.get("hi", 1), N)
    cases = [
        (L.vidar_msda_rows_forward, (N,) * 9 + (1, 6, 0, 100, 8, 32, 4, 50, 50, 8, 1, 0, 1, N), b"null pointer"),
        (L.vidar_msda_rows_forward, rows_fwd(rows=60), b"exceed the pillar count"),
        (L.vidar_msda_rows_forward, rows_fwd(idx=N, rows=40), b"without an index list"),
        (L.vidar_msda_rows_forward, rows_fwd(S=4, lo=3, hi=5), b"bad sub-slice"),
        (L.vidar_msda_rows_forward, rows_fwd(C=24), b"head dim must be 16, 32 or 64"),
        (L.vidar_msda_rows_forward, rows_fwd(cam0=-1), b"bad sizes"),
        (L.vidar_msda_rows_forward, rows_fwd(slots=N), b"null output"),
        (L.vidar_msda_rows_backward, (X,) * 9 + (N, X, X, 1, 6, 0, 100, 8, 32, 4, 50, 50, 8, 1, 0, 1, N), b"null gradient pointer"),
        (L.vidar_msda_sca_rows_forward, (X, X, X, N, X, X, X, X, X, X, 1, 6, 0, 100, 8, 32, 4, 50, 50, 8, 4, 1, 0, 1, N), b"null reference points"),
        (L.vidar_sca_compact, (N, N, N, N, 6, 1, 100, 4, N), b"null pointer"),
        (L.vidar_sca_compact, (X, X, X, X, 6, 1, 0, 4, N), b"bad sizes"),
        (L.vidar_linear_tf32x3, (N, N, N, N, N, 10, 128, 128, N), b"null pointer"),
        (L.vidar_linear_tf32x3, (X, X, X, X, X, 10, 128, 100, N), b"in_features must be a multiple of 32"),
        (L.vidar_linear_tf32x3, (X, X, X, X, X, 10, 96, 128, N), b"out_features of 128"),
        (L.vidar_linear_tf32x3, (X, X, X, X, X, 0, 128, 128, N), b"bad sizes"),
        (L.vidar_linear_tf32x3, (ctypes.c_void_p(0x1004), X, X, X, X, 10, 128, 128, N), b"16-byte aligned"),
    ]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())


def test_python_call_sites_pass_as_many_arguments_as_the_header_declares():
    """Static: every `<lib>.vidar_xxx(...)` call in the package, bench, tools and tests passes the number of
    arguments `include/vidar_b200.h` declares (ctypes would only notice at run time, on the GPU box)."""
    import ast
    import glob
    decl = {n: len(a) for n, a in _lib.declared_symbols()}
    seen, bad = 0, []
    files = [p for pat in ("vidar_b200/**/*.py", "tests/*.py", "tools/*.py", "*.py") for p in glob.glob(os.path.join(ROOT, pat), recursive=True)]
    for path in files:
        with open(path) as fh:
            tree = ast.parse(fh.read())
        for n in ast.walk(tree):
            if (isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr in decl
                    and not any(isinstance(a, ast.Starred) for a in n.args) and not n.keywords):
                seen += 1
                if len(n.args) != decl[n.func.attr]:
                    bad.append(f"{os.path.relpath(path, ROOT)}:{n.lineno} {n.func.attr}: {len(n.args)} args, header says {decl[n.func.attr]}")
    assert seen >= 30 and not bad, "\n".join(bad)
