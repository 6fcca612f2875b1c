"""vidar_msda_tsa_forward / _backward reject bad arguments with a message before anything touches the device, and
the modules keep CPU tensors on the reference's statements.  No GPU needed: pointers are only compared with NULL
on these paths, so a dummy non-null address stands in for device memory (every call fails validation)."""
import ctypes

import torch

from tests import module_cases as mc
import vidar_b200.modules  # noqa: F401  (registers the classes)
from vidar_b200 import _lib
from vidar_b200.modules import deform_attn
from vidar_b200.registry import build_attention


def test_argument_validation_of_the_queue_fused_entry_points():
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    # B, G, K, H, C, L, Q, P
    fwd = lambda ref=X, out=X, G=2, C=32, Lv=1, P=4: (X, X, X, ref, X, X, out, 1, G, 100, 8, C, Lv, 50, P, N)
    bwd = lambda grad=X: (X, X, X, X, X, X, grad, X, X, X, 1, 2, 100, 8, 32, 1, 50, 4, N)
    cases = [
        (L.vidar_msda_tsa_forward, (N,) * 7 + (1, 2, 100, 8, 32, 1, 50, 4, N), b"null pointer"),
        (L.vidar_msda_tsa_forward, fwd(ref=N), b"null reference points"),
        (L.vidar_msda_tsa_forward, fwd(P=3), b"num_levels * num_points in {1, 2, 4, 8, 16, 32}"),
        (L.vidar_msda_tsa_forward, fwd(Lv=4, P=16), b"num_levels * num_points in {1, 2, 4, 8, 16, 32}"),
        (L.vidar_msda_tsa_forward, fwd(G=3, P=16), b"at most 32"),
        (L.vidar_msda_tsa_forward, fwd(G=0), b"at most 32"),
        (L.vidar_msda_tsa_forward, fwd(C=24), b"head dim must be 16, 32 or 64"),
        (L.vidar_msda_tsa_forward, fwd(out=N), b"null output"),
        (L.vidar_msda_tsa_backward, (N,) * 10 + (1, 2, 100, 8, 32, 1, 50, 4, N), b"null pointer"),
        (L.vidar_msda_tsa_backward, bwd(grad=N), b"null gradient pointer"),
    ]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())


def test_cpu_modules_keep_the_reference_statements(monkeypatch):
    """CPU tensors never reach the fused Function (it needs CUDA); the plain op is called instead."""
    calls = []
    monkeypatch.setattr(deform_attn, "msda_queue_fused_apply", lambda *a: calls.append("fused"))
    monkeypatch.setattr(deform_attn, "msda_apply", lambda v, s, i, loc, w, step: calls.append("plain") or
                        v.new_zeros(loc.shape[0], loc.shape[1], v.shape[2] * v.shape[3]))
    for cfg, case in ((mc.TSA_CFG, mc.tsa_case), (mc.PRED_CFG, mc.pred_case)):
        m = build_attention(cfg)
        c = case()
        with torch.no_grad():
            m(c["query"], None, c["value"], query_pos=c["query_pos"], reference_points=c["reference_points"],
              spatial_shapes=c["spatial_shapes"], level_start_index=c["level_start_index"])
        assert m.fuse_epilogue
    assert calls == ["plain", "plain"]
