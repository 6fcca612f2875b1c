"""The configs' optimizer without a GPU: `paramwise_groups` restates mmcv 1.4's custom_keys rule (key order, substring
matches, frozen parameters, decay_mult) and gives SyntheticViDAR's trainable backbone tensors, and only those, the
0.1 rate; `optim.AdamW` rejects what it cannot step before any CUDA call, and `vidar_adamw_step` rejects bad
arguments with a message."""
import ctypes
import threading

import numpy as np
import pytest
import torch
import torch.nn as nn

from vidar_b200 import _lib, optim


class _Toy(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone = nn.Module()
        self.backbone.stem = nn.Linear(2, 2)
        self.backbone.layer4 = nn.Linear(2, 2)
        self.neck = nn.Linear(2, 1, bias=False)
        self.neck_backbone_adapter = nn.Linear(1, 1)     # 'backbone' in the middle of the name
        self.head = nn.Linear(1, 1)
        self.backbone.stem.weight.requires_grad_(False)  # frozen: base values although 'backbone' matches


def test_paramwise_groups_follow_mmcv_custom_keys():
    keys = {"backbone": dict(lr_mult=0.1), "backbone.layer4": dict(lr_mult=0.5, decay_mult=0.0),
            "head": dict(decay_mult=2.0), "ck": dict(lr_mult=3.0)}
    groups = optim.paramwise_groups(_Toy(), 1.0, 0.01, keys)
    got = [(g["lr"], g["weight_decay"]) for g in groups]
    want = [
        (1.0, 0.01),            # backbone.stem.weight: frozen
        (0.1, 0.01),            # backbone.stem.bias: 'backbone'
        (0.5, 0.0),             # backbone.layer4.weight: the longer key first
        (0.5, 0.0),             # backbone.layer4.bias
        (3.0, 0.01),            # neck.weight: 'ck' inside 'neck'
        (0.1, 0.01),            # neck_backbone_adapter.weight: 'backbone' (longer than 'ck') wins
        (0.1, 0.01),            # neck_backbone_adapter.bias
        (1.0, 0.02),            # head.weight: decay_mult only
        (1.0, 0.02),            # head.bias
    ]
    assert [n for n, _ in _Toy().named_parameters()][:3] == ["backbone.stem.weight", "backbone.stem.bias",
                                                             "backbone.layer4.weight"]
    assert all(len(g["params"]) == 1 for g in groups)
    np.testing.assert_allclose(got, want, rtol=1e-15)


def test_equal_length_keys_are_tried_alphabetically():
    m = nn.Module()
    m.ab_cd = nn.Linear(1, 1, bias=False)
    groups = optim.paramwise_groups(m, 1.0, 0.0, {"cd": dict(lr_mult=2.0), "ab": dict(lr_mult=3.0)})
    assert groups[0]["lr"] == 3.0


def test_synthetic_vidar_backbone_gets_a_tenth_of_the_rate():
    from vidar_b200 import pretrain
    model = pretrain.SyntheticViDAR(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(20, 20))
    groups = optim.paramwise_groups(model, 2e-4, 0.01, {"backbone": dict(lr_mult=0.1)})
    names = [n for n, _ in model.named_parameters()]
    assert len(groups) == len(names)
    for name, g in zip(names, groups):
        (p,) = g["params"]
        slow = name.startswith("backbone.") and p.requires_grad
        assert g["lr"] == pytest.approx(2e-5 if slow else 2e-4, rel=1e-12), name
        assert g["weight_decay"] == 0.01
    assert sum(g["lr"] < 1e-4 for g in groups) > 100


def test_rejects_what_it_cannot_step():
    with pytest.raises(RuntimeError, match="fp32 CUDA parameters"):
        optim.AdamW([nn.Parameter(torch.zeros(3))])
    with pytest.raises(RuntimeError, match="fp32 CUDA parameters"):
        optim.AdamW(optim.paramwise_groups(nn.Linear(2, 2), 1e-3, 0.01, {}))
    with pytest.raises(ValueError, match="amsgrad"):
        optim.AdamW([], amsgrad=True)
    with pytest.raises(ValueError, match="max_grad_norm"):
        optim.AdamW([], max_grad_norm=0.0)


def test_adamw_step_rejects_bad_arguments():
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    i64 = lambda *v: np.array(v, np.int64)
    sc = np.zeros((2, 7), np.float32)
    ptr, odd, numel = i64(0x1000, 0x2000), i64(0x1000, 0x2002), i64(4, 5)
    null_param, neg = i64(0x1000, 0), i64(4, -1)          # named: ctypes gets only their addresses
    cases = [
        ((N, N, N, N, -1, X, X, 9, 0, 0.0, N, N), b"bad sizes"),
        ((N, N, N, N, 2, X, X, 9, 0, 0.0, N, N), b"null pointer argument (table)"),
        ((ptr.ctypes.data, ptr.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, X, X, 9, 1, 35.0, N, N),
         b"null pointer argument (grad_norm)"),
        ((ptr.ctypes.data, ptr.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, X, X, 8, 0, 0.0, N, N),
         b"does not fit the state"),
        ((ptr.ctypes.data, odd.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, X, X, 9, 0, 0.0, N, N),
         b"not 4-byte aligned"),
        ((null_param.ctypes.data, ptr.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, X, X, 9, 0, 0.0, N, N),
         b"null pointer argument (parameter 1)"),
        ((ptr.ctypes.data, ptr.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, N, N, 9, 0, 0.0, N, N),
         b"exp_avg"),
        ((ptr.ctypes.data, ptr.ctypes.data, numel.ctypes.data, sc.ctypes.data, 2, ctypes.c_void_p(0x1002), X, 9, 0,
          0.0, N, N), b"4-byte aligned"),
        ((ptr.ctypes.data, ptr.ctypes.data, neg.ctypes.data, sc.ctypes.data, 2, X, X, 9, 0, 0.0, N, N),
         b"does not fit the state"),
    ]
    got = []

    def run():                      # on a thread of its own: the last-error text is per thread
        for args, _ in cases:
            got.append((L.vidar_adamw_step(*args), L.vidar_last_error()))
        got.append((L.vidar_adamw_step(N, N, N, N, 0, N, N, 0, 0, 0.0, N, N), None))   # nothing to step: a no-op

    t = threading.Thread(target=run)
    t.start()
    t.join()
    for (rc, msg), (_, needle) in zip(got, cases):
        assert rc == 1 and needle in msg, (needle, rc, msg)
    assert got[-1][0] == 0 and len(got) == len(cases) + 1
