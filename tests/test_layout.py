"""The product package never touches oracle/ or the reference tree."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _py_and_cu(top):
    for d, _, files in os.walk(top):
        if "__pycache__" in d or d.endswith("/build"):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                yield os.path.join(d, f)


def test_product_does_not_import_oracle_or_reference():
    pat = re.compile(r"^\s*(from|import)\s+oracle\b|/root/reference|oracle/_", re.M)
    bad = []
    for path in _py_and_cu(os.path.join(ROOT, "vidar_b200")):
        with open(path) as fh:
            if pat.search(fh.read()):
                bad.append(path)
    assert not bad, f"product files reference oracle/ or /root/reference: {bad}"


def test_native_library_reads_no_environment():
    """What libvidar_b200.so computes and which kernels it launches depend only on its arguments."""
    bad = []
    for path in _py_and_cu(os.path.join(ROOT, "vidar_b200", "csrc")):
        with open(path) as fh:
            if re.search(r"\bgetenv\b", fh.read()):
                bad.append(path)
    assert not bad, f"native sources read environment variables: {bad}"


def test_no_cpu_fallback_on_cpu_tensors():
    import pytest
    import torch
    from vidar_b200 import msda, render
    v = torch.zeros(1, 4, 1, 32)
    shapes = torch.tensor([[2, 2]])
    lsi = torch.tensor([0])
    loc = torch.zeros(1, 1, 1, 1, 1, 2)
    aw = torch.zeros(1, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        msda.ext_module.ms_deform_attn_forward(v, shapes, lsi, loc, aw, im2col_step=64)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        render.dvr.render_forward(torch.zeros(1, 1, 2, 2, 2), torch.zeros(1, 1, 3),
                                  torch.zeros(1, 1, 3), torch.zeros(1, 1), [1, 2, 2, 2], "test")
    with pytest.raises(ValueError, match="UNKNOWN LOSS TYPE"):
        render.dvr.render(None, None, None, None, "huber")
