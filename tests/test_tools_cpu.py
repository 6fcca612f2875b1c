"""The scripts under tools/ compile, and their measuring code lives in tools/gpu_timing.py alone: no other tool builds
CUDA events, reads nvidia-smi, counts syncs or allocates an L2 flush buffer of its own."""
import glob
import os
import py_compile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = sorted(glob.glob(os.path.join(ROOT, "tools", "*.py")))
MEASURING = ("torch.cuda.Event(", "nvidia-smi", "set_sync_debug_mode", "256 << 20")


@pytest.mark.parametrize("path", TOOLS, ids=os.path.basename)
def test_tool_compiles(path, tmp_path):
    py_compile.compile(path, cfile=str(tmp_path / "tool.pyc"), doraise=True)


def test_measuring_code_only_in_gpu_timing():
    found = []
    for path in glob.glob(os.path.join(ROOT, "tools", "*")):
        if os.path.isfile(path) and os.path.basename(path) != "gpu_timing.py":
            with open(path, errors="replace") as fh:
                text = fh.read()
            found += [f"{os.path.basename(path)}: {s}" for s in MEASURING if s in text]
    assert not found, "\n".join(found)
