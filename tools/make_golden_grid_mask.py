"""Write tests/golden/grid_mask.npz from the reference's OWN `GridMask` (projects/mmdet3d_plugin/models/utils/
grid_mask.py), loaded from the reference checkout with `mmcv.runner` stubbed by tools/ref_shim.py and `.cuda()` made
the identity on CPU.  Test infrastructure: nothing of the reference is copied, only its outputs.

For every case the reference's forward runs once with numpy seeded, on x = ones [1, 1, h, w] (the output is the
mask, or mask + offset * (1 - mask) with `offset`, whose offset never equals 1, so mask = (out == 1)) and, for the
small cases, once more with the same seed on a seeded x [1, 2, h, w] (quarter steps in [-2, 2], with inf, -inf,
NaN and -0.0 in fixed places) in float32, float16 and bfloat16.  The numpy
calls it makes are logged, which gives the draws.  Per case:
  <case>/params  [h, w, use_h, use_w, rotate, offset, ratio * 1000, mode, prob * 1000, training, seed]
  <case>/draws   [d, l, st_h, st_w, r] ([] when the prob gate returned x)
  <case>/mask    np.packbits of the [h, w] mask (0 / 1 after mode), when masked
  <case>/state_keys, <case>/state_pos: numpy's MT19937 state after the call
  <case>/x, <case>/out_f32, <case>/out_f16 / out_bf16 (raw 16-bit patterns), small cases only
and sig/init, sig/set_prob (the signatures as text), sig/attrs (the public attributes of a fresh module).

    python tools/make_golden_grid_mask.py
"""
import importlib.util
import inspect
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ref_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "grid_mask.npz")
REF = os.path.join(os.path.dirname(ref_shim.REF_BEVFORMER), "models", "utils", "grid_mask.py")   # the plugin checkout ref_shim uses
SMALL = 25000        # pixels: cases up to this size also store x and the outputs
# (name, h, w, use_h, use_w, rotate, offset, ratio, mode, prob, training, seed)
CASES = [
    ("cfg_928x1600", 928, 1600, True, True, 1, False, 0.5, 1, 0.7, True, 0),
    ("rot360_928x1600", 928, 1600, True, True, 360, False, 0.5, 0, 1.0, True, 1),
    ("rot360_58x100_m0", 58, 100, True, True, 360, False, 0.5, 0, 1.0, True, 2),
    ("rot360_58x100_m1", 58, 100, True, True, 360, False, 0.5, 1, 1.0, True, 3),
    ("rows_58x100", 58, 100, True, False, 360, False, 0.5, 0, 1.0, True, 4),
    ("cols_58x100", 58, 100, False, True, 360, False, 0.5, 1, 1.0, True, 5),
    ("none_58x100", 58, 100, False, False, 360, False, 0.5, 0, 1.0, True, 6),
    ("rot1_200x200", 200, 200, True, True, 1, False, 0.5, 1, 1.0, True, 7),
    ("rot360_200x200", 200, 200, True, True, 360, False, 0.5, 0, 1.0, True, 8),
    ("offset_58x100", 58, 100, True, True, 360, True, 0.5, 0, 1.0, True, 9),
    ("offset_57x99_m1", 57, 99, True, True, 360, True, 0.5, 1, 1.0, True, 10),
    ("ratio1_58x100", 58, 100, True, True, 360, False, 1.0, 0, 1.0, True, 11),
    ("ratio1_offset_31x47", 31, 47, True, True, 90, True, 1.0, 1, 1.0, True, 12),
    ("d2_3x7", 3, 7, True, True, 360, False, 0.5, 0, 1.0, True, 13),
    ("d2_3x8_offset", 3, 8, True, True, 360, True, 0.5, 1, 1.0, True, 14),
    ("odd_101x203", 101, 203, True, True, 360, False, 0.5, 1, 1.0, True, 15),
    ("gate_closed", 58, 100, True, True, 360, False, 0.5, 0, 0.0, True, 16),
    ("eval", 58, 100, True, True, 360, True, 0.5, 0, 1.0, False, 17),
]


def load_reference():
    ref_shim.install()                      # mmcv.runner.auto_fp16 becomes a pass-through decorator
    spec = importlib.util.spec_from_file_location("vidar_ref_grid_mask", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.GridMask


class DrawLog:
    """Wraps np.random.rand / randint for the duration of a call and records every value they return."""

    def __enter__(self):
        self.calls, self._orig = [], (np.random.rand, np.random.randint)
        rand, randint = self._orig

        def log_rand(*a):
            v = rand(*a)
            self.calls.append(("rand", a, v))
            return v

        def log_randint(*a):
            v = randint(*a)
            self.calls.append(("randint", a, v))
            return v
        np.random.rand, np.random.randint = log_rand, log_randint
        return self

    def __exit__(self, *exc):
        np.random.rand, np.random.randint = self._orig


def run(module, x, seed):
    """One reference forward with numpy seeded -> (output, logged calls, numpy state after)."""
    np.random.seed(seed)
    with DrawLog() as log, torch.no_grad():
        y = module(x)
    return y, log.calls, np.random.get_state()


def main():
    GridMask = load_reference()
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference uploads the mask; here it stays on CPU
    g = torch.Generator().manual_seed(2025)
    out = {}
    for name, h, w, use_h, use_w, rotate, offset, ratio, mode, prob, training, seed in CASES:
        m = GridMask(use_h, use_w, rotate=rotate, offset=offset, ratio=ratio, mode=mode, prob=prob)
        m.train(training)
        ones = torch.ones(1, 1, h, w)
        y, calls, state = run(m, ones, seed)
        masked = y is not ones
        draws = []
        if masked:
            ints = [v for kind, _, v in calls if kind == "randint"]
            d, st_h, st_w, r = (int(v) for v in ints)
            draws = [d, m.l, st_h, st_w, r]
            mask = (y[0, 0].numpy() == 1).astype(np.uint8)
            out[f"{name}/mask"] = np.packbits(mask)
        p = f"{name}/"
        out[p + "params"] = np.array([h, w, use_h, use_w, rotate, offset, round(ratio * 1000), mode,
                                      round(prob * 1000), training, seed], np.int64)
        out[p + "draws"] = np.array(draws, np.int64)
        out[p + "state_keys"] = state[1].astype(np.uint32)
        out[p + "state_pos"] = np.array(state[2], np.int64)
        if h * w <= SMALL:
            x = torch.randint(-8, 9, (1, 2, h, w), generator=g) / 4.0           # few bits per value: a small file
            x[0, 0, 0, :3] = torch.tensor([float("inf"), -float("inf"), float("nan")])
            x[0, 1, -1, -1] = -0.0
            out[p + "x"] = x.numpy()
            for dt, key in ((torch.float32, "out_f32"), (torch.float16, "out_f16"), (torch.bfloat16, "out_bf16")):
                y2, _, state2 = run(m, x.to(dt), seed)
                assert (state2[1] == state[1]).all() and state2[2] == state[2]
                y2 = y2.contiguous()
                out[p + key] = y2.numpy() if dt == torch.float32 else y2.view(torch.int16).numpy()
    out["sig/init"] = np.array(str(inspect.signature(GridMask.__init__)))
    out["sig/set_prob"] = np.array(str(inspect.signature(GridMask.set_prob)))
    out["sig/attrs"] = np.array(sorted(k for k in vars(GridMask(True, True)) if not k.startswith("_")))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
