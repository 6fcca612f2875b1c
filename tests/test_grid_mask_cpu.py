"""GridMask without a GPU: the numpy oracle (oracle/grid_mask_ref.py) against PIL's `Image.rotate` and against the
reference module's own masks and outputs (tests/golden/grid_mask.npz, written by tools/make_golden_grid_mask.py),
the module's numpy draws against the reference's RNG stream, every argument check of vidar_b200.grid_mask, and its
signatures and attributes against the reference class."""
import inspect
import os

import numpy as np
import pytest
import torch

from oracle import grid_mask_ref as ref
from vidar_b200 import _lib, grid_mask

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grid_mask.npz")
ANGLES = [0, 1, 7, 30, 45, 89, 90, 91, 135, 180, 181, 200, 270, 271, 359, 360]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def golden_cases(z):
    return sorted({k.split("/")[0] for k in z.files if k.endswith("/params")})


def case_module(z, name):
    """(GridMask built from the case's params, h, w, seed)."""
    h, w, use_h, use_w, rotate, offset, ratio, mode, prob, training, seed = (int(v) for v in z[f"{name}/params"])
    m = grid_mask.GridMask(bool(use_h), bool(use_w), rotate=rotate, offset=bool(offset), ratio=ratio / 1000,
                           mode=mode, prob=prob / 1000)
    return m.train(bool(training)), h, w, seed


def pil_rotate(img, angle):
    from PIL import Image
    return np.asarray(Image.fromarray(img).rotate(angle))


@pytest.mark.parametrize("hw", [(87, 150), (300, 451), (301, 300), (300, 300), (87, 87), (3, 10), (1, 1)])
def test_oracle_rotation_equals_pil_at_every_integer_angle(hw):
    img = (np.random.default_rng(hw[0] * 1000 + hw[1]).random(hw) < 0.5).astype(np.uint8)
    for angle in range(-1, 362):
        np.testing.assert_array_equal(ref.rotate_nearest(img, angle), pil_rotate(img, angle), err_msg=f"angle {angle}")


@pytest.mark.parametrize("hw", [(1392, 2400), (87, 3000), (1393, 2401)])
def test_oracle_rotation_equals_pil_on_large_frames(hw):
    img = (np.random.default_rng(0).random(hw) < 0.5).astype(np.uint8)
    for angle in ANGLES:
        np.testing.assert_array_equal(ref.rotate_nearest(img, angle), pil_rotate(img, angle), err_msg=f"angle {angle}")


def test_oracle_equals_the_reference_construction():
    """The stripe test at the rotated pixel against the stripes written into a frame, rotated by PIL and cropped."""
    rng = np.random.default_rng(3)
    for h, w in ((58, 100), (57, 99), (200, 200), (3, 8), (31, 47)):
        for _ in range(40):
            d = int(rng.integers(2, h))
            l = int(rng.integers(0, d + 1))  # noqa: E741
            st_h, st_w, r = int(rng.integers(d)), int(rng.integers(d)), int(rng.integers(360))
            use_h, use_w, mode = (bool(v) for v in rng.integers(0, 2, 3))
            args = (h, w, d, l, st_h, st_w, r, use_h, use_w, int(mode))
            np.testing.assert_array_equal(ref.grid_mask(*args), ref.pil_mask(*args), err_msg=str(args))


def test_golden_covers_the_cases(golden):
    names = golden_cases(golden)
    draws = {n: golden[f"{n}/draws"] for n in names}
    assert any(len(d) and d[0] == 2 for d in draws.values())                          # the smallest period
    assert any(len(d) and d[1] == d[0] - 1 and d[0] > 2 for d in draws.values())      # l clamped to d - 1
    assert any(len(d) and d[4] % 90 for d in draws.values())                          # a true rotation
    assert {"gate_closed", "eval", "cfg_928x1600"} <= set(names)


def test_module_draws_follow_the_reference_rng_stream(golden):
    """Seeded like the reference's call, `sample` returns its draws and leaves numpy in the state it left."""
    for name in golden_cases(golden):
        m, h, w, seed = case_module(golden, name)
        np.random.seed(seed)
        draw = m.sample(h, w)
        want = golden[f"{name}/draws"]
        if len(want) == 0:
            assert draw is None, name
        else:
            assert [draw.d, draw.l, draw.st_h, draw.st_w, draw.r] == want.tolist(), name
            assert m.l == want[1]
            assert (draw.offset is not None) == bool(m.offset)
        state = np.random.get_state()
        np.testing.assert_array_equal(state[1], golden[f"{name}/state_keys"], err_msg=name)
        assert state[2] == int(golden[f"{name}/state_pos"]), name


def _same_bits(got, want, name):
    """Bitwise equal, except that any NaN matches any NaN (x86 and CUDA make NaNs of different sign)."""
    g, w = got.contiguous().view(-1), want.contiguous().view(-1)
    nan_g, nan_w = torch.isnan(g.float()), torch.isnan(w.float())
    assert torch.equal(nan_g, nan_w), name
    bits = {4: torch.int32, 2: torch.int16}[g.element_size()]
    assert torch.equal(g[~nan_g].view(bits), w[~nan_w].view(bits)), name


def test_oracle_equals_golden_masks_and_outputs(golden):
    checked = 0
    for name in golden_cases(golden):
        if len(golden[f"{name}/draws"]) == 0:
            continue
        m, h, w, seed = case_module(golden, name)
        np.random.seed(seed)
        draw = m.sample(h, w)
        mask = ref.grid_mask(h, w, draw.d, draw.l, draw.st_h, draw.st_w, draw.r, m.use_h, m.use_w, m.mode)
        want = np.unpackbits(golden[f"{name}/mask"], count=h * w).reshape(h, w)
        np.testing.assert_array_equal(mask, want, err_msg=name)
        if f"{name}/x" not in golden.files:
            continue
        x = torch.from_numpy(golden[f"{name}/x"])
        for dt, key in ((torch.float32, "out_f32"), (torch.float16, "out_f16"), (torch.bfloat16, "out_bf16")):
            want = torch.from_numpy(golden[f"{name}/{key}"])
            want = want if dt == torch.float32 else want.view(dt)
            _same_bits(ref.apply(x.to(dt), mask, draw.offset), want, f"{name} {dt}")
            checked += 1
    assert checked >= 30


def test_gate_and_eval_return_the_input_itself_without_touching_cuda(monkeypatch):
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    x = torch.zeros(1, 1, 5, 5)          # a CPU tensor: returned before any check, as the reference returns it
    m = grid_mask.GridMask(True, True, prob=0.0)
    np.random.seed(0)
    assert m(x) is x
    m = grid_mask.GridMask(True, True, offset=True).eval()
    np.random.seed(0)
    assert m(x) is x
    pos = np.random.get_state()[2]
    np.random.seed(0)
    np.random.rand()
    assert pos == np.random.get_state()[2]          # one rand() for the prob gate, in eval mode too


@pytest.mark.parametrize("x, exc, match", [
    (torch.zeros(2, 5, 5), ValueError, "4-D"),
    (torch.zeros(1, 1, 5, 5, dtype=torch.float64), TypeError, "float32, float16 or bfloat16"),
    (torch.zeros(1, 1, 5, 5, dtype=torch.int32), TypeError, "float32, float16 or bfloat16"),
    (torch.zeros(1, 1, 2, 5), ValueError, "image size"),
    (torch.zeros(1, 1, 5, 8193), ValueError, "image size"),
    (torch.zeros(1, 1, 5, 5), RuntimeError, "must be a CUDA tensor"),
    ("not a tensor", TypeError, "must be a tensor"),
])
def test_argument_checks_run_before_any_cuda_call(monkeypatch, x, exc, match):
    monkeypatch.setattr(_lib, "lib", lambda: pytest.fail("the library was loaded"))
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a: pytest.fail("pinned memory was allocated"))
    m = grid_mask.GridMask(True, True, rotate=360, offset=True)
    np.random.seed(0)
    with pytest.raises(exc, match=match):
        m(x)
    np.random.seed(0)
    with pytest.raises(exc, match=match):
        m.masked(x, grid_mask.GridDraw(2, 1, 0, 0, 0, np.zeros((5, 5))))


def test_signatures_and_attributes_match_the_reference_class(golden):
    assert str(inspect.signature(grid_mask.GridMask.__init__)) == str(golden["sig/init"])
    assert str(inspect.signature(grid_mask.GridMask.set_prob)) == str(golden["sig/set_prob"])
    m = grid_mask.GridMask(True, True)
    attrs = sorted(k for k in vars(m) if not k.startswith("_"))
    assert attrs == golden["sig/attrs"].tolist()
    m = grid_mask.GridMask(True, False, prob=0.7)
    m.set_prob(3, 4)
    assert m.prob == 0.7 * 3 / 4 and m.st_prob == 0.7


def test_dtype_codes_match_the_header():
    with open(_lib.HEADER) as fh:
        src = fh.read()
    assert "VIDAR_DTYPE_F32 = 0" in src and "VIDAR_DTYPE_F16 1" in src and "VIDAR_DTYPE_BF16 2" in src
    assert grid_mask.DTYPE_CODES == {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def test_c_entry_point_rejects_bad_arguments_before_any_launch():
    """Pointers are only compared with NULL (or checked for alignment) before a launch, so a dummy address stands
    in for device memory; every call here fails validation and launches nothing."""
    import ctypes
    L = _lib.lib()
    X, N = ctypes.c_void_p(0x1000), None
    ok = dict(x=X, offset=N, out=X, dtype=0, N=1, C=3, h=8, w=8, d=4, l=2, st_h=0, st_w=1, r=0, use_h=1, use_w=1,
              mode=0)
    cases = [
        (dict(x=N), b"null pointer"),
        (dict(dtype=3), b"unsupported dtype"),
        (dict(h=0), b"bad sizes"),
        (dict(w=8193), b"bad sizes"),
        (dict(N=-1), b"bad sizes"),
        (dict(d=1), b"bad draw"),
        (dict(l=5), b"bad draw"),
        (dict(st_w=4), b"bad draw"),
        (dict(mode=2), b"must be 0 or 1"),
        (dict(use_h=2), b"must be 0 or 1"),
        (dict(out=ctypes.c_void_p(0x1002)), b"aligned"),
        (dict(dtype=1, offset=ctypes.c_void_p(0x1001)), b"aligned"),
    ]
    n0 = _lib.launch_count()
    for change, needle in cases:
        a = dict(ok, **change)
        rc = L.vidar_grid_mask_apply(a["x"], a["offset"], a["out"], a["dtype"], a["N"], a["C"], a["h"], a["w"],
                                     a["d"], a["l"], a["st_h"], a["st_w"], a["r"], a["use_h"], a["use_w"], a["mode"],
                                     None)
        assert rc == 1, (change, rc)
        assert needle in L.vidar_last_error(), (change, L.vidar_last_error())
    assert _lib.launch_count() == n0
