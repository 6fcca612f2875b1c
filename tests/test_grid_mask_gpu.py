"""GridMask on the H100 (csrc/grid_mask.cu through vidar_b200.grid_mask): bit for bit the oracle
(oracle/grid_mask_ref.py) and the reference module's outputs (tests/golden/grid_mask.npz) in every dtype, mode, stripe
set, rotation and offset setting, on vector and scalar paths; the prob gate and eval mode return the input; the
gradient is grad_out * mask; no host sync; and the synthetic pre-training harness masks the current frame's images
exactly as the reference's statements do."""
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import grid_mask_ref as ref
from vidar_b200 import _lib, grid_mask
from vidar_b200.grid_mask import GridDraw, GridMask, grid_mask_apply

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grid_mask.npz")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def same_bits(got, want, what):
    """Bitwise equal, except that any NaN matches any NaN (x86 and CUDA make NaNs of different sign)."""
    g, w = got.detach().cpu().contiguous().view(-1), want.contiguous().view(-1)
    assert g.dtype == w.dtype, what
    nan_g, nan_w = torch.isnan(g.float()), torch.isnan(w.float())
    assert torch.equal(nan_g, nan_w), f"{what}: NaN positions differ"
    bits = {4: torch.int32, 2: torch.int16}[g.element_size()]
    bad = (g[~nan_g].view(bits) != w[~nan_w].view(bits)).sum().item()
    assert bad == 0, f"{what}: {bad} values differ"


def inputs(n, c, h, w, dtype, seed):
    """Quarter steps in [-4, 4] with inf, -inf, NaN and -0.0 in fixed places, on the CPU."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randint(-16, 17, (n, c, h, w), generator=g) / 4.0)
    x.view(-1)[:4] = torch.tensor([float("inf"), -float("inf"), float("nan"), -0.0])
    return x.to(dtype)


def oracle(x, draw, use_h, use_w, mode):
    h, w = x.shape[-2:]
    m = ref.grid_mask(h, w, draw.d, draw.l, draw.st_h, draw.st_w, draw.r, use_h, use_w, mode)
    return ref.apply(x, m, draw.offset), m


def device_offset(draw, dtype, dev):
    return None if draw.offset is None else torch.from_numpy(draw.offset).to(dtype).to(dev)


@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_equals_oracle_at_every_setting(cuda, dtype):
    """dtype x mode x use_h / use_w x rotation x offset on aligned, odd-width and misaligned buffers."""
    rng = np.random.default_rng(0)
    shapes = [(2, 3, 58, 100), (1, 2, 57, 99), (1, 3, 3, 8), (2, 1, 40, 40)]
    count = 0
    for (n, c, h, w), mode, use_h, use_w, r, with_offset in itertools.product(
            shapes, (0, 1), (False, True), (False, True), (0, 37, 90, 180, 271), (False, True)):
        d = int(rng.integers(2, h))
        draw = GridDraw(d, min(max(int(d * 0.5 + 0.5), 1), d - 1), int(rng.integers(d)), int(rng.integers(d)), r,
                        2 * (rng.random((h, w)) - 0.5) if with_offset else None)
        x = inputs(n, c, h, w, dtype, count)
        want, _ = oracle(x, draw, use_h, use_w, mode)
        what = f"{dtype} {(n, c, h, w)} mode {mode} use {use_h, use_w} r {r} offset {with_offset}"
        got = grid_mask_apply(x.to(cuda), draw, use_h, use_w, mode, device_offset(draw, dtype, cuda))
        same_bits(got, want, what)
        # misaligned: views one element into their storage take the scalar path
        xs = torch.empty(x.numel() + 1, dtype=dtype, device=cuda)[1:].view(x.shape).copy_(x)
        off = device_offset(draw, dtype, cuda)
        if off is not None:
            off = torch.empty(off.numel() + 1, dtype=dtype, device=cuda)[1:].view(off.shape).copy_(off)
        same_bits(grid_mask_apply(xs, draw, use_h, use_w, mode, off), want, what + " misaligned")
        count += 1
    assert count == 4 * 2 * 4 * 5 * 2


def test_every_integer_angle(cuda):
    """All 360 angles (and 360, 725, -3) on a non-square and a square frame: the host's Pillow coefficients."""
    for (h, w) in ((31, 47), (40, 40)):
        x = inputs(1, 2, h, w, torch.float32, h)
        for r in list(range(361)) + [725, -3]:
            draw = GridDraw(9, 4, 3, 5, r)
            want, _ = oracle(x, draw, True, True, 0)
            same_bits(grid_mask_apply(x.to(cuda), draw, True, True, 0), want, f"{h}x{w} r {r}")


def test_module_equals_the_reference_golden(cuda):
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files if k.endswith("/params")})
    checked = 0
    for name in names:
        h, w, use_h, use_w, rotate, offset, ratio, mode, prob, training, seed = (int(v) for v in z[f"{name}/params"])
        m = GridMask(bool(use_h), bool(use_w), rotate=rotate, offset=bool(offset), ratio=ratio / 1000, mode=mode,
                     prob=prob / 1000).train(bool(training))
        if f"{name}/mask" in z.files:          # x = ones gives the mask (offset off) or mask + offset * (1 - mask)
            np.random.seed(seed)
            y = m(torch.ones(1, 1, h, w, device=cuda))
            want = np.unpackbits(z[f"{name}/mask"], count=h * w).reshape(h, w)
            assert ((y[0, 0] == 1).cpu().numpy() == want.astype(bool)).all(), name
            checked += 1
        if f"{name}/x" not in z.files:
            continue
        x = torch.from_numpy(z[f"{name}/x"])
        for dt, key in ((torch.float32, "out_f32"), (torch.float16, "out_f16"), (torch.bfloat16, "out_bf16")):
            np.random.seed(seed)
            xd = x.to(dt).to(cuda)
            y = m(xd)
            want = torch.from_numpy(z[f"{name}/{key}"])
            same_bits(y, want if dt == torch.float32 else want.view(dt), f"{name} {dt}")
            assert (y is xd) == (len(z[f"{name}/draws"]) == 0), name
            state = np.random.get_state()
            assert (state[1] == z[f"{name}/state_keys"]).all() and state[2] == int(z[f"{name}/state_pos"]), name
            checked += 1
    assert checked >= 40


def test_prob_gate_and_eval_return_the_input_object(cuda):
    x = torch.randn(2, 3, 16, 16, device=cuda)
    n0 = _lib.launch_count()
    np.random.seed(0)
    assert GridMask(True, True, prob=0.0)(x) is x
    assert GridMask(True, True, offset=True).eval()(x) is x
    assert _lib.launch_count() == n0
    m = GridMask(True, True, prob=1.0)
    np.random.seed(0)
    assert m(x) is not x and _lib.launch_count() == n0 + 1


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("offset", [False, True])
def test_gradient_is_grad_out_times_mask(cuda, dtype, offset):
    m = GridMask(True, True, rotate=360, offset=offset, mode=1)
    x = inputs(2, 3, 58, 100, dtype, 5).to(cuda).requires_grad_(True)
    np.random.seed(7)
    y = m(x)
    g = inputs(2, 3, 58, 100, dtype, 6)
    n0 = _lib.launch_count()
    y.backward(g.to(cuda))
    assert _lib.launch_count() == n0 + 1                       # the same launch, no other kernel of ours
    np.random.seed(7)
    draw = m.sample(58, 100)
    mask = ref.grid_mask(58, 100, draw.d, draw.l, draw.st_h, draw.st_w, draw.r, True, True, 1)
    same_bits(x.grad, g * torch.from_numpy(mask).to(dtype), f"grad {dtype} offset {offset}")


@pytest.mark.parametrize("offset", [False, True])
def test_no_host_sync(cuda, offset):
    m = GridMask(True, True, rotate=360, offset=offset, mode=1)
    x = torch.randn(6, 3, 116, 200, device=cuda, requires_grad=True)
    m(x).sum()                                                  # warm up: module load, pinned allocator
    torch.cuda.synchronize()
    np.random.seed(1)
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = m(x)
        y.backward(torch.ones_like(y))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert y is not x


def test_pretrain_harness_masks_the_current_frame_like_the_reference(cuda):
    """The backbone's first conv sees, for the current frame, the reference's statements applied to the images with
    the same numpy seed (the history's eval-mode gate draw first), and the history frames unmasked."""
    from vidar_b200 import pretrain
    small = dict(encoder_layers=1, decoder_layers=1, future_frames=1, bev_hw=(20, 20), ray_grid_num=32,
                 grid_mask=True)
    model, opt = pretrain.build(cuda, None, seed=1, **small)
    model.grid_mask.prob = 1.0                                  # the cfg's 0.7 gate: open it for the comparison
    sample = pretrain.synthetic_sample(cuda, frames=3, img_hw=(64, 96), rays_per_frame=300, future_frames=1,
                                       bev_hw=(20, 20))
    seen = []
    hook = model.backbone.stem[0].register_forward_hook(lambda mod, inp, out: seen.append(inp[0].detach().clone()))
    np.random.seed(123)
    loss, _ = pretrain.train_step(model, opt, sample)
    hook.remove()
    assert torch.isfinite(loss)
    img = sample["img"][0]                                      # [frames, cams, 3, H, W]
    assert len(seen) == 3
    for t in range(2):
        assert torch.equal(seen[t], img[t])
    # the reference's statements (grid_mask.py:86-124) on the current frame, with the same seed
    np.random.seed(123)
    np.random.rand()                                            # obtain_history_bev's eval-mode call
    np.random.rand()                                            # the current frame's gate (prob 1 here)
    d = np.random.randint(2, img.shape[-2])
    l = min(max(int(d * 0.5 + 0.5), 1), d - 1)  # noqa: E741
    st_h, st_w, r = np.random.randint(d), np.random.randint(d), np.random.randint(1)
    mask = ref.pil_mask(*img.shape[-2:], d, l, st_h, st_w, r, True, True, 1)
    mask = torch.from_numpy(mask).to(img.dtype).to(cuda)
    want = img[2] * mask.expand_as(img[2])
    assert torch.equal(seen[2], want)
    assert not torch.equal(want, img[2])
    # the default harness has no mask and draws nothing
    model2, _ = pretrain.build(cuda, None, seed=1, **dict(small, grid_mask=False))
    assert model2.grid_mask is None
    assert grid_mask.GridMask not in {type(m) for m in model2.modules()}
