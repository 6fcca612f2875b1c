"""Corner-pair records of the tile-aggregating rows backward (msda_backward_tile_kernel in csrc/msda.cu).  A record
holds the two horizontally adjacent corners of one row of a sample, keyed by the left pixel's slot in the level's
rows padded by one column in front, and the sorted-run pass keeps accumulators for two neighbouring slots.  These
cases put pairs where that bookkeeping can go wrong: cut by every image border, on levels one pixel wide or high, in
runs of consecutive slots across the 64-record group segments, and at the end of an image row next to the
following row's first pixel.  MSDARowsFunction is checked against the fp64 oracle and against the plain op
(grad_sampling_loc / grad_attn_weight bit-identical, grad_value at 1e-5), SCARowsFunction, which shares the kernel,
against the oracle and the fused plain op."""
import pytest
import torch

from tests.inputs import SCA_LEVELS
from tests.test_msda_rows_gpu import _check, _check_sca, _inputs, _inv
from vidar_b200 import sca

pytestmark = pytest.mark.gpu

CAMS, QD, H, P = 2, 600, 8, 8
THIN = ((40, 1), (1, 40), (16, 16), (8, 8))         # a level one pixel wide and one one pixel high


def _run(dev, levels, px, py, seed):
    """px, py [cams, Qd, H, L, P] pixel coordinates -> MSDARowsFunction against the oracle and the plain op"""
    shapes, lsi, (value, _, attn) = _inputs(dev, CAMS, QD, "local", seed, levels)
    wh = torch.tensor([[w, h] for h, w in levels], dtype=torch.float64).view(1, 1, 1, len(levels), 1, 2)
    loc = ((torch.stack([px, py], -1) + 0.5) / wh).float().to(dev)
    _check(dev, sca.unit_plan(1, 0, CAMS), 1, QD, [(value, loc, attn)], shapes, lsi, inv=_inv(dev, 1, QD, seed + 1))


def _frac(gen, shape):
    """fractional pixel parts off the pixel-centre lines"""
    return 0.05 + 0.9 * torch.rand(shape, generator=gen, dtype=torch.float64)


def _border(size, gen, shape):
    """pixel coordinates whose floor is -1, size - 1 or an inner pixel, a third each"""
    pick = torch.randint(0, 3, shape, generator=gen)
    inner = torch.randint(0, max(size - 1, 1), shape, generator=gen).double()
    base = torch.where(pick == 0, -1.0, torch.where(pick == 1, float(size - 1), inner))
    return base + _frac(gen, shape)


def _per_level(levels, fn):
    """stack fn(l, Hl, Wl) -> (px, py) [cams, Qd, H, P] over the levels"""
    xs, ys = zip(*(fn(l, hl, wl) for l, (hl, wl) in enumerate(levels)))
    return torch.stack(xs, 3), torch.stack(ys, 3)


@pytest.mark.parametrize("levels", [SCA_LEVELS, THIN], ids=["sca", "thin"])
def test_pairs_cut_by_borders(cuda, levels):
    """w_low = -1 (no left corner), w_low = Wl - 1 (no right corner), h_low = -1 (no top pair), h_low = Hl - 1 (no
    bottom pair) and inner pixels in every combination; on the thin levels every pair is cut."""
    gen = torch.Generator().manual_seed(200)
    shape = (CAMS, QD, H, P)
    px, py = _per_level(levels, lambda l, hl, wl: (_border(wl, gen, shape), _border(hl, gen, shape)))
    _run(cuda, levels, px, py, 201)


def test_runs_across_group_segments(cuda):
    """Every row samples one image row band: even heads spread over 130 consecutive pixels (runs of ~16 pairs per
    slot, so segment boundaries fall between consecutive slots), odd heads over 4 pixels (runs that span several
    64-record segments)."""
    gen = torch.Generator().manual_seed(210)
    shape = (CAMS, QD, H, P)
    width = torch.tensor([130.0 if h % 2 == 0 else 4.0 for h in range(H)], dtype=torch.float64).view(1, 1, H, 1)

    def level(l, hl, wl):
        x0, y0 = float(wl // 10), float(int(0.4 * hl))
        w = torch.clamp(width, max=wl - x0 - 1)
        px = x0 + torch.floor(torch.rand(shape, generator=gen, dtype=torch.float64) * w) + _frac(gen, shape)
        return px, y0 + _frac(gen, shape)
    px, py = _per_level(SCA_LEVELS, level)
    _run(cuda, SCA_LEVELS, px, py, 211)


def test_row_end_next_to_next_row_start(cuda):
    """Samples at the last pixel column of rows 10..12 (their right corner is outside: in an unpadded index it would
    be the next row's first pixel) mixed with samples at w_low = -1 and w_low = 0 of the same and following rows."""
    gen = torch.Generator().manual_seed(220)
    shape = (CAMS, QD, H, P)

    def level(l, hl, wl):
        pick = torch.randint(0, 3, shape, generator=gen)
        base = torch.where(pick == 0, float(wl - 1), torch.where(pick == 1, -1.0, 0.0))
        row = torch.randint(min(10, hl - 2), min(13, hl - 1), shape, generator=gen).double()
        return base + _frac(gen, shape), row + _frac(gen, shape)
    px, py = _per_level(SCA_LEVELS, level)
    _run(cuda, SCA_LEVELS, px, py, 221)


def test_sca_rows_thin_levels(cuda):
    """SCARowsFunction (the fused-epilogue instantiation of the tile kernel) on the thin levels."""
    cams = 3
    _check_sca(cuda, cams, QD, sca.unit_plan(1, 0, cams), inv=_inv(cuda, 1, QD, 231), seed=230, levels=THIN)
