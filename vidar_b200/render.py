"""Voxel ray-caster op boundary (dvr / dvxlr / dvxlr_v2), H100-native.

Drop-in for the reference's JIT-compiled pybind modules and their autograd wrappers:

  * ``dvr``      -- ``init``, ``render``, ``render_forward``      (third_lib/dvr/dvr.cpp:65-69)
  * ``dvxlr``    -- ``init``, ``render``, ``get_grad_sigma``      (third_lib/dvxlr/dvxlr.cpp:61-65)
  * ``dvxlr_v2`` -- ``render_v2``, ``get_grad_sigma_v2``          (third_lib/dvxlr/dvxlr_v2.cpp:67-70)
    same positional arguments, same returned lists of tensors, all fp32 (tindex and indices
    included), CUDA + contiguous inputs required (dvr.cpp:28-34);
  * ``DifferentiableVoxelRendering`` / ``...V2`` (+ ``...Layer`` classes)
    (projects/mmdet3d_plugin/bevformer/utils/e2e_predictor_utils.py:91-143), same call
    signature and outputs.  They run the *fused* path: forward produces only what the caller
    sees, backward re-walks the rays and scatters straight into grad_sigma, so the
    [N, M, 1026(, 3)] dd_dsigma / indices lists (0.5 GB at 30k rays) are never written.
    ``DifferentiableVoxelRenderingLayerLists`` keeps the reference's two-step dataflow
    (render -> gradpred*dd_dsigma -> get_grad_sigma) for comparison.

Unknown loss / phase names raise ValueError (the reference prints and calls exit(1),
dvr.cu:362-365, 669-672).  Nothing here synchronises the device (the reference calls
cudaDeviceSynchronize after every launch, dvr.cu:379,688,735; callers do not rely on it).
"""
import types

import torch
from torch.autograd.function import once_differentiable

from . import _lib

MAX_D = 1026  # third_lib/dvxlr/dvxlr.cu:10: third dim of the list outputs

_LOSS = {"l1": 0, "bce": 0, "l2": 1, "absrel": 2}
_PHASE = {"test": 0, "train": 1}


def _check(sigma, origin, points, tindex, **extra):
    _lib.require_cuda(sigma=sigma, origin=origin, points=points, tindex=tindex, **extra)
    for name, t in dict(sigma=sigma, origin=origin, points=points, tindex=tindex, **extra).items():
        if t is not None and t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32 (got {t.dtype})")
    if sigma.dim() != 5 or origin.dim() != 3 or points.dim() != 3 or tindex.dim() != 2:
        raise RuntimeError("expected sigma [N,T,H,L,W], origin [N,T,3], points [N,M,3], tindex [N,M]")
    N, T, Z, Y, X = sigma.shape
    M = points.shape[1]
    To = origin.shape[1]
    if points.shape[0] != N or origin.shape[0] != N or tuple(tindex.shape) != (N, M):
        raise RuntimeError("batch / ray dimensions of sigma, origin, points, tindex disagree")
    return N, M, T, To, Z, Y, X


def _call(fn, device, *args, rays=1):
    if rays == 0:       # empty ray set: outputs keep their initial values (null data_ptr)
        return
    with torch.cuda.device(device):
        _lib.check(fn(*args, _lib.stream_ptr(device)))


def init(points, tindex, grid):
    """dvr.init / dvxlr.init -> occupancy [N, T, H, L, W] (dvr.cu:705-738)."""
    _lib.require_cuda(points=points, tindex=tindex)
    T, Z, Y, X = (int(g) for g in grid)
    N, M = points.shape[:2]
    occ = torch.zeros((N, T, Z, Y, X), dtype=points.dtype, device=points.device)
    if points.dtype != torch.float32 or tindex.dtype != torch.float32:
        raise RuntimeError("points / tindex must be float32")
    _call(_lib.lib().vidar_dvr_init, points.device, _lib.ptr(points), _lib.ptr(tindex),
          _lib.ptr(occ), N, M, T, Z, Y, X, rays=M)
    return occ


def render_forward(sigma, origin, points, tindex, grid, phase_name):
    """dvr.render_forward -> [pred_dist, gt_dist] (dvr.cu:327-383).  `grid` is accepted and,
    as in the reference, unused by the computation."""
    if phase_name not in _PHASE:
        raise ValueError(f"UNKNOWN PHASE NAME: {phase_name}")
    N, M, T, To, Z, Y, X = _check(sigma, origin, points, tindex)
    pred = torch.full((N, M), -1.0, dtype=torch.float32, device=sigma.device)
    gt = torch.full((N, M), -1.0, dtype=torch.float32, device=sigma.device)
    _call(_lib.lib().vidar_dvr_render_forward, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
          _lib.ptr(points), _lib.ptr(tindex), _lib.ptr(pred), _lib.ptr(gt),
          N, M, T, To, Z, Y, X, _PHASE[phase_name], rays=M)
    return [pred, gt]


def render(sigma, origin, points, tindex, loss_name):
    """dvr.render -> [pred_dist, gt_dist, grad_sigma] (dvr.cu:639-694)."""
    if loss_name not in _LOSS:
        raise ValueError(f"UNKNOWN LOSS TYPE: {loss_name}")
    N, M, T, To, Z, Y, X = _check(sigma, origin, points, tindex)
    pred = torch.full((N, M), -1.0, dtype=torch.float32, device=sigma.device)
    gt = torch.full((N, M), -1.0, dtype=torch.float32, device=sigma.device)
    grad_sigma = torch.zeros_like(sigma)
    _call(_lib.lib().vidar_dvr_render, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
          _lib.ptr(points), _lib.ptr(tindex), _lib.ptr(pred), _lib.ptr(gt), _lib.ptr(grad_sigma),
          N, M, T, To, Z, Y, X, _LOSS[loss_name], rays=M)
    return [pred, gt, grad_sigma]


def _dvxlr_render(sigma, origin, points, tindex, sigma_regul=None, lists=True, max_d=MAX_D):
    N, M, T, To, Z, Y, X = _check(sigma, origin, points, tindex, sigma_regul=sigma_regul)
    dev = sigma.device
    if sigma_regul is not None and sigma_regul.shape != sigma.shape:
        raise RuntimeError("sigma_regul must have the shape of sigma")
    pred = torch.full((N, M), -1.0, dtype=torch.float32, device=dev)
    gt = torch.full((N, M), -1.0, dtype=torch.float32, device=dev)
    dd = idx = ray_pred = indicator = None
    if lists:
        dd = torch.zeros((N, M, max_d), dtype=torch.float32, device=dev)
        idx = torch.zeros((N, M, max_d, 3), dtype=torch.float32, device=dev)
    if sigma_regul is not None:
        ray_pred = torch.zeros((N, M, max_d), dtype=torch.float32, device=dev)
        indicator = torch.full((N, M, max_d), -1.0, dtype=torch.float32, device=dev)
    if not lists and sigma_regul is None:
        _call(_lib.lib().vidar_dvxlr_forward, dev, _lib.ptr(sigma), _lib.ptr(origin),
              _lib.ptr(points), _lib.ptr(tindex), _lib.ptr(pred), _lib.ptr(gt),
              N, M, T, To, Z, Y, X, rays=M)
    else:
        _call(_lib.lib().vidar_dvxlr_render, dev, _lib.ptr(sigma), _lib.ptr(origin),
              _lib.ptr(points), _lib.ptr(tindex), _lib.ptr(sigma_regul), _lib.ptr(pred),
              _lib.ptr(gt), _lib.ptr(dd), _lib.ptr(idx), _lib.ptr(ray_pred), _lib.ptr(indicator),
              N, M, T, To, Z, Y, X, max_d, rays=M)
    return pred, gt, dd, idx, ray_pred, indicator


def dvxlr_render(sigma, origin, points, tindex):
    """dvxlr.render -> [pred_dist, gt_dist, dd_dsigma, indices] (dvxlr.cu:469-517)."""
    pred, gt, dd, idx, _, _ = _dvxlr_render(sigma, origin, points, tindex)
    return [pred, gt, dd, idx]


def dvxlr_render_v2(sigma, origin, points, tindex, sigma_regul):
    """dvxlr_v2.render_v2 -> [pred, gt, dd_dsigma, indices, ray_pred, indicator]
    (dvxlr_v2.cu:439-493)."""
    if sigma_regul is None:
        raise RuntimeError("sigma_regul must be a CUDA tensor")
    return list(_dvxlr_render(sigma, origin, points, tindex, sigma_regul))


def _get_grad_sigma(elementwise_mult, indices, tindex, sigma_shape, indicator=None,
                    grad_ray_pred=None):
    _lib.require_cuda(elementwise_mult=elementwise_mult, indices=indices, tindex=tindex,
                      sigma_shape=sigma_shape, indicator=indicator, grad_ray_pred=grad_ray_pred)
    N, T, Z, Y, X = sigma_shape.shape
    M, max_d = elementwise_mult.shape[1], elementwise_mult.shape[2]
    if tuple(indices.shape) != (N, M, max_d, 3):
        raise RuntimeError("indices must be [N, M, MAX_D, 3]")
    g = torch.zeros_like(sigma_shape)
    g2 = torch.zeros_like(sigma_shape) if indicator is not None else None
    _call(_lib.lib().vidar_dvxlr_get_grad_sigma, sigma_shape.device, _lib.ptr(elementwise_mult),
          _lib.ptr(indices), _lib.ptr(tindex), _lib.ptr(indicator), _lib.ptr(grad_ray_pred),
          _lib.ptr(g), _lib.ptr(g2), N, M, T, Z, Y, X, max_d, rays=M)
    return [g] if g2 is None else [g, g2]


def dvxlr_get_grad_sigma(elementwise_mult, indices, tindex, sigma_shape):
    """dvxlr.get_grad_sigma -> [grad_sigma] (dvxlr.cu:123-156); `sigma_shape` is a tensor
    used for its shape/dtype only."""
    return _get_grad_sigma(elementwise_mult, indices, tindex, sigma_shape)


def dvxlr_get_grad_sigma_v2(elementwise_mult, indices, tindex, sigma_shape, indicator,
                            grad_ray_pred):
    """dvxlr_v2.get_grad_sigma_v2 -> [grad_sigma, grad_sigma_regul] (dvxlr_v2.cu:78-115)."""
    return _get_grad_sigma(elementwise_mult, indices, tindex, sigma_shape, indicator,
                           grad_ray_pred.contiguous())


def _backward_fused(sigma, origin, points, tindex, grad_pred, grad_ray_pred=None, max_d=MAX_D):
    N, M, T, To, Z, Y, X = _check(sigma, origin, points, tindex)
    grad_sigma = torch.zeros_like(sigma)
    grad_regul = torch.zeros_like(sigma) if grad_ray_pred is not None else None
    grad_pred = grad_pred.float().contiguous()
    if grad_ray_pred is not None:
        grad_ray_pred = grad_ray_pred.float().contiguous()
    _call(_lib.lib().vidar_dvxlr_backward_fused, sigma.device, _lib.ptr(sigma), _lib.ptr(origin),
          _lib.ptr(points), _lib.ptr(tindex), _lib.ptr(grad_pred), _lib.ptr(grad_ray_pred),
          _lib.ptr(grad_sigma), _lib.ptr(grad_regul), N, M, T, To, Z, Y, X, max_d, rays=M)
    return grad_sigma, grad_regul


# pybind-module look-alikes -----------------------------------------------------------------
dvr = types.SimpleNamespace(init=init, render=render, render_forward=render_forward)
dvxlr = types.SimpleNamespace(init=init, render=dvxlr_render, get_grad_sigma=dvxlr_get_grad_sigma)
dvxlr_v2 = types.SimpleNamespace(render_v2=dvxlr_render_v2, get_grad_sigma_v2=dvxlr_get_grad_sigma_v2)


class DifferentiableVoxelRenderingLayer(torch.autograd.Function):
    """e2e_predictor_utils.py:91-112, fused (no per-ray lists)."""

    @staticmethod
    def forward(ctx, sigma, origin, points, tindex):
        pred_dist, gt_dist, _, _, _, _ = _dvxlr_render(sigma, origin, points, tindex, lists=False)
        ctx.save_for_backward(sigma, origin, points, tindex)
        ctx.mark_non_differentiable(gt_dist)
        return pred_dist, gt_dist

    @staticmethod
    @once_differentiable
    def backward(ctx, gradpred, gradgt):
        sigma, origin, points, tindex = ctx.saved_tensors
        grad_sigma, _ = _backward_fused(sigma, origin, points, tindex, gradpred)
        return grad_sigma, None, None, None


class DifferentiableVoxelRenderingLayerLists(torch.autograd.Function):
    """The reference's own dataflow (render -> lists -> get_grad_sigma), e2e_predictor_utils.py:91-112."""

    @staticmethod
    def forward(ctx, sigma, origin, points, tindex):
        pred_dist, gt_dist, dd_dsigma, indices = dvxlr.render(sigma, origin, points, tindex)
        ctx.save_for_backward(dd_dsigma, indices, tindex, sigma)
        ctx.mark_non_differentiable(gt_dist)
        return pred_dist, gt_dist

    @staticmethod
    @once_differentiable
    def backward(ctx, gradpred, gradgt):
        dd_dsigma, indices, tindex, sigma_shape = ctx.saved_tensors
        elementwise_mult = gradpred[..., None] * dd_dsigma
        elementwise_mult = torch.nan_to_num(elementwise_mult, nan=0.0, posinf=float("inf"),
                                            neginf=float("-inf"))
        grad_sigma = dvxlr.get_grad_sigma(elementwise_mult, indices, tindex, sigma_shape)[0]
        return grad_sigma, None, None, None


class DifferentiableVoxelRenderingLayerV2(torch.autograd.Function):
    """e2e_predictor_utils.py:122-141, fused: ray_pred / indicator are produced (the caller
    consumes them), dd_dsigma / indices are not."""

    @staticmethod
    def forward(ctx, sigma, origin, points, tindex, sigma_regul):
        pred_dist, gt_dist, _, _, ray_pred, indicator = _dvxlr_render(
            sigma, origin, points, tindex, sigma_regul.contiguous(), lists=False)
        ctx.save_for_backward(sigma, origin, points, tindex)
        ctx.mark_non_differentiable(gt_dist, indicator)
        return pred_dist, gt_dist, ray_pred, indicator

    @staticmethod
    @once_differentiable
    def backward(ctx, gradpred, gradgt, grad_ray_pred, grad_indicator):
        sigma, origin, points, tindex = ctx.saved_tensors
        grad_sigma, grad_sigma_regul = _backward_fused(sigma, origin, points, tindex, gradpred,
                                                       grad_ray_pred)
        return grad_sigma, None, None, None, grad_sigma_regul


DifferentiableVoxelRendering = DifferentiableVoxelRenderingLayer.apply
DifferentiableVoxelRenderingV2 = DifferentiableVoxelRenderingLayerV2.apply
