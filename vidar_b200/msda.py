"""Multi-scale deformable attention op boundary, H100-native.

Drop-in for projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py
of the reference:

  * ``ext_module.ms_deform_attn_forward / ms_deform_attn_backward`` -- same names, argument
    order, keyword (``im2col_step=``) and in-place contract as mmcv's ``_ext`` (reference
    call sites :42-48, :74-84, :118-124, :150-160);
  * ``MultiScaleDeformableAttnFunction_fp32`` / ``_fp16`` -- same ``apply`` signature and
    returned gradients ``(grad_value, None, None, grad_loc, grad_attn, None)`` (:162-163).

The arithmetic runs in vidar_b200/csrc/msda.cu through the C ABI (include/vidar_b200.h).
No CPU path: CPU tensors raise, as mmcv's CUDA op does.
"""
import torch
from torch.autograd.function import Function, once_differentiable

from . import _lib


def _dims(value, sampling_locations, attention_weights, spatial_shapes, level_start_index):
    if value.dim() != 4:
        raise RuntimeError(f"value must be [bs, num_keys, num_heads, dim], got {tuple(value.shape)}")
    if sampling_locations.dim() != 6 or sampling_locations.shape[-1] != 2:
        raise RuntimeError("sampling_locations must be [bs, num_queries, num_heads, num_levels, num_points, 2]")
    B, K, H, Cd = value.shape
    Bq, Q, Hq, L, P, _ = sampling_locations.shape
    if (Bq, Hq) != (B, H):
        raise RuntimeError("sampling_locations batch/heads do not match value")
    if tuple(attention_weights.shape) != (B, Q, H, L, P):
        raise RuntimeError(f"attention_weights must be {(B, Q, H, L, P)}, got {tuple(attention_weights.shape)}")
    if tuple(spatial_shapes.shape) != (L, 2) or level_start_index.numel() != L:
        raise RuntimeError("spatial_shapes must be [num_levels, 2] and level_start_index [num_levels]")
    if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
        raise RuntimeError("spatial_shapes / level_start_index must be int64 tensors")
    return B, K, H, Cd, L, Q, P


def ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index,
                           sampling_locations, attention_weights, im2col_step=64):
    """-> Tensor[bs, num_queries, num_heads*dim] (fp32).  All tensors CUDA + contiguous."""
    _lib.require_cuda(value=value, value_spatial_shapes=value_spatial_shapes,
                      value_level_start_index=value_level_start_index,
                      sampling_locations=sampling_locations, attention_weights=attention_weights)
    for name, t in (("value", value), ("sampling_locations", sampling_locations),
                    ("attention_weights", attention_weights)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32 (got {t.dtype})")
    B, K, H, Cd, L, Q, P = _dims(value, sampling_locations, attention_weights,
                                 value_spatial_shapes, value_level_start_index)
    _lib.require_aligned(value=value, sampling_locations=sampling_locations, attention_weights=attention_weights)
    out = torch.empty((B, Q, H * Cd), dtype=torch.float32, device=value.device)
    if out.numel() == 0:
        return out
    with torch.cuda.device(value.device):
        _lib.check(_lib.lib().vidar_msda_forward(
            _lib.ptr(value), _lib.ptr(value_spatial_shapes), _lib.ptr(value_level_start_index),
            _lib.ptr(sampling_locations), _lib.ptr(attention_weights), _lib.ptr(out),
            B, K, H, Cd, L, Q, P, int(im2col_step), _lib.stream_ptr(value.device)))
    return out


def ms_deform_attn_backward(value, value_spatial_shapes, value_level_start_index,
                            sampling_locations, attention_weights, grad_output, grad_value,
                            grad_sampling_loc, grad_attn_weight, im2col_step=64):
    """Fills the caller-allocated, caller-zeroed grad_* tensors in place; returns None."""
    _lib.require_cuda(value=value, value_spatial_shapes=value_spatial_shapes,
                      value_level_start_index=value_level_start_index,
                      sampling_locations=sampling_locations, attention_weights=attention_weights,
                      grad_output=grad_output, grad_value=grad_value,
                      grad_sampling_loc=grad_sampling_loc, grad_attn_weight=grad_attn_weight)
    for name, t in (("value", value), ("sampling_locations", sampling_locations),
                    ("attention_weights", attention_weights), ("grad_output", grad_output),
                    ("grad_value", grad_value), ("grad_sampling_loc", grad_sampling_loc),
                    ("grad_attn_weight", grad_attn_weight)):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32 (got {t.dtype})")
    B, K, H, Cd, L, Q, P = _dims(value, sampling_locations, attention_weights,
                                 value_spatial_shapes, value_level_start_index)
    if grad_output.numel() != B * Q * H * Cd:
        raise RuntimeError("grad_output has the wrong number of elements")
    if (grad_value.shape != value.shape or grad_sampling_loc.shape != sampling_locations.shape
            or grad_attn_weight.shape != attention_weights.shape):
        raise RuntimeError("grad_* tensors must have the shapes of value / sampling_locations / attention_weights")
    if grad_output.numel() == 0:
        return None
    _lib.require_aligned(value=value, sampling_locations=sampling_locations, attention_weights=attention_weights,
                         grad_output=grad_output, grad_value=grad_value, grad_sampling_loc=grad_sampling_loc,
                         grad_attn_weight=grad_attn_weight)
    with torch.cuda.device(value.device):
        _lib.check(_lib.lib().vidar_msda_backward(
            _lib.ptr(value), _lib.ptr(value_spatial_shapes), _lib.ptr(value_level_start_index),
            _lib.ptr(sampling_locations), _lib.ptr(attention_weights), _lib.ptr(grad_output),
            _lib.ptr(grad_value), _lib.ptr(grad_sampling_loc), _lib.ptr(grad_attn_weight),
            B, K, H, Cd, L, Q, P, int(im2col_step), _lib.stream_ptr(value.device)))
    return None


class _ExtModule:
    """Stand-in for ``mmcv.utils.ext_loader.load_ext('_ext', [...])``."""
    ms_deform_attn_forward = staticmethod(ms_deform_attn_forward)
    ms_deform_attn_backward = staticmethod(ms_deform_attn_backward)


ext_module = _ExtModule()


def load_ext(name, funcs):
    """``ext_loader.load_ext('_ext', ['ms_deform_attn_backward', 'ms_deform_attn_forward'])``."""
    for f in funcs:
        if not hasattr(ext_module, f):
            raise AttributeError(f"{f} miss in module {name}")
    _lib.lib()
    return ext_module


class MultiScaleDeformableAttnFunction_fp32(Function):
    """multi_scale_deformable_attn_function.py:90-163 (inputs cast to fp32, :93)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index,
                sampling_locations, attention_weights, im2col_step):
        ctx.im2col_step = im2col_step
        ctx.in_dtypes = (value.dtype, sampling_locations.dtype, attention_weights.dtype)
        value = _lib.aligned(value.float().contiguous())
        sampling_locations = _lib.aligned(sampling_locations.float().contiguous())
        attention_weights = _lib.aligned(attention_weights.float().contiguous())
        value_spatial_shapes = value_spatial_shapes.contiguous()
        value_level_start_index = value_level_start_index.contiguous()
        output = ext_module.ms_deform_attn_forward(
            value, value_spatial_shapes, value_level_start_index, sampling_locations,
            attention_weights, im2col_step=ctx.im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index,
                              sampling_locations, attention_weights)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (value, value_spatial_shapes, value_level_start_index, sampling_locations,
         attention_weights) = ctx.saved_tensors
        grad_value = torch.zeros_like(value)
        grad_sampling_loc = torch.empty_like(sampling_locations)   # fully overwritten by the kernel
        grad_attn_weight = torch.empty_like(attention_weights)
        ext_module.ms_deform_attn_backward(
            value, value_spatial_shapes, value_level_start_index, sampling_locations,
            attention_weights, _lib.aligned(grad_output.float().contiguous()), grad_value, grad_sampling_loc,
            grad_attn_weight, im2col_step=ctx.im2col_step)
        dv, dl, da = ctx.in_dtypes
        return grad_value.to(dv), None, None, grad_sampling_loc.to(dl), grad_attn_weight.to(da), None


class MultiScaleDeformableAttnFunction_fp16(MultiScaleDeformableAttnFunction_fp32):
    """multi_scale_deformable_attn_function.py:15-88.  The reference never selects it
    (spatial_cross_attention.py:385-388 routes fp16 to _fp32 too); kept for name parity, it
    computes in fp32 and returns half."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index,
                sampling_locations, attention_weights, im2col_step):
        out = MultiScaleDeformableAttnFunction_fp32.forward(
            ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations,
            attention_weights, im2col_step)
        return out.half()


class MSDeformAttn3DFusedFunction(Function):
    """MSDeformableAttention3D's sampling with its elementwise prologue inside the kernel
    (spatial_cross_attention.py:339-371): softmax over the L*P logits of a (query, head) and
    loc = offsets / (W_l, H_l) + reference_points_cam[..., p % D, :].  Never materialises
    `sampling_locations` / `attention_weights` (0.74 GB at 6 x 40000 queries) nor their gradients.

    apply(value [B,K,H,C], spatial_shapes, level_start_index, reference_points [B,Q,D,2],
          offsets [B,Q,H,L,P,2] (raw Linear output), logits [B,Q,H,L*P]) -> [B,Q,H*C]
    Gradients: value, offsets, logits (reference points come from the camera geometry)."""

    @staticmethod
    def supported(num_levels, num_points, head_dim, num_anchors):
        return num_levels * num_points == 32 and head_dim in (16, 32, 64) and num_points % num_anchors == 0

    @staticmethod
    def forward(ctx, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        value = _lib.aligned(value.float().contiguous())
        ref = _lib.aligned(reference_points.float().contiguous())
        offsets = _lib.aligned(offsets.float().contiguous())
        logits = _lib.aligned(logits.float().contiguous())
        spatial_shapes = spatial_shapes.contiguous()
        level_start_index = level_start_index.contiguous()
        _lib.require_cuda(value=value, spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                          reference_points=ref, offsets=offsets, logits=logits)
        if value.dim() != 4:
            raise RuntimeError(f"value must be [bs, num_keys, num_heads, dim], got {tuple(value.shape)}")
        if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
            raise RuntimeError("spatial_shapes / level_start_index must be int64 tensors")
        B, K, H, C = value.shape
        if ref.dim() != 4 or ref.shape[0] != B or ref.shape[-1] != 2:
            raise RuntimeError(f"reference_points must be [bs, num_queries, num_Z_anchors, 2], got {tuple(ref.shape)}")
        Q, D = ref.shape[1], ref.shape[2]
        if spatial_shapes.dim() != 2 or spatial_shapes.shape[1] != 2:
            raise RuntimeError("spatial_shapes must be [num_levels, 2]")
        L = spatial_shapes.shape[0]
        if level_start_index.numel() != L:
            raise RuntimeError("level_start_index must be [num_levels]")
        if B * Q * H * L == 0 or offsets.numel() % (B * Q * H * L * 2):
            raise RuntimeError("offsets must be [bs, num_queries, num_heads, num_levels, num_points, 2]")
        P = offsets.numel() // (B * Q * H * L * 2)
        if logits.numel() != B * Q * H * L * P:
            raise RuntimeError("reference_points must be [B,Q,D,2], offsets [B,Q,H,L,P,2], logits [B,Q,H,L*P]")
        out = torch.empty((B, Q, H * C), dtype=torch.float32, device=value.device)
        with torch.cuda.device(value.device):
            _lib.check(_lib.lib().vidar_msda_sca_forward(
                _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref), _lib.ptr(offsets),
                _lib.ptr(logits), _lib.ptr(out), B, K, H, C, L, Q, P, D, _lib.stream_ptr(value.device)))
        ctx.save_for_backward(value, spatial_shapes, level_start_index, ref, offsets, logits)
        ctx.dims = (B, K, H, C, L, Q, P, D)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, spatial_shapes, level_start_index, ref, offsets, logits = ctx.saved_tensors
        B, K, H, C, L, Q, P, D = ctx.dims
        grad_output = _lib.aligned(grad_output.float().contiguous())
        grad_value = torch.zeros_like(value)
        grad_offsets = torch.empty_like(offsets)
        grad_logits = torch.empty_like(logits)
        with torch.cuda.device(value.device):
            _lib.check(_lib.lib().vidar_msda_sca_backward(
                _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref), _lib.ptr(offsets),
                _lib.ptr(logits), _lib.ptr(grad_output), _lib.ptr(grad_value), _lib.ptr(grad_offsets),
                _lib.ptr(grad_logits), B, K, H, C, L, Q, P, D, _lib.stream_ptr(value.device)))
        return grad_value, None, None, None, grad_offsets, grad_logits


class MSDeformAttnQueueFusedFunction(Function):
    """TemporalSelfAttention's and the future decoder's sampling with their elementwise prologue and TSA's queue
    mean inside the kernel (temporal_self_attention.py:196-261, vidar_decoder.py:466-506): per (query, head, queue
    entry g) softmax over the L*P logits, loc = offsets / (W_l, H_l) + reference_points[b*G + g, q, l], and the mean
    of the G per-entry outputs.  Never materialises `sampling_locations`, `attention_weights`, the [B*G, Q, H*C]
    per-entry output or their gradients.

    apply(value [B*G,K,H,C], spatial_shapes, level_start_index, reference_points [B*G,Q,L,2],
          offsets [B,Q,H,G,L,P,2] (raw Linear output), logits [B,Q,H,G,L*P]) -> [B,Q,H*C]
    G = 2 for TemporalSelfAttention, 1 for the decoder.  Gradients: value, offsets, logits."""

    @staticmethod
    def supported(num_levels, num_points, num_queue, head_dim, num_value=0, num_heads=1):
        """The shapes the kernel takes; num_value / num_heads (when given) also bound the G value batches of an
        item to 2^25 floats, the vector kernels' 32-bit slab offsets."""
        lp = num_levels * num_points
        return (lp in (1, 2, 4, 8, 16, 32) and 0 < num_queue * lp <= 32 and head_dim in (16, 32, 64)
                and num_queue * num_value * num_heads * head_dim < 2 ** 25)

    @staticmethod
    def forward(ctx, value, spatial_shapes, level_start_index, reference_points, offsets, logits):
        value = _lib.aligned(value.float().contiguous())
        ref = _lib.aligned(reference_points.float().contiguous())
        offsets = _lib.aligned(offsets.float().contiguous())
        logits = _lib.aligned(logits.float().contiguous())
        spatial_shapes = spatial_shapes.contiguous()
        level_start_index = level_start_index.contiguous()
        _lib.require_cuda(value=value, spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                          reference_points=ref, offsets=offsets, logits=logits)
        if value.dim() != 4:
            raise RuntimeError(f"value must be [bs * num_queue, num_keys, num_heads, dim], got {tuple(value.shape)}")
        if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
            raise RuntimeError("spatial_shapes / level_start_index must be int64 tensors")
        if spatial_shapes.dim() != 2 or spatial_shapes.shape[1] != 2 or level_start_index.numel() != spatial_shapes.shape[0]:
            raise RuntimeError("spatial_shapes must be [num_levels, 2] and level_start_index [num_levels]")
        BG, K, H, C = value.shape
        L = spatial_shapes.shape[0]
        if offsets.dim() != 7 or offsets.shape[2] != H or offsets.shape[4] != L or offsets.shape[6] != 2:
            raise RuntimeError("offsets must be [bs, num_queries, num_heads, num_queue, num_levels, num_points, 2], "
                               f"got {tuple(offsets.shape)}")
        B, Q, _, G, _, P, _ = offsets.shape
        if B * G != BG:
            raise RuntimeError(f"value batch ({BG}) must be bs * num_queue ({B} x {G})")
        if tuple(ref.shape) != (BG, Q, L, 2):
            raise RuntimeError(f"reference_points must be {(BG, Q, L, 2)}, got {tuple(ref.shape)}")
        if tuple(logits.shape) != (B, Q, H, G, L * P):
            raise RuntimeError(f"logits must be {(B, Q, H, G, L * P)}, got {tuple(logits.shape)}")
        out = torch.empty((B, Q, H * C), dtype=torch.float32, device=value.device)
        ctx.save_for_backward(value, spatial_shapes, level_start_index, ref, offsets, logits)
        ctx.dims = (B, G, K, H, C, L, Q, P)
        if out.numel() == 0:
            return out
        with torch.cuda.device(value.device):
            _lib.check(_lib.lib().vidar_msda_tsa_forward(
                _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref), _lib.ptr(offsets),
                _lib.ptr(logits), _lib.ptr(out), B, G, K, H, C, L, Q, P, _lib.stream_ptr(value.device)))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, spatial_shapes, level_start_index, ref, offsets, logits = ctx.saved_tensors
        B, G, K, H, C, L, Q, P = ctx.dims
        grad_value = torch.zeros_like(value)
        grad_offsets = torch.empty_like(offsets)      # fully overwritten by the kernel
        grad_logits = torch.empty_like(logits)
        if grad_output.numel():
            grad_output = _lib.aligned(grad_output.float().contiguous())
            with torch.cuda.device(value.device):
                _lib.check(_lib.lib().vidar_msda_tsa_backward(
                    _lib.ptr(value), _lib.ptr(spatial_shapes), _lib.ptr(level_start_index), _lib.ptr(ref),
                    _lib.ptr(offsets), _lib.ptr(logits), _lib.ptr(grad_output), _lib.ptr(grad_value),
                    _lib.ptr(grad_offsets), _lib.ptr(grad_logits), B, G, K, H, C, L, Q, P,
                    _lib.stream_ptr(value.device)))
        return grad_value, None, None, None, grad_offsets, grad_logits

