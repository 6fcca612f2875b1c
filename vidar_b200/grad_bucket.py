"""Every trainable parameter's gradient in one flat fp32 bucket, and back (csrc/grad_bucket.cu).

`pack` gathers the gradients of a parameter list, each times its own scale, into one bucket in one launch (one per
1024 parameters); a parameter without a gradient packs as zeros.  `unpack` writes the bucket back into every `.grad`
in one launch, allocating the gradients that are None.  The data-parallel step (`sharding.allreduce_grid_grads`)
all-reduces the bucket in between: it replaces a `torch.cat` of hundreds of tensors and one copy per parameter.
Gradients must be fp32, CUDA and contiguous; there is no fallback."""
import numpy as np
import torch

from . import _lib


def _table(params, want_grad):
    """(ptr, numel, offset) int64 host arrays of `params` laid end to end in a bucket, and the bucket's device."""
    n = len(params)
    ptr, numel = np.zeros(n, np.int64), np.zeros(n, np.int64)
    device = None
    for i, p in enumerate(params):
        if p.dtype != torch.float32 or not p.is_cuda:
            raise RuntimeError(f"parameter {i}: the gradient bucket takes fp32 CUDA parameters (got {p.dtype} on {p.device})")
        if device is None:
            device = p.device
        elif p.device != device:
            raise RuntimeError(f"parameter {i} is on {p.device}, parameter 0 on {device}")
        g = p.grad
        if g is not None:
            if g.dtype != torch.float32 or not g.is_cuda or g.device != device:
                raise RuntimeError(f"parameter {i}: gradient must be fp32 on {device} (got {g.dtype} on {g.device})")
            if not g.is_contiguous():
                raise RuntimeError(f"parameter {i}: gradient must be contiguous")
            if g.shape != p.shape:
                raise RuntimeError(f"parameter {i}: gradient shape {tuple(g.shape)} != parameter shape {tuple(p.shape)}")
            ptr[i] = g.data_ptr()
        elif want_grad and p.numel():
            raise RuntimeError(f"parameter {i} has no gradient")
        numel[i] = p.numel()
    offset = np.zeros(n, np.int64)
    if n:
        offset[1:] = np.cumsum(numel)[:-1]
    return ptr, numel, offset, device


def pack(params, scales, out=None):
    """Flat fp32 bucket [sum numel] = cat(p.grad.reshape(-1) * scale for every parameter), zeros for a None gradient.
    `out`: a bucket to fill (fp32, contiguous, right size) instead of a new one."""
    if len(scales) != len(params):
        raise RuntimeError(f"{len(params)} parameters but {len(scales)} scales")
    if not params:
        raise RuntimeError("pack: no parameters")
    ptr, numel, offset, device = _table(params, False)
    total = int(numel.sum())
    if out is None:
        out = torch.empty(total, dtype=torch.float32, device=device)
    elif out.dtype != torch.float32 or out.device != device or not out.is_contiguous() or out.numel() != total:
        raise RuntimeError(f"out must be a contiguous fp32 tensor of {total} elements on {device}")
    sc = np.asarray(scales, np.float32)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().vidar_grad_bucket_pack(ptr.ctypes.data, numel.ctypes.data, offset.ctypes.data,
                                                     sc.ctypes.data, len(params), _lib.ptr(out), total,
                                                     _lib.stream_ptr(device)))
    return out


def unpack(bucket, params):
    """Write `bucket` (pack's layout) back into every parameter's gradient; a None gradient is allocated first."""
    if not params:
        raise RuntimeError("unpack: no parameters")
    for p in params:
        if p.grad is None and p.dtype == torch.float32 and p.is_cuda:
            p.grad = torch.empty_like(p, memory_format=torch.contiguous_format)
    ptr, numel, offset, device = _table(params, True)
    total = int(numel.sum())
    if bucket.dtype != torch.float32 or bucket.device != device or not bucket.is_contiguous() or bucket.numel() != total:
        raise RuntimeError(f"bucket must be a contiguous fp32 tensor of {total} elements on {device}")
    with torch.cuda.device(device):
        _lib.check(_lib.lib().vidar_grad_bucket_unpack(_lib.ptr(bucket), total, ptr.ctypes.data, numel.ctypes.data,
                                                       offset.ctypes.data, len(params), _lib.stream_ptr(device)))
    return params
