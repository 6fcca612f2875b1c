"""Time the modulated deformable convolution (vidar_b200/dcn.py) at the reference backbone's DCN layer shapes.

    python tools/bench_dcn.py [--steps 20] [--warmup 3] [--no-backbone] [--dtype {float32,float16,bfloat16}]

Shapes (the 6 x 3 x 928 x 1600 input of the pre-training step): stage 3 = 6 x 256 x 58 x 100 -> 256, stage 4 =
6 x 512 x 29 x 50 -> 512, 3x3, stride 1, padding 1, no bias, offsets ~ N(0, 2^2) px, channels_last input as the
backbone produces it.  Per shape, forward and forward+backward of
  * this op (im2col + 3xTF32 wgmma GEMM; backward cuBLAS grad_W, 3xTF32 grad_cols, col2im),
  * torchvision.ops.deform_conv2d in fp32 on the same card (what a user would otherwise run),
  * a cuDNN 3x3 convolution of the same shape in fp32 (TF32 off): the floor of a plain convolution;
plus the im2col and col2im kernels alone with the bytes they must move (input, offsets and mask read; columns written /
read; grad_input reduced) and their share of the H100 SXM's 3.35 TB/s, and the forward GEMM alone with its
fp32-equivalent rate (2 M N K / time).  With the backbone: ImageBackbone(dcn=True) against dcn=False, forward + backward
of 6 x 3 x 928 x 1600.  CUDA events around each call, every candidate warmed up, median of --steps, the candidates of
one shape alternating.  The card's name, power limit and clocks are read in the same run.  Prints one JSON line.

--dtype float16 / bfloat16 times the 16-bit path instead (every tensor of the op in that dtype): per shape, forward
and forward+backward of this op in that dtype against this op in fp32 and the cuDNN convolution in that dtype; the
16-bit im2col and col2im kernels with the bytes they must move for that storage type (grad_input, grad_offset and
grad_mask are fp32); and the backbone's forward + backward under torch.autocast in that dtype, with DCN and with
plain convolutions."""
import argparse
import contextlib
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.gpu_timing import card, event_ms  # noqa: E402
from vidar_b200 import _lib, dcn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SHAPES = {"stage3": (6, 256, 58, 100), "stage4": (6, 512, 29, 50)}


def layer(shape, steps, warmup):
    import torchvision
    N, C, H, W = shape
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(N, C, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    off = torch.randn(N, 18, H, W, device=dev, generator=g) * 2.0
    mask = torch.rand(N, 9, H, W, device=dev, generator=g)
    w = torch.randn(C, C, 3, 3, device=dev, generator=g) / (9 * C) ** 0.5
    gy = torch.randn(N, C, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    leaves = [t.clone().requires_grad_(True) for t in (x, off, mask, w)]

    def ours_f():
        with torch.no_grad():
            dcn.modulated_deform_conv2d(x, off, mask, w, None, 1, 1, 1, 1, 1)

    def tv_f():
        with torch.no_grad():
            torchvision.ops.deform_conv2d(x, off, w, None, padding=1, mask=mask)

    def conv_f():
        with torch.no_grad():
            F.conv2d(x, w, None, padding=1)

    def ours_fb():
        xa, oa, ma, wa = leaves
        dcn.modulated_deform_conv2d(xa, oa, ma, wa, None, 1, 1, 1, 1, 1).backward(gy)

    def tv_fb():
        xa, oa, ma, wa = leaves
        torchvision.ops.deform_conv2d(xa, oa, wa, None, padding=1, mask=ma).backward(gy)

    def conv_fb():
        xa, wa = leaves[0], leaves[3]
        F.conv2d(xa, wa, None, padding=1).backward(gy)

    # the two kernels and the forward GEMM alone, on the buffers the op uses
    K = 9 * C
    M = N * H * W
    xl = x.permute(0, 2, 3, 1).contiguous()
    cols = torch.empty(M, K, device=dev)
    w2 = w.permute(0, 2, 3, 1).reshape(C, K).contiguous()
    y = torch.empty(M, C, device=dev)
    scratch = torch.empty(2 * C * K, device=dev)
    gx, go, gm = torch.zeros_like(xl), torch.empty_like(off), torch.empty_like(mask)
    geom = (N, C, H, W, H, W, 3, 3, 1, 1, 1, 1, 1, 1)
    L, st = _lib.lib(), _lib.stream_ptr(dev)

    def im2col():
        _lib.check(L.vidar_dcn_im2col(_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cols), *geom, 0, N, st))

    def col2im():
        _lib.check(L.vidar_dcn_col2im(_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cols), _lib.ptr(gx),
                                      _lib.ptr(go), _lib.ptr(gm), *geom, 0, N, st))

    def gemm():
        dcn._gemm(cols, w2, None, y, scratch)

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    fwd = event_ms(dict(ours=ours_f, torchvision=tv_f, cudnn_conv=conv_f), steps, warmup)
    fwdbwd = event_ms(dict(ours=ours_fb, torchvision=tv_fb, cudnn_conv=conv_fb), steps, warmup)
    kern = event_ms(dict(im2col=im2col, col2im=col2im, gemm=gemm), steps, warmup)
    side = N * 27 * H * W * 4                                       # offsets + mask
    im2col_bytes = N * H * W * C * 4 + side + M * K * 4             # input once, columns written
    col2im_bytes = M * K * 4 + N * H * W * C * 4 * 2 + side * 2     # grad_cols + input read, grad_input, grad_off/mask
    flop = 2.0 * M * C * K
    return dict(
        shape=dict(N=N, C=C, H=H, W=W, Cout=C, M=M, K=K), fwd_ms=fwd, fwd_bwd_ms=fwdbwd, kernels_ms=kern,
        im2col=dict(bytes=im2col_bytes, hbm_share=round(im2col_bytes / (kern["im2col"] * 1e-3) / HBM_BYTES_PER_S, 3)),
        col2im=dict(bytes=col2im_bytes, hbm_share=round(col2im_bytes / (kern["col2im"] * 1e-3) / HBM_BYTES_PER_S, 3)),
        gemm=dict(flop=flop, fp32_equiv_tflops=round(flop / (kern["gemm"] * 1e-3) / 1e12, 1)),
        speedup_vs_torchvision=dict(fwd=round(fwd["torchvision"] / fwd["ours"], 2),
                                    fwd_bwd=round(fwdbwd["torchvision"] / fwdbwd["ours"], 2)))


def layer_half(shape, dt, steps, warmup):
    N, C, H, W = shape
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(N, C, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    off = torch.randn(N, 18, H, W, device=dev, generator=g) * 2.0
    mask = torch.rand(N, 9, H, W, device=dev, generator=g)
    w = torch.randn(C, C, 3, 3, device=dev, generator=g) / (9 * C) ** 0.5
    gy = torch.randn(N, C, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    half = [t.to(dt) for t in (x, off, mask, w, gy)]
    leaves32 = [t.clone().requires_grad_(True) for t in (x, off, mask, w)]
    leaves16 = [t.clone().requires_grad_(True) for t in half[:4]]

    def op_f(ts):
        def fn():
            with torch.no_grad():
                dcn.modulated_deform_conv2d(*ts, None, 1, 1, 1, 1, 1)
        return fn

    def op_fb(ts, gout):
        def fn():
            dcn.modulated_deform_conv2d(*ts, None, 1, 1, 1, 1, 1).backward(gout)
        return fn

    def conv_f():
        with torch.no_grad():
            F.conv2d(half[0], half[3], None, padding=1)

    def conv_fb():
        F.conv2d(leaves16[0], leaves16[3], None, padding=1).backward(half[4])

    K = 9 * C
    M = N * H * W
    s = torch.empty((), dtype=dt).element_size()
    xl = half[0].permute(0, 2, 3, 1).contiguous()
    cols = torch.empty(M, K, device=dev, dtype=dt)
    gx, go, gm = torch.zeros(xl.shape, device=dev), torch.empty(off.shape, device=dev), torch.empty(mask.shape, device=dev)
    geom = (N, C, H, W, H, W, 3, 3, 1, 1, 1, 1, 1, 1)
    L, st, code = _lib.lib(), _lib.stream_ptr(dev), dcn.HALF_DTYPE_CODES[dt]
    o16, m16 = half[1], half[2]

    def im2col():
        _lib.check(L.vidar_dcn_im2col_half(_lib.ptr(xl), _lib.ptr(o16), _lib.ptr(m16), _lib.ptr(cols), code, *geom, 0, N,
                                           st))

    def col2im():
        _lib.check(L.vidar_dcn_col2im_half(_lib.ptr(xl), _lib.ptr(o16), _lib.ptr(m16), _lib.ptr(cols), _lib.ptr(gx),
                                           _lib.ptr(go), _lib.ptr(gm), code, *geom, 0, N, st))

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    name = str(dt).replace("torch.", "")
    fwd = event_ms({f"ours_{name}": op_f(half[:4]), "ours_float32": op_f((x, off, mask, w)),
                    f"cudnn_conv_{name}": conv_f}, steps, warmup)
    fwdbwd = event_ms({f"ours_{name}": op_fb(leaves16, half[4]), "ours_float32": op_fb(leaves32, gy),
                       f"cudnn_conv_{name}": conv_fb}, steps, warmup)
    kern = event_ms(dict(im2col=im2col, col2im=col2im), steps, warmup)
    side = N * 27 * H * W
    im2col_bytes = N * H * W * C * s + side * s + M * K * s                          # input once, columns written
    col2im_bytes = M * K * s + N * H * W * C * (s + 4) + side * (s + 4)             # + fp32 grad_input / offset / mask
    return dict(
        shape=dict(N=N, C=C, H=H, W=W, Cout=C, M=M, K=K), fwd_ms=fwd, fwd_bwd_ms=fwdbwd, kernels_ms=kern,
        im2col=dict(bytes=im2col_bytes, hbm_share=round(im2col_bytes / (kern["im2col"] * 1e-3) / HBM_BYTES_PER_S, 3)),
        col2im=dict(bytes=col2im_bytes, hbm_share=round(col2im_bytes / (kern["col2im"] * 1e-3) / HBM_BYTES_PER_S, 3)),
        speedup_vs_float32=dict(fwd=round(fwd["ours_float32"] / fwd[f"ours_{name}"], 2),
                                fwd_bwd=round(fwdbwd["ours_float32"] / fwdbwd[f"ours_{name}"], 2)))


def backbone(steps, warmup, amp=None):
    """Forward + backward of ImageBackbone with and without DCN, under torch.autocast(amp) when amp is a dtype."""
    from vidar_b200.pretrain import ImageBackbone
    dev = torch.device("cuda")
    torch.manual_seed(0)
    models = {"dcn": ImageBackbone(dcn=True).to(dev).train(), "plain": ImageBackbone(dcn=False).to(dev).train()}
    img = torch.randn(6, 3, 928, 1600, device=dev)

    def run(m):
        def fn():
            m.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=amp) if amp is not None else contextlib.nullcontext():
                feats = m(img)
            sum(f.float().mean() for f in feats).backward()
        return fn

    return event_ms({k: run(m) for k, m in models.items()}, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-backbone", action="store_true")
    ap.add_argument("--dtype", choices=("float32", "float16", "bfloat16"), default="float32")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn needs a CUDA device")
    res = dict(tool="bench_dcn", card=card(), steps=a.steps, tf32="off (cuDNN and cuBLAS fp32)")
    if a.dtype == "float32":
        for k, s in SHAPES.items():
            res[k] = layer(s, a.steps, a.warmup)
        if not a.no_backbone:
            res["backbone_fwd_bwd_ms"] = backbone(a.steps, a.warmup)
    else:
        dt = getattr(torch, a.dtype)
        res["dtype"] = a.dtype
        for k, s in SHAPES.items():
            res[k] = layer_half(s, dt, a.steps, a.warmup)
        if not a.no_backbone:
            res[f"backbone_autocast_{a.dtype}_fwd_bwd_ms"] = backbone(a.steps, a.warmup, dt)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
