"""Time DCNv3 (vidar_b200.dcnv3, csrc/dcnv3.cu) at InternImage-T and -B stage shapes over a 6 x 3x928x1600 input.

The stem has stride 4, so the four stages are 232x400, 116x200, 58x100 and 29x50; every stage has group_channels 16
(T: channels 64/128/256/512, groups 4/8/16/32; B: 112/224/448/896, groups 7/14/28/56), kernel 3, stride 1, pad 1.
For each stage and dtype (fp32 / fp16 / bf16) it times the forward and forward + backward of the op (CUDA events,
median of --iters after --warmup), the reference's own compiled extension (oracle/_ref/ref_dcnv3.so, fp32 and fp16,
where it was built) and the eager grid-sample formulation (one-level MSDA on the padded input with F.grid_sample and
autograd, oracle/dcnv3_ref.py + oracle/msda_ref.py), and prints the card's name and power limit from the same run.

Byte model, computed from shapes (not measured): per output pixel the forward must read C input values, K*G*3 =
27*C/16 offset and mask values and write C outputs; the backward reads input, grad_output, offset and mask and writes
grad_input, grad_offset and grad_mask, 3*C + 54*C/16 values.  `GB/s` is that minimum over the measured time.

    python tools/bench_dcnv3.py [--model T|B|both] [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dcnv3_ref, msda_ref  # noqa: E402
from tools.gpu_timing import card, event_ms  # noqa: E402
from vidar_b200.dcnv3 import ext  # noqa: E402

STAGES = [(232, 400), (116, 200), (58, 100), (29, 50)]
MODELS = {"T": [64, 128, 256, 512], "B": [112, 224, 448, 896]}
CG, BATCH, K = 16, 6, 9
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def min_bytes(C, H, W, esize):
    pix = BATCH * H * W
    fwd = pix * (2 * C + 27 * C // 16) * esize
    bwd = pix * (3 * C + 54 * C // 16) * esize
    return fwd, bwd


def eager(x, off, mask, args, gy=None):
    leaves = [t.detach().requires_grad_(gy is not None) for t in (x, off, mask)]
    value, shapes, loc, attn = dcnv3_ref.as_msda(*leaves, *args)
    y = msda_ref.msda_grid_sample(value, shapes, loc, attn)
    if gy is not None:
        y.backward(gy.reshape(y.shape))
    return y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="both", choices=["T", "B", "both"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dcnv3 needs a CUDA device"
    dev = torch.device("cuda:0")
    try:
        from oracle import build_ref_dcnv3
        ref = build_ref_dcnv3.load()
    except (FileNotFoundError, ImportError, OSError):
        ref = None
    print(f"# {json.dumps(card())}; batch {BATCH}, group_channels {CG}, kernel 3; median of {a.iters} (ms)")
    print("| model | stage | dtype | op fwd | op fwd+bwd | fwd GB/s | fwd+bwd GB/s | ref fwd | ref fwd+bwd | "
          "eager fwd | eager fwd+bwd |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for model in (["T", "B"] if a.model == "both" else [a.model]):
        for si, ((H, W), C) in enumerate(zip(STAGES, MODELS[model])):
            G = C // CG
            args = (3, 3, 1, 1, 1, 1, 1, 1, G, CG, 1.0)
            g = torch.Generator(device=dev).manual_seed(si)
            for dname, dt in DTYPES.items():
                x = torch.randn(BATCH, H, W, C, device=dev, generator=g).to(dt)
                off = (torch.randn(BATCH, H, W, G * K * 2, device=dev, generator=g) * 2).to(dt)
                mask = torch.softmax(torch.randn(BATCH, H, W, G, K, device=dev, generator=g), -1).reshape(
                    BATCH, H, W, -1).to(dt)
                gy = torch.randn(BATCH, H, W, C, device=dev, generator=g).to(dt)
                f = event_ms(lambda: ext.dcnv3_forward(x, off, mask, *args, 256), a.iters, a.warmup)
                fb = event_ms(lambda: (ext.dcnv3_forward(x, off, mask, *args, 256),
                                       ext.dcnv3_backward(x, off, mask, *args, gy, 256)), a.iters, a.warmup)
                bf, bb = min_bytes(C, H, W, x.element_size())
                row = dict(model=model, stage=si + 1, dtype=dname, fwd_ms=f, fwd_bwd_ms=fb,
                           fwd_gbs=bf / f / 1e6, fwd_bwd_gbs=(bf + bb) / fb / 1e6, min_fwd_mb=bf / 1e6,
                           min_bwd_mb=bb / 1e6)
                if ref is not None and dt != torch.bfloat16:
                    row["ref_fwd_ms"] = event_ms(lambda: ref.dcnv3_forward(x, off, mask, *args, 256), a.iters,
                                                 a.warmup)
                    row["ref_fwd_bwd_ms"] = event_ms(lambda: (ref.dcnv3_forward(x, off, mask, *args, 256),
                                                              ref.dcnv3_backward(x, off, mask, *args, gy, 256)),
                                                     a.iters, a.warmup)
                row["eager_fwd_ms"] = event_ms(lambda: eager(x, off, mask, args), a.iters, a.warmup)
                row["eager_fwd_bwd_ms"] = event_ms(lambda: eager(x, off, mask, args, gy), a.iters, a.warmup)
                fmt = lambda k: f"{row[k]:.3f}" if k in row else "-"  # noqa: E731
                print(f"| {model} | {si + 1} ({H}x{W}, C {C}) | {dname} | {fmt('fwd_ms')} | {fmt('fwd_bwd_ms')} | "
                      f"{row['fwd_gbs']:.0f} | {row['fwd_bwd_gbs']:.0f} | {fmt('ref_fwd_ms')} | "
                      f"{fmt('ref_fwd_bwd_ms')} | {fmt('eager_fwd_ms')} | {fmt('eager_fwd_bwd_ms')} |", flush=True)
                print("#", json.dumps(row), flush=True)
                del x, off, mask, gy
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
