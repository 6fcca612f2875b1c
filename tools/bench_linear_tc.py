"""value_proj's GEMM (6 x 30825 rows, 256 -> 256, SURVEY.md 8f-4): the wgmma 3xTF32 kernel against cuBLAS fp32
(what the reference runs) and cuBLAS TF32 (faster, but 5e-4 off) on the same GPU.  JSON on stdout."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gpu_timing import card, window_ms  # noqa: E402
from vidar_b200 import linear  # noqa: E402

dev = torch.device("cuda:0")
M, N, K = 6 * 30825, 256, 256
g = torch.Generator(device=dev).manual_seed(0)
x = torch.randn(M, K, device=dev, generator=g)
w = torch.randn(N, K, device=dev, generator=g) / 16
b = torch.randn(N, device=dev, generator=g)


ref = (x[:4096].double() @ w.double().t() + b.double())
out = {"card": card(), "shape": [M, N, K], "flop": 2.0 * M * N * K}
torch.backends.cuda.matmul.allow_tf32 = False
out["cublas_fp32_ms"] = window_ms(lambda: torch.nn.functional.linear(x, w, b), 20, 5)
out["cublas_fp32_err"] = float((torch.nn.functional.linear(x[:4096], w, b).double() - ref).abs().max() / ref.abs().max())
torch.backends.cuda.matmul.allow_tf32 = True
out["cublas_tf32_ms"] = window_ms(lambda: torch.nn.functional.linear(x, w, b), 20, 5)
out["cublas_tf32_err"] = float((torch.nn.functional.linear(x[:4096], w, b).double() - ref).abs().max() / ref.abs().max())
torch.backends.cuda.matmul.allow_tf32 = False
out["wgmma_3xtf32_ms"] = window_ms(lambda: linear.linear_tf32x3(x, w, b), 20, 5)
out["wgmma_3xtf32_err"] = float((linear.linear_tf32x3(x[:4096], w, b).double() - ref).abs().max() / ref.abs().max())
out["wgmma_tflops_effective"] = out["flop"] / (out["wgmma_3xtf32_ms"] * 1e-3) / 1e12
out["speedup_vs_cublas_fp32"] = out["cublas_fp32_ms"] / out["wgmma_3xtf32_ms"]
print(json.dumps(out))
