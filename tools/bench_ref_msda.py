"""Same-box CUDA baseline for MSDA (VERDICT r01 9b): the reference-lineage thread mapping
(tools/ref_lineage_msda.cu) against vidar_b200's kernels at the cfg2 shapes, correctness-checked against
each other first.  Build here (CPU box, cross-compile), run on the GPU box:
    python tools/bench_ref_msda.py --build            # -> tools/libref_lineage_msda.so (travels with gpurun)
    gpurun -- 'python tools/bench_ref_msda.py > gpurun_out/ref_msda.json'"""
import ctypes as C
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
LIB = os.path.join(HERE, "libref_lineage_msda.so")


def build():
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-shared", "-Xcompiler", "-fPIC",
           "-cudart", "static", os.path.join(HERE, "ref_lineage_msda.cu"), "-o", LIB]
    subprocess.check_call(cmd)
    return LIB


def main():
    import torch
    from tools.gpu_timing import card, window_ms
    from vidar_b200 import msda, synthetic
    L_ = C.CDLL(LIB)
    dev = torch.device("cuda:0")
    p = lambda t: C.c_void_p(t.data_ptr())
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)

    res = {"what": "MSDA forward / backward, ms per 6-camera pass (cfg2): reference-lineage CUDA mapping vs vidar_b200",
           "card": card()}
    for tag, rows in (("dense_40000", None), ("rebatched_10240", 10240)):
        d = synthetic.sca_like_inputs(dev, rows=rows)
        B, K, H, Cd = d["value"].shape
        Q, Lv, P = d["loc"].shape[1], d["loc"].shape[3], d["loc"].shape[4]
        out_r = torch.empty(B, Q, H * Cd, device=dev)
        gv_r, gl_r, ga_r = torch.zeros_like(d["value"]), torch.zeros_like(d["loc"]), torch.zeros_like(d["attn"])
        gv_o, gl_o, ga_o = torch.zeros_like(d["value"]), torch.zeros_like(d["loc"]), torch.zeros_like(d["attn"])

        def ref_f():
            assert L_.lineage_msda_forward(p(d["value"]), p(d["shapes"]), p(d["lsi"]), p(d["loc"]), p(d["attn"]), p(out_r),
                                           B, K, H, Cd, Lv, Q, P, st()) == 0

        def ref_b():
            assert L_.lineage_msda_backward(p(d["value"]), p(d["shapes"]), p(d["lsi"]), p(d["loc"]), p(d["attn"]),
                                            p(d["grad_out"]), p(gv_r), p(gl_r), p(ga_r), B, K, H, Cd, Lv, Q, P, st()) == 0

        def our_f():
            return msda.ext_module.ms_deform_attn_forward(d["value"], d["shapes"], d["lsi"], d["loc"], d["attn"], im2col_step=64)

        def our_b():
            msda.ext_module.ms_deform_attn_backward(d["value"], d["shapes"], d["lsi"], d["loc"], d["attn"], d["grad_out"],
                                                    gv_o, gl_o, ga_o, im2col_step=64)
        # agreement first (both accumulate grad_value: zero, run once)
        ref_f(); ref_b(); out_o = our_f(); our_b()
        torch.cuda.synchronize()
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
        agree = {"out": rel(out_o, out_r), "grad_value": rel(gv_o, gv_r), "grad_attn": rel(ga_o, ga_r)}
        r = {"agreement_max_rel": agree,
             "ref_lineage_fwd_ms": window_ms(ref_f, 5, 2), "ref_lineage_bwd_ms": window_ms(ref_b, 5, 2),
             "vidar_fwd_ms": window_ms(our_f, 5, 2), "vidar_bwd_ms": window_ms(our_b, 5, 2)}
        r["speedup_fwd"] = r["ref_lineage_fwd_ms"] / r["vidar_fwd_ms"]
        r["speedup_bwd"] = r["ref_lineage_bwd_ms"] / r["vidar_bwd_ms"]
        res[tag] = r
        del d, out_r, gv_r, gl_r, ga_r, gv_o, gl_o, ga_o
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    if "--build" in sys.argv:
        print(build())
    else:
        main()
