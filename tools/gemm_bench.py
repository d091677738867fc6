"""Device-timed throughput of the wgmma GEMM on the BERT-large shapes vs torch.matmul (cuBLAS) ->
gpurun_out/gemm_bench.json.  CUDA events, warm-up, L2 flush between iterations."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bert_pytorch_b200.ops import api as K  # noqa: E402


def timeit(fn, iters=20, warm=5):
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.fill_(0.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None
    M = 12288
    out = []
    shapes = [("qkv_fwd", K.NT, M, 3072, 1024), ("attn_out_fwd", K.NT, M, 1024, 1024), ("ffn1_fwd", K.NT, M, 4096, 1024),
              ("ffn2_fwd", K.NT, M, 1024, 4096), ("ffn1_dgrad", K.NN, M, 1024, 4096), ("ffn2_dgrad", K.NN, M, 4096, 1024),
              ("ffn1_wgrad", K.TN, 4096, 1024, M), ("ffn2_wgrad", K.TN, 1024, 4096, M), ("qkv_wgrad", K.TN, 3072, 1024, M),
              ("decoder_fwd", K.NT, 1920, 30528, 1024), ("big", K.NT, 8192, 8192, 8192)]
    for name, layout, m, n, k in shapes:
        if only is not None and name != only:
            continue
        if layout == K.NT:
            a, b = torch.randn(m, k, device="cuda").bfloat16(), torch.randn(n, k, device="cuda").bfloat16()
            ref = lambda: a @ b.t()
        elif layout == K.NN:
            a, b = torch.randn(m, k, device="cuda").bfloat16(), torch.randn(k, n, device="cuda").bfloat16()
            ref = lambda: a @ b
        else:
            a, b = torch.randn(k, m, device="cuda").bfloat16(), torch.randn(k, n, device="cuda").bfloat16()
            ref = lambda: a.t() @ b
        flops = 2.0 * m * n * k
        rec = {"name": name, "M": m, "N": n, "K": k}
        t_ref = timeit(ref)
        rec["cublas_ms"], rec["cublas_tflops"] = round(t_ref, 4), round(flops / t_ref / 1e9, 1)
        for bn in (128, 256):
            if layout == K.TN:
                o = torch.zeros(m, n, device="cuda")
                for sp in (1, 2, 4, 8, -1):                 # -1: as many K ranges as fill the SMs
                    t = timeit(lambda: K.gemm(a, b, layout=layout, epi=K.EPI_ACCUM_F32, out=o, block_n=bn, k_splits=sp))
                    rec[f"ours_bn{bn}_s{'auto' if sp < 0 else sp}_tflops"] = round(flops / t / 1e9, 1)
            else:
                o = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, block_n=bn))
                rec[f"ours_bn{bn}_ms"], rec[f"ours_bn{bn}_tflops"] = round(t, 4), round(flops / t / 1e9, 1)
        if "--fp8" in sys.argv:          # same shape with e4m3 (e5m2 for the gradient operand) bytes
            a_e5 = layout != K.NT
            meta = K.Fp8Meta(["a", "b"], [a_e5, False], "cuda")
            qa, qb = meta.quantize(a, "a", calibrate=True), meta.quantize(b, "b", calibrate=True)
            kw = dict(layout=layout, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"), a_e5m2=a_e5)
            if layout == K.TN:
                o = torch.zeros(m, n, device="cuda")
                for sp in (1, 2, 4, -1):
                    t = timeit(lambda: K.gemm(qa, qb, epi=K.EPI_ACCUM_F32, out=o, k_splits=sp, **kw))
                    rec[f"fp8_s{'treamk' if sp < 0 else sp}_tflops"] = round(flops / t / 1e9, 1)
            else:
                o = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
                t = timeit(lambda: K.gemm(qa, qb, out=o, **kw))
                rec["fp8_ms"], rec["fp8_tflops"] = round(t, 4), round(flops / t / 1e9, 1)
            t = timeit(lambda: meta.quantize(a, "a", out=qa))
            rec["quantize_a_gbs"] = round(a.numel() * 3 / t / 1e6, 1)
        if "--epi" in sys.argv and name in ("ffn1_fwd", "ffn2_dgrad", "attn_out_fwd", "ffn2_fwd"):
            # the fused epilogues the engine runs on this shape, against the plain bf16 store
            o = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
            if name == "ffn1_fwd":
                bias, aux = torch.randn(n, device="cuda").bfloat16(), torch.empty_like(o)
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, epi=K.EPI_BIAS_GELU_DG, bias=bias, aux_out=aux))
                rec["epi_bias_gelu_dg_tflops"] = round(flops / t / 1e9, 1)
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, epi=K.EPI_BIAS, bias=bias))
                rec["epi_bias_tflops"] = round(flops / t / 1e9, 1)
            elif name == "ffn2_dgrad":
                res, cs = torch.randn(m, n, device="cuda").bfloat16(), torch.zeros(n, device="cuda")
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, epi=K.EPI_MUL, res=res, colsum=cs))
                rec["epi_mul_colsum_tflops"] = round(flops / t / 1e9, 1)
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, epi=K.EPI_MUL, res=res))
                rec["epi_mul_tflops"] = round(flops / t / 1e9, 1)
            else:
                bias, res = torch.randn(n, device="cuda").bfloat16(), torch.randn(m, n, device="cuda").bfloat16()
                t = timeit(lambda: K.gemm(a, b, layout=layout, out=o, epi=K.EPI_BIAS_DROP_RES, bias=bias, res=res, p_drop=0.1,
                                          seed=1, stream=3))
                rec["epi_bias_drop_res_tflops"] = round(flops / t / 1e9, 1)
        out.append(rec)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
