"""Device-timed throughput of the wgmma GEMM on the BERT-large shapes vs torch.matmul (cuBLAS), printed as one JSON
line per shape.  CUDA events, warm-up, L2 flush between iterations.

    python tools/gemm_bench.py [--epi] [--fp8] [--only NAME]

``--epi`` also times every shape with the epilogue the fused engine runs on it (wgrad: ``wgrad_accumulate``, the
split-K factor the engine picks)."""
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


M = 12288          # phase 1: micro-batch 96 x seq 128
# (name, layout, M, N, K, engine epilogue): every GEMM of one encoder layer, then the MLM decoder and a square check
SHAPES = [("qkv_fwd", K.NT, M, 3072, 1024, "bias"), ("attn_out_fwd", K.NT, M, 1024, 1024, "bias_drop_res"),
          ("ffn1_fwd", K.NT, M, 4096, 1024, "bias_gelu_dg"), ("ffn2_fwd", K.NT, M, 1024, 4096, "bias_drop_res"),
          ("ffn2_dgrad", K.NN, M, 4096, 1024, "mul_colsum"), ("ffn1_dgrad", K.NN, M, 1024, 4096, "add"),
          ("attn_out_dgrad", K.NN, M, 1024, 1024, "none"), ("qkv_dgrad", K.NN, M, 1024, 3072, "add"),
          ("ffn2_wgrad", K.TN, 1024, 4096, M, "wgrad"), ("ffn1_wgrad", K.TN, 4096, 1024, M, "wgrad"),
          ("attn_out_wgrad", K.TN, 1024, 1024, M, "wgrad"), ("qkv_wgrad", K.TN, 3072, 1024, M, "wgrad"),
          ("decoder_fwd", K.NT, 1920, 30528, 1024, "bias"), ("big", K.NT, 8192, 8192, 8192, "none")]


def engine_call(a, b, layout, m, n, epi, block_n=None):
    """the GEMM call the fused engine makes on this shape, with its fused epilogue (``block_n``: force a tile width)"""
    if epi == "wgrad":
        g = torch.zeros(m, n, device="cuda")
        return lambda: K.wgrad_accumulate(a, b, g)
    o = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
    kw = dict(layout=layout, out=o, block_n=block_n)
    if epi == "bias":
        kw.update(epi=K.EPI_BIAS, bias=torch.randn(n, device="cuda").bfloat16())
    elif epi == "bias_gelu_dg":
        kw.update(epi=K.EPI_BIAS_GELU_DG, bias=torch.randn(n, device="cuda").bfloat16(), aux_out=torch.empty_like(o))
    elif epi == "bias_drop_res":
        kw.update(epi=K.EPI_BIAS_DROP_RES, bias=torch.randn(n, device="cuda").bfloat16(),
                  res=torch.randn(m, n, device="cuda").bfloat16(), p_drop=0.1,
                  mask_in=K.dropout_mask(m, n, 0.1, 1, 3, "cuda"))
    elif epi == "mul_colsum":
        kw.update(epi=K.EPI_MUL, res=torch.randn(m, n, device="cuda").bfloat16(), colsum=torch.zeros(n, device="cuda"))
    elif epi == "add":
        kw.update(epi=K.EPI_ADD, res=torch.randn(m, n, device="cuda").bfloat16())
    return lambda: K.gemm(a, b, **kw)


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None
    for name, layout, m, n, k, epi in SHAPES:
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
        if "--epi" in sys.argv:
            t = timeit(engine_call(a, b, layout, m, n, epi))
            rec[f"engine_{epi}_ms"], rec[f"engine_{epi}_tflops"] = round(t, 4), round(flops / t / 1e9, 1)
            if layout != K.TN:
                for bn in (128, 256):
                    t = timeit(engine_call(a, b, layout, m, n, epi, bn))
                    rec[f"engine_{epi}_bn{bn}_tflops"] = round(flops / t / 1e9, 1)
        if "--fp8" in sys.argv:          # same shape with e4m3 (e5m2 for the gradient operand) bytes
            a_e5 = layout != K.NT
            meta = K.Fp8Meta(["a", "b"], [a_e5, False], "cuda")
            qa, qb = meta.quantize(a, "a", calibrate=True), meta.quantize(b, "b", calibrate=True)
            kw = dict(layout=layout, scale_a=meta.inv_scale("a"), scale_b=meta.inv_scale("b"), a_e5m2=a_e5)
            if layout == K.TN:
                o = torch.zeros(m, n, device="cuda")
                for sp in (1, 2, 4, -1):
                    t = timeit(lambda: K.gemm(qa, qb, epi=K.EPI_ACCUM_F32, out=o, k_splits=sp, **kw))
                    rec[f"fp8_s{'auto' if sp < 0 else sp}_tflops"] = round(flops / t / 1e9, 1)
            else:
                o = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
                t = timeit(lambda: K.gemm(qa, qb, out=o, **kw))
                rec["fp8_ms"], rec["fp8_tflops"] = round(t, 4), round(flops / t / 1e9, 1)
            t = timeit(lambda: meta.quantize(a, "a", out=qa))
            rec["quantize_a_gbs"] = round(a.numel() * 3 / t / 1e6, 1)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
