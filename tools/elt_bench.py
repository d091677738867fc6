"""Device-timed bandwidth kernels (LayerNorm fwd/bwd, GELU fwd/bwd, column sums, fp8 quantise) at the BERT-large
phase-1 shapes, with the algorithmic bytes and the fraction of the measured copy bandwidth (MEASURED_PEAKS.json).
The LayerNorm rows cover each variant the engine runs: bf16 encoder LNs, the fp8 side outputs of the fp8 config, the
embedding LN backward (input-side dropout, no dropped copy) and H = 768 (BERT-base)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        peak = 6577.0
    M, H, I = 12288, 1024, 4096
    x = torch.randn(M, H, device="cuda").bfloat16()
    dy = torch.randn(M, H, device="cuda").bfloat16()
    g, b = torch.ones(H, device="cuda"), torch.zeros(H, device="cuda")
    dg, db, dbias = torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda"), torch.zeros(H, device="cuda")
    y, mean, rstd = K.layer_norm_fwd(x, g, b)
    ln8 = K.Fp8Meta(["y", "dxd"], [False, True], "cuda")
    H2 = 768
    x2, dy2 = x[:, :H2].contiguous(), dy[:, :H2].contiguous()
    g2, b2, dg2, db2, dbias2 = g[:H2], b[:H2], dg[:H2], db[:H2], dbias[:H2]
    y2, mean2, rstd2 = K.layer_norm_fwd(x2, g2, b2)
    xi = torch.randn(M, I, device="cuda").bfloat16()
    di = torch.randn(M, I, device="cuda").bfloat16()
    dbi = torch.zeros(I, device="cuda")
    rows = [
        ("layer_norm_fwd", lambda: K.layer_norm_fwd(x, g, b), 2 * M * H * 2),
        ("layer_norm_bwd(+dropped copy, dgamma/dbeta/dbias)", lambda: K.layer_norm_bwd(
            dy, x, mean, rstd, g, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True, p_drop=0.1, seed=3, drop_stream=5),
         4 * M * H * 2),
        ("layer_norm_fwd(+fp8 copy)", lambda: K.layer_norm_fwd(x, g, b, fp8=(ln8, "y")), 2 * M * H * 2 + M * H),
        ("layer_norm_bwd(+dropped copy +fp8 copy, dgamma/dbeta/dbias)", lambda: K.layer_norm_bwd(
            dy, x, mean, rstd, g, dgamma=dg, dbeta=db, dbias=dbias, want_dropped=True, p_drop=0.1, seed=3, drop_stream=5,
            fp8=(ln8, "dxd")), 4 * M * H * 2 + M * H),
        ("layer_norm_bwd(input dropout: embedding LN, dgamma/dbeta)", lambda: K.layer_norm_bwd(
            dy, x, mean, rstd, g, dgamma=dg, dbeta=db, p_drop=0.1, seed=3, in_stream=1023 * 8), 3 * M * H * 2),
        ("layer_norm_fwd H=768", lambda: K.layer_norm_fwd(x2, g2, b2), 2 * M * H2 * 2),
        ("layer_norm_bwd(+dropped copy, dgamma/dbeta/dbias) H=768", lambda: K.layer_norm_bwd(
            dy2, x2, mean2, rstd2, g2, dgamma=dg2, dbeta=db2, dbias=dbias2, want_dropped=True, p_drop=0.1, seed=3,
            drop_stream=5), 4 * M * H2 * 2),
        ("gelu_fwd [M,4096]", lambda: K.gelu_fwd(xi), 2 * M * I * 2),
        ("dgelu_bwd(+bias grad) [M,4096]", lambda: K.dgelu_bwd(di, xi, dbi), 3 * M * I * 2),
        ("colsum [M,3072]", lambda: K.colsum_accumulate(torch.narrow(xi, 1, 0, 3072).contiguous(), dbi[:3072]), M * 3072 * 2),
    ]
    meta = K.Fp8Meta(["a"], [False], "cuda")
    q = meta.quantize(xi, "a", calibrate=True)
    rows.append(("fp8_quantize [M,4096]", lambda: meta.quantize(xi, "a", out=q), 3 * M * I))
    for name, fn, nbytes in rows:
        if name.startswith("colsum"):
            src = torch.narrow(xi, 1, 0, 3072).contiguous()
            fn = (lambda s=src: K.colsum_accumulate(s, dbi[:3072]))
        t = timeit(fn)
        gbs = nbytes / t / 1e6
        print(json.dumps({"kernel": name, "ms": round(t, 4), "algorithmic_MB": round(nbytes / 1e6, 1), "GBps": round(gbs, 1),
                          "frac_of_measured_copy_bw": round(gbs / peak, 3)}), flush=True)


if __name__ == "__main__":
    main()
