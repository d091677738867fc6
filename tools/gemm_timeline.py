"""Where the time of a GEMM work unit goes: in-kernel clock64 stamps of the wgmma GEMM, on the forward and dgrad
shapes of ``tools/gemm_bench.py`` with the epilogues the engine uses, at both tile widths.  One JSON line per run.

    B200_NVCC_EXTRA=-DB200_GEMM_TIMELINE python -m bert_pytorch_b200.ops.build
    python tools/gemm_timeline.py [--only NAME]

Per unit (mean over units, SM clock cycles):
  ``mma``      first operand slot ready -> wgmma_wait<0> returned (main loop, including operand waits inside it)
  ``op_wait``  cycles the consumer waited on full_bar (operands not yet loaded)
  ``epi``      wgmma_wait<0> returned -> epilogue done
  ``exposed``  part of ``epi`` no MMA of the CTA ran under: the whole epilogue for the cooperative 128 x 256 tile;
               for the ping-pong 128 x 128 tile, the time from the other warpgroup's last MMA issue of the next unit
               to this epilogue's end
  ``hidden``   share of units whose epilogue was fully hidden (ping-pong only)
  ``unit``     CTA span / units of the CTA (throughput view)
  ``prod_blocked``  cycles the producer waited on empty_bar (ring full) per unit"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bert_pytorch_b200.ops import api as K  # noqa: E402
from tools.gemm_bench import SHAPES, engine_call  # noqa: E402


def analyse(rec: torch.Tensor, bn: int) -> dict:
    r = rec.cpu().numpy().astype("float64")
    units, grid = r.shape[0], int(r[0, 13])
    mma, opw, epi, exposed, hidden = [], [], [], [], 0
    spans = []
    for b in range(grid):
        us = list(range(b, units, grid))
        t_first, t_last = None, None
        for j, u in enumerate(us):
            cws = [0, 1] if bn == 256 else [j & 1]
            for cw in cws:
                s = r[u, 6 * cw: 6 * cw + 6]
                mma.append(s[3] - s[1]); opw.append(s[5]); epi.append(s[4] - s[3])
                t_first = s[0] if t_first is None else min(t_first, s[0])
                t_last = s[4] if t_last is None else max(t_last, s[4])
            if bn == 256:
                exposed.append(max(r[u, 4] - r[u, 3], r[u, 10] - r[u, 9]))
            else:
                cw = j & 1
                if j + 1 < len(us):
                    nxt = r[us[j + 1], 6 * (1 - cw) + 2]          # other warpgroup's last MMA issue, next unit
                    e = max(0.0, r[u, 6 * cw + 4] - nxt)
                else:
                    e = r[u, 6 * cw + 4] - r[u, 6 * cw + 3]
                exposed.append(e)
                hidden += e == 0.0
        spans.append((t_last - t_first) / len(us))
    mean = lambda v: round(sum(v) / len(v) / 1e3, 2)          # noqa: E731  (kilocycles)
    out = {"units": units, "grid": grid, "unit_kcyc": mean(spans), "mma_kcyc": mean(mma), "op_wait_kcyc": mean(opw),
           "epi_kcyc": mean(epi), "exposed_epi_kcyc": mean(exposed),
           "prod_blocked_kcyc": round(float(r[:, 12].mean()) / 1e3, 2)}
    if bn == 128:
        out["hidden_share"] = round(hidden / units, 3)
    return out


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None
    probe = torch.zeros(1, 16, dtype=torch.int64, device="cuda")
    if not K.extension().gemm_timeline(probe):
        sys.exit("the extension was built without -DB200_GEMM_TIMELINE")
    K.extension().gemm_timeline(None)
    for name, layout, m, n, k, epi in SHAPES:
        if layout == K.TN or (only is not None and name != only):
            continue
        a = torch.randn(m, k, device="cuda").bfloat16()
        b = (torch.randn(n, k, device="cuda") if layout == K.NT else torch.randn(k, n, device="cuda")).bfloat16()
        for bn in (128, 256):
            fn = engine_call(a, b, layout, m, n, epi, bn)
            for _ in range(3):
                fn()
            units = ((m + 127) // 128) * ((n + bn - 1) // bn)
            buf = torch.zeros(units, 16, dtype=torch.int64, device="cuda")
            K.extension().gemm_timeline(buf)
            fn()
            torch.cuda.synchronize()
            K.extension().gemm_timeline(None)
            rec = {"name": name, "epi": epi, "block_n": bn}
            rec.update(analyse(buf, bn))
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
