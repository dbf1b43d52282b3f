#!/usr/bin/env python3
"""bf16 decode timing on one GPU: the fused bf16 routes of QuantLinearLUT.forward for 1 to 79 rows against what it ran before, on
the LLaMA-7B layers as the model runs them (q/k/v and gate/up stacked) and one 65B w3 layer.

Arms, all on the same inputs:
  bf16        the new bf16 route: quant_cuda.lutgemv_fused (1 row; the one-GEMV kernel) or quant_cuda.lutgemv_rows_bf16
              (2 rows and more; the multi-row GEMV)
  bf16_old    what forward ran for bf16 x before: 1 row the reference's sequence (torch.zeros, x.float(), the hybrid symbol,
              y.to(bf16)), more rows the batched one (torch.zeros, x.float(), the _batched hybrid symbol, out.to(bf16))
  fp16        the fp16 route of the same row count: lutgemv_fused (1 row), lutgemv_rows (2 to 63), lutgemm_fused (64 and more)

Per (shape, M) one JSON line: ms of every arm and the max relative difference of each arm against the bf16 arm.  The arms are
alternated inside each repetition and the median of 5 is kept.  Per M one more line sums the four launches of one 7B decoder layer
per arm: that table sets QuantLinearLUT.BF16_ROWS_MAX.  The first line names the card and its power limit (nvidia-smi, read-only
query).

    python tests/perf/decode_bf16_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from prefill_tc_timing import SHAPES, batched_call, rel, synth, time_ms  # noqa: E402
from squeezellm_b200.quant import QuantLinearLUT  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

ROWS = [1, 2, 4, 8, 16, 32, 48, 63, 64, 72, 79]


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    shapes, rows = (SHAPES[:2], [1, 8]) if quick else (SHAPES, ROWS)
    layer_ms = {}
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        lay = (L["qweight"], L["lut"], bits, None, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        one_row = getattr(qc, f"vecquant{bits}matmul_spmv_hybrid_nuq_perchannel")
        for M in rows:
            xb = torch.randn((M, K), device="cuda").bfloat16()
            x16 = xb.half()
            out = {}

            def new():
                out["bf16"] = qc.lutgemv_fused(xb[0], *lay)[None] if M == 1 else qc.lutgemv_rows_bf16(xb, *lay)

            def old():
                if M == 1:  # QuantLinearLUT's 12-symbol branch for a layer without bias
                    y = torch.zeros((N,), device="cuda", dtype=torch.float32)
                    one_row(L["rows"], L["cols"], L["vals"], xb.float(), L["full_rows"], L["fri"], y, N, L["qweight"], L["lut"])
                    out["bf16_old"] = y.to(torch.bfloat16)[None]
                else:
                    y = torch.zeros((M, N), device="cuda", dtype=torch.float32)
                    batched_call(qc, L, xb.float(), y)
                    out["bf16_old"] = y.to(torch.bfloat16)

            def fp16():
                if M == 1:
                    out["fp16"] = qc.lutgemv_fused(x16[0], *lay)[None]
                elif M <= QuantLinearLUT.ROWS_MAX:
                    out["fp16"] = qc.lutgemv_rows(x16, *lay)
                else:
                    out["fp16"] = qc.lutgemm_fused(x16, *lay)

            arms = {"bf16": new, "bf16_old": old, "fp16": fp16}
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: out[a].float().clone() for a in arms}
            t = {a: [] for a in arms}
            n = {}
            for a, fn in arms.items():  # warm-up, and size the loop to about 20 ms per measurement
                t0 = time_ms(fn, 1)
                n[a] = max(1, min(500, int(20.0 / max(t0, 1e-3))))
            for _ in range(3 if quick else 5):
                for a, fn in arms.items():
                    t[a].append(time_ms(fn, n[a]))
            rec = dict(kind="bf16-decode", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(statistics.median(t[a]), 5)
                if a != "bf16":
                    rec[a + "_max_rel_diff_vs_bf16"] = float(f"{rel(got[a], got['bf16']):.3e}")
            rec["bf16_speedup_vs_old"] = round(rec["bf16_old_ms"] / rec["bf16_ms"], 2)
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                layer_ms.setdefault(M, {})[name] = {a: rec[a + "_ms"] for a in arms}
            del out, got
    for M, per in layer_ms.items():
        if len(per) == 4:
            rec = dict(kind="7B-decoder-layer", M=M, launches=list(per))
            for a in ("bf16", "bf16_old", "fp16"):
                rec[a + "_ms"] = round(sum(v[a] for v in per.values()), 4)
            rec["bf16_speedup_vs_old"] = round(rec["bf16_old_ms"] / rec["bf16_ms"], 2)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
