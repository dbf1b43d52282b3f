#!/usr/bin/env python3
"""Few-row timing on one GPU: the multi-row LUT-GEMV (`quant_cuda.lutgemv_rows`, fp16 x) against the other ways of running 2 to 63
rows, on the LLaMA-7B layers as the model runs them (q/k/v and gate/up stacked) and one 65B w3 layer, at M = 2 ... 63 rows.

Arms:
  rows        quant_cuda.lutgemv_rows (one launch)
  batched     the _batched symbols as QuantLinearLUT.forward runs them: torch.zeros, x.float(), the hybrid symbol, out.to(fp16)
  tc          quant_cuda.lutgemm_fused (the tensor-core kernel of 64 rows and more)
  gemv_xM     M calls of quant_cuda.lutgemv_fused (the one-GEMV kernel), one per row
  reference   where oracle/_ref was built: the reference's batched kernels, onto a zeroed fp32 output

Per (shape, M) one JSON line: ms of every arm and the max relative error of each arm against the rows arm on the timed inputs.
The arms are alternated inside each repetition and the median of 5 is kept.  Per M one more line sums the four launches of one
7B decoder layer per arm.  The first line names the card and its power limit (nvidia-smi, read-only query).

    python tests/perf/rows_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import build_ref  # noqa: E402
from prefill_tc_timing import SHAPES, batched_call, rel, synth, time_ms  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

ROWS = [2, 4, 8, 16, 32, 48, 63]


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    ref = build_ref.load() if build_ref.have_ref_so() else None
    shapes, rows = (SHAPES[:2], [2, 8]) if quick else (SHAPES, ROWS)
    layer_ms = {}
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        lay = (L["qweight"], L["lut"], bits, None, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        for M in rows:
            x16 = torch.randn((M, K), device="cuda").half()
            out = {}

            def module_batched():
                y = torch.zeros((M, N), device="cuda", dtype=torch.float32)
                batched_call(qc, L, x16.float(), y)
                out["batched"] = y.to(torch.float16)

            arms = {
                "rows": lambda: out.__setitem__("rows", qc.lutgemv_rows(x16, *lay)),
                "batched": module_batched,
                "tc": lambda: out.__setitem__("tc", qc.lutgemm_fused(x16, *lay)),
                "gemv_xM": lambda: out.__setitem__("gemv_xM", [qc.lutgemv_fused(x16[i], *lay) for i in range(M)]),
            }
            if ref is not None:
                yref = torch.zeros((M, N), device="cuda")
                x32 = x16.float()

                def reference():
                    yref.zero_()
                    batched_call(ref, L, x32, yref)
                    out["reference"] = yref
                arms["reference"] = reference
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: (torch.stack(out[a]) if a == "gemv_xM" else out[a]).float().clone() for a in arms}
            t = {a: [] for a in arms}
            for a, fn in arms.items():  # warm-up, and size the loop to about 20 ms per measurement
                t0 = time_ms(fn, 1)
                t[a + "_n"] = max(1, min(200, int(20.0 / max(t0, 1e-3))))
            for _ in range(3 if quick else 5):
                for a, fn in arms.items():
                    t[a].append(time_ms(fn, t[a + "_n"]))
            rec = dict(kind="rows", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(statistics.median(t[a]), 5)
                if a != "rows":
                    rec[a + "_max_rel_err_vs_rows"] = float(f"{rel(got[a], got['rows']):.3e}")
            rec["rows_speedup_vs_batched"] = round(rec["batched_ms"] / rec["rows_ms"], 2)
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                layer_ms.setdefault(M, {})[name] = {a: rec[a + "_ms"] for a in arms}
            del out, got
    for M, per in layer_ms.items():
        if len(per) == 4:
            arms = list(next(iter(per.values())))
            rec = dict(kind="7B-decoder-layer", M=M, launches=list(per))
            for a in arms:
                rec[a + "_ms"] = round(sum(v[a] for v in per.values()), 4)
            rec["rows_speedup_vs_batched"] = round(rec["batched_ms"] / rec["rows_ms"], 2)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
