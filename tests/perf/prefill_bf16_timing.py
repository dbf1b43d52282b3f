#!/usr/bin/env python3
"""bf16 prefill / evaluation timing on one GPU: the tensor-core LUT-GEMM with bf16 x (`quant_cuda.lutgemm_fused`, three bf16 weight
parts) against the same kernel on the same values rounded to fp16 (what the third part costs) and the route bf16 x takes without it,
as QuantLinearLUT runs it (zeros, x.float(), the _batched hybrid symbol, .to(bf16)).  Same layers and rules as
prefill_tc_timing.py: the LLaMA-7B layers as the model runs them (q/k/v and gate/up stacked) and one 65B w3 layer, at M = 32 ... 2048.

Per (shape, M) one JSON line: ms and TFLOP/s (2 M K N / t) of every arm, and the max relative error of the other two arms against
the bf16 tensor-core arm on the timed inputs.  The arms are alternated inside each repetition and the median is kept.  After the
shapes, one line per M sums the four launches of one 7B decoder layer: where the tensor cores beat the batched route picks
QuantLinearLUT.BF16_TC_MIN_ROWS.  The first line names the card and its power limit (nvidia-smi, read-only query).

    python tests/perf/prefill_bf16_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from prefill_tc_timing import SHAPES, batched_call, qc, rel, synth, time_ms  # noqa: E402

ROWS = [32, 48, 64, 80, 96, 128, 512, 2048]
ARMS = ("bf16_tc", "fp16_tc", "bf16_batched")


def timed_arms(arms, quick):
    """Median ms of each arm: warm-up, loops sized to about 20 ms, the arms alternated inside each repetition."""
    t = {a: [] for a in arms}
    n = {a: max(1, min(50, int(20.0 / max(time_ms(fn, 1), 1e-3)))) for a, fn in arms.items()}
    for _ in range(3 if quick else 5):
        for a, fn in arms.items():
            t[a].append(time_ms(fn, n[a]))
    return {a: statistics.median(v) for a, v in t.items()}


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    shapes, rows = (SHAPES[:2], [64, 512]) if quick else (SHAPES, ROWS)
    layer = {}  # M -> launches and ms per arm summed over the 7B shapes
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        lay = (L["qweight"], L["lut"], bits, None, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        for M in rows:
            xb = torch.randn((M, K), device="cuda").bfloat16()
            x16 = xb.half()  # the same values: bf16 values of this range are exact in fp16
            out = {}

            def batched():  # QuantLinearLUT's batched branch for bf16 x
                y = torch.zeros((M, N), device="cuda")
                batched_call(qc, L, xb.float(), y)
                out["bf16_batched"] = y.to(torch.bfloat16)
            arms = {
                "bf16_tc": lambda: out.__setitem__("bf16_tc", qc.lutgemm_fused(xb, *lay)),
                "fp16_tc": lambda: out.__setitem__("fp16_tc", qc.lutgemm_fused(x16, *lay)),
                "bf16_batched": batched,
            }
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: out[a].float() for a in arms}
            ms = timed_arms(arms, quick)
            rec = dict(kind="prefill_bf16", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(ms[a], 4)
                rec[a + "_tflops"] = round(2.0 * M * K * N / ms[a] / 1e9, 2)
            for a in ("fp16_tc", "bf16_batched"):
                rec[a + "_max_rel_err_vs_bf16_tc"] = float(f"{rel(got[a], got['bf16_tc']):.3e}")
            rec["bf16_tc_speedup_vs_bf16_batched"] = round(ms["bf16_batched"] / ms["bf16_tc"], 2)
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                acc = layer.setdefault(M, {"launches": [], **{a: 0.0 for a in ARMS}})
                acc["launches"].append(name)
                for a in ARMS:
                    acc[a] += ms[a]
            del out, got
    for M, acc in layer.items():
        if len(acc["launches"]) == 4:
            print(json.dumps(dict(kind="7B-decoder-layer-bf16", M=M, launches=acc["launches"],
                                  **{a + "_ms": round(acc[a], 3) for a in ARMS},
                                  bf16_tc_speedup_vs_bf16_batched=round(acc["bf16_batched"] / acc["bf16_tc"], 2),
                                  bf16_tc_over_fp16_tc=round(acc["bf16_tc"] / acc["fp16_tc"], 2))), flush=True)


if __name__ == "__main__":
    main()
