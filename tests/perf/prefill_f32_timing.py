#!/usr/bin/env python3
"""fp32 prefill / evaluation timing on one GPU: the tensor-core LUT-GEMM with fp32 x (`quant_cuda.lutgemm_fused_f32`: x and the
weights each split exactly into three bf16 parts, six part products per k-step) against the route fp32 x takes without it, as
QuantLinearLUT runs it (zeros, the _batched hybrid symbol), and against the bf16 tensor-core kernel on the bf16-rounded x (what the
x split costs).  Same layers and rules as prefill_tc_timing.py: the LLaMA-7B w4-s45 layers with 10 dense rows as the model runs them
(q/k/v and gate/up stacked) and one 65B w3 layer, at M = 32 ... 2048.

Per (shape, M) one JSON line: median ms of every arm, TFLOP/s counted once (2 M K N / t) and the MMA work actually issued by the
tensor-core arms (M and N padded to the 128 x 128 tile, K to the 64-k chunk; 6 part products for fp32 x, 3 for bf16 x), the max
relative error between the arms, and the max relative error of the two fp32 arms against the fp64 oracle on sampled rows of the
timed inputs.  The arms are alternated inside each repetition.  After the shapes, one line per M sums the four launches of one 7B
decoder layer, and a last line names the smallest measured M from which the tensor cores are faster on that layer at every larger
measured M as well (QuantLinearLUT.FP32_TC_MIN_ROWS).  The first line names the card, its power limit and max SM clock
(nvidia-smi, read-only query).

    python tests/perf/prefill_f32_timing.py [--quick]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from prefill_bf16_timing import timed_arms  # noqa: E402
from prefill_tc_timing import ROOT, SHAPES, batched_call, qc, rel, synth  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import oracle as orc  # noqa: E402

ROWS = [32, 64, 96, 128, 192, 256, 512, 2048]
ARMS = ("f32_tc", "f32_batched", "bf16_tc")


def oracle_layer(L):
    """The synthetic layer (torch, prefill_tc_timing.synth) as the oracle's numpy dict."""
    c = lambda k: L[k].cpu().numpy()
    return dict(bits=L["bits"], infeatures=L["K"], outfeatures=L["N"], qweight=c("qweight"), lookup_table=c("lut"), rows=c("rows"),
                cols=c("cols"), vals=c("vals"), full_rows=c("full_rows"), full_row_indices=c("fri"))


def issued_flops(M, K, N, parts):
    return 2.0 * parts * (-(-M // 128) * 128) * (-(-K // 64) * 64) * (-(-N // 128) * 128)


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    shapes, rows = (SHAPES[:2], [64, 512]) if quick else (SHAPES, ROWS)
    layer = {}  # M -> launches and ms per arm summed over the 7B shapes
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        OL = oracle_layer(L)
        lay = (L["qweight"], L["lut"], bits, None, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        for M in rows:
            x32 = torch.randn((M, K), device="cuda")  # full 24-bit mantissas: x_l is non-zero
            xb = x32.bfloat16()
            out = {}

            def batched():  # QuantLinearLUT's batched branch for fp32 x
                y = torch.zeros((M, N), device="cuda")
                batched_call(qc, L, x32, y)
                out["f32_batched"] = y
            arms = {
                "f32_tc": lambda: out.__setitem__("f32_tc", qc.lutgemm_fused_f32(x32, *lay)),
                "f32_batched": batched,
                "bf16_tc": lambda: out.__setitem__("bf16_tc", qc.lutgemm_fused(xb, *lay)),
            }
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: out[a].float() for a in arms}
            ms = timed_arms(arms, quick)
            rec = dict(kind="prefill_f32", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(ms[a], 4)
                rec[a + "_tflops"] = round(2.0 * M * K * N / ms[a] / 1e9, 2)
            rec["f32_tc_issued_tflops"] = round(issued_flops(M, K, N, 6) / ms["f32_tc"] / 1e9, 2)
            rec["bf16_tc_issued_tflops"] = round(issued_flops(M, K, N, 3) / ms["bf16_tc"] / 1e9, 2)
            for a in ("f32_batched", "bf16_tc"):
                rec[a + "_max_rel_err_vs_f32_tc"] = float(f"{rel(got[a], got['f32_tc']):.3e}")
            sample = sorted({0, M // 2, M - 1})
            want = torch.from_numpy(orc.forward_f64(OL, x32[sample].cpu().numpy()))
            for a in ("f32_tc", "f32_batched"):
                rec[a + "_max_rel_err_vs_oracle"] = float(f"{rel(got[a][sample].cpu(), want):.3e}")
            rec["f32_tc_speedup_vs_f32_batched"] = round(ms["f32_batched"] / ms["f32_tc"], 2)
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                acc = layer.setdefault(M, {"launches": [], **{a: 0.0 for a in ARMS}})
                acc["launches"].append(name)
                for a in ARMS:
                    acc[a] += ms[a]
            del out, got
    faster = {}
    for M, acc in sorted(layer.items()):
        if len(acc["launches"]) == 4:
            faster[M] = acc["f32_tc"] < acc["f32_batched"]
            print(json.dumps(dict(kind="7B-decoder-layer-f32", M=M, launches=acc["launches"],
                                  **{a + "_ms": round(acc[a], 3) for a in ARMS},
                                  f32_tc_speedup_vs_f32_batched=round(acc["f32_batched"] / acc["f32_tc"], 2),
                                  f32_tc_over_bf16_tc=round(acc["f32_tc"] / acc["bf16_tc"], 2))), flush=True)
    if faster:
        ms_ = sorted(faster)
        pick = next((m for i, m in enumerate(ms_) if all(faster[n] for n in ms_[i:])), None)
        print(json.dumps(dict(kind="fp32_tc_min_rows", measured=ms_, faster=[faster[m] for m in ms_], smallest_from_which_faster=pick)),
              flush=True)


if __name__ == "__main__":
    main()
