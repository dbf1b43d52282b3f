#!/usr/bin/env python3
"""Input-gradient timing on one GPU: dx = dy . W^T of the LLaMA-7B layers as the model runs them (q/k/v and gate/up stacked) and
one 65B w3 layer, at M = 1 ... 2048 rows of fp16 dy.

Arms:
  tc          quant_cuda.lutgemm_t(path="tc"): the transposed LUT-GEMM on the tensor cores (one launch)
  cuda        quant_cuda.lutgemm_t(path="cuda"): the transposed LUT-GEMM on the CUDA cores (one launch)
  dense       W dequantized once to fp16 (outliers and dense rows included, outside the timing), then dy @ W.T (cuBLAS): the speed
              a user with memory to spare for a dense copy of every layer could get

Per (shape, M) one JSON line: ms of every arm and the max relative error of the tc and dense arms against the cuda arm.  The arms are
alternated inside each repetition and the median of 5 is kept.  Per M one more line sums the four launches of one 7B decoder
layer per arm.  The first line names the card and its power limit (nvidia-smi, read-only query).

    python tests/perf/backward_timing.py [--quick]
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
from prefill_tc_timing import SHAPES, rel, synth, time_ms  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

ROWS = [1, 8, 32, 64, 96, 128, 512, 2048]


def dense_w(L):
    """W [K, N] fp16 from the layer's buffers: codebook gather, CSR entries and dense rows folded in (fp32, then one rounding)."""
    K, N, bits = L["K"], L["N"], L["bits"]
    eye = torch.eye(N, device="cuda", dtype=torch.float16)
    # dx of the identity: row c of dy = e_c gives column c of W (exact: one product per output)
    W = torch.cat([qc.lutgemm_t(eye[c0:c0 + 1024].float(), L["qweight"], L["lut"], bits, L["rows"], L["cols"], L["vals"],
                                L["full_rows"], L["fri"], path="cuda") for c0 in range(0, N, 1024)]).t()
    return W.contiguous().half()


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    shapes, rows = (SHAPES[:2], [1, 64]) if quick else (SHAPES, ROWS)
    layer_ms = {}
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        lay = (L["qweight"], L["lut"], bits, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        W = dense_w(L)
        for M in rows:
            dy = torch.randn((M, N), device="cuda").half()
            out = {}
            arms = {
                "tc": lambda: out.__setitem__("tc", qc.lutgemm_t(dy, *lay, path="tc")),
                "cuda": lambda: out.__setitem__("cuda", qc.lutgemm_t(dy, *lay, path="cuda")),
                "dense": lambda: out.__setitem__("dense", dy @ W.t()),
            }
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: out[a].float().clone() for a in arms}
            t = {a: [] for a in arms}
            for a, fn in arms.items():  # warm-up, and size the loop to about 20 ms per measurement
                t0 = time_ms(fn, 1)
                t[a + "_n"] = max(1, min(200, int(20.0 / max(t0, 1e-3))))
            for _ in range(3 if quick else 5):
                for a, fn in arms.items():
                    t[a].append(time_ms(fn, t[a + "_n"]))
            rec = dict(kind="backward", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(statistics.median(t[a]), 5)
            rec["tc_max_rel_err_vs_cuda"] = float(f"{rel(got['tc'], got['cuda']):.3e}")
            rec["dense_max_rel_err_vs_cuda"] = float(f"{rel(got['dense'], got['cuda']):.3e}")
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                layer_ms.setdefault(M, {})[name] = {a: rec[a + "_ms"] for a in arms}
            del out, got
        del W
    for M, per in layer_ms.items():
        if len(per) == 4:
            rec = dict(kind="7B-decoder-layer", M=M, launches=list(per))
            for a in ("tc", "cuda", "dense"):
                rec[a + "_ms"] = round(sum(v[a] for v in per.values()), 4)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
