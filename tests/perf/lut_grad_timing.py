#!/usr/bin/env python3
"""Codebook-gradient timing on one GPU: (dlut, dvals, dfull_rows) of the LLaMA-7B layers as the model runs them (q/k/v and gate/up
stacked) and one 65B 8192 x 8192 layer, all 4-bit with 0.45 % CSR outliers and 10 dense rows, at M = 1 ... 2048 rows of fp16 x
and dy.

Arms:
  tc          quant_cuda.lut_grad(path="tc"): G = x^T . dy on the tensor cores, bucketed in the epilogue (one launch)
  cuda        quant_cuda.lut_grad(path="cuda"): the same on the CUDA cores (one launch)
  cuda_mixed  the CUDA cores with fp16 x and fp32 dy (the gradient of a layer with a bias under fp16 activations)
  torch       G = x.float().T @ dy.float() (fp32 cuBLAS), then index_add_ into the bins; the indices are unpacked and turned into
              bin keys outside the timed region; dlut only
  lutgemm_t   the layer's input gradient dx = dy . W^T (quant_cuda.lutgemm_t, path auto), for scale

Per (shape, M) one JSON line: ms of every arm (median of 5, arms alternated inside each repetition), TFLOP/s of the tc, cuda and
cuda_mixed arms from 2 M K N, and the max relative difference of the dlut of the cuda, cuda_mixed and torch arms against the tc
arm.  Per M one more
line sums one 7B decoder layer's four launches per arm.  The first line names the card and its power limit (nvidia-smi,
read-only query).

    python tests/perf/lut_grad_timing.py [--quick]
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
from prefill_tc_timing import rel, synth, time_ms  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

SHAPES = [  # (name, bits, K, N, sparsity, topX)
    ("7B-qkv", 4, 4096, 12288, 0.0045, 10),
    ("7B-o", 4, 4096, 4096, 0.0045, 10),
    ("7B-gate_up", 4, 4096, 22016, 0.0045, 10),
    ("7B-down", 4, 11008, 4096, 0.0045, 10),
    ("65B-8192", 4, 8192, 8192, 0.0045, 10),
]
ROWS = [1, 8, 64, 128, 512, 2048]


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
        nv = 1 << bits
        key = (qc.unpack_indices(L["qweight"], bits).long() + torch.arange(N, device="cuda")[None, :] * nv).reshape(-1)
        for M in rows:
            g = torch.Generator(device="cuda").manual_seed(M)
            x = torch.randn((M, K), device="cuda", generator=g).half()
            dy = torch.randn((M, N), device="cuda", generator=g).half()
            dy32 = dy.float()
            out = {}

            def grad(path, d=dy):
                return qc.lut_grad(x, d, *lay, want_lut=True, want_vals=True, want_full_rows=True, path=path)

            def torch_arm():
                G = x.float().t() @ dy.float()
                return torch.zeros(N * nv, device="cuda").index_add_(0, key, G.reshape(-1)).reshape(N, nv)

            arms = {
                "tc": lambda: out.__setitem__("tc", grad("tc")[0]),
                "cuda": lambda: out.__setitem__("cuda", grad("cuda")[0]),
                "cuda_mixed": lambda: out.__setitem__("cuda_mixed", grad("cuda", dy32)[0]),
                "torch": lambda: out.__setitem__("torch", torch_arm()),
                "lutgemm_t": lambda: qc.lutgemm_t(dy, *lay),
            }
            for fn in arms.values():
                fn()
            torch.cuda.synchronize()
            got = {a: out[a].clone() for a in ("tc", "cuda", "cuda_mixed", "torch")}
            t = {a: [] for a in arms}
            n = {}
            for a, fn in arms.items():  # warm-up, and size the loop to about 20 ms per measurement
                n[a] = max(1, min(200, int(20.0 / max(time_ms(fn, 1), 1e-3))))
            for _ in range(3 if quick else 5):
                for a, fn in arms.items():
                    t[a].append(time_ms(fn, n[a]))
            rec = dict(kind="lut_grad", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                rec[a + "_ms"] = round(statistics.median(t[a]), 5)
            for a in ("tc", "cuda", "cuda_mixed"):
                rec[a + "_tflops"] = round(2.0 * M * K * N / (rec[a + "_ms"] * 1e-3) / 1e12, 2)
            rec["cuda_dlut_max_rel_diff_vs_tc"] = float(f"{rel(got['cuda'], got['tc']):.3e}")
            rec["cuda_mixed_dlut_max_rel_diff_vs_tc"] = float(f"{rel(got['cuda_mixed'], got['tc']):.3e}")
            rec["torch_dlut_max_rel_diff_vs_tc"] = float(f"{rel(got['torch'], got['tc']):.3e}")
            print(json.dumps(rec), flush=True)
            if name.startswith("7B"):
                layer_ms.setdefault(M, {})[name] = {a: rec[a + "_ms"] for a in arms}
            del out, got
        del key
    for M, per in layer_ms.items():
        if len(per) == 4:
            rec = dict(kind="7B-decoder-layer", M=M, launches=list(per))
            for a in ("tc", "cuda", "cuda_mixed", "torch", "lutgemm_t"):
                rec[a + "_ms"] = round(sum(v[a] for v in per.values()), 4)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
