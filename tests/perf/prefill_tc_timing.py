#!/usr/bin/env python3
"""Prefill / evaluation timing on one GPU: the tensor-core LUT-GEMM (`quant_cuda.lutgemm_fused`, fp16 x) against our batched
symbols (CUDA cores, fp32 x) and, where oracle/_ref was built, the reference's own batched kernels, on the LLaMA-7B layers as the
model runs them (q/k/v and gate/up stacked) and one 65B w3 layer, at M = 8 ... 2048 rows.

Per (shape, M) one JSON line: ms and TFLOP/s (2 M K N / t) of every arm, and the max relative error of each arm against the
tensor-core arm on the timed inputs.  The arms are alternated inside each repetition and the median is kept.  A last line sums
the four launches of one 7B decoder layer at M = 2048 into a prefill tokens/s figure.  The first line names the card and its
power limit (nvidia-smi, read-only query).

    python tests/perf/prefill_tc_timing.py [--quick]
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
import build_ref  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

SHAPES = [  # (name, bits, K, N, sparsity, topX)
    ("7B-qkv", 4, 4096, 12288, 0.0045, 10),
    ("7B-o", 4, 4096, 4096, 0.0045, 10),
    ("7B-gate_up", 4, 4096, 22016, 0.0045, 10),
    ("7B-down", 4, 11008, 4096, 0.0045, 10),
    ("65B-qkvo-w3", 3, 8192, 8192, 0.0045, 10),
]
ROWS = [8, 16, 32, 64, 128, 512, 2048]


def synth(bits, K, N, sp, topx, dev="cuda"):
    """Random layer in the checkpoint format: CSR rows with ascending columns (as the reference packer writes them), topX
    non-zero dense rows on distinct channels."""
    g = torch.Generator(device=dev).manual_seed(K * 31 + N)
    L = dict(bits=bits, K=K, N=N)
    L["qweight"] = torch.randint(-2**31, 2**31 - 1, (K // 32 * bits, N), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
    L["lut"] = torch.sort(torch.randn((N, 2**bits), device=dev, generator=g) * 0.02, dim=1).values.contiguous()
    nnz = int(round(sp * K * N))
    r = torch.randint(0, N, (nnz,), device=dev, generator=g)
    c = torch.randint(0, K, (nnz,), device=dev, generator=g)
    key = torch.unique(r.to(torch.int64) * K + c)  # sorted: by row, then column; duplicates dropped
    r, c = key // K, key % K
    rows = torch.zeros(N + 1, dtype=torch.int32, device=dev)
    rows[1:] = torch.cumsum(torch.bincount(r, minlength=N), 0).to(torch.int32)
    L["rows"], L["cols"] = rows, c.to(torch.int32).contiguous()
    L["vals"] = torch.randn(key.numel(), device=dev, generator=g) * 0.1
    L["full_rows"] = torch.randn((K, topx), device=dev, generator=g) * 0.05
    L["fri"] = torch.randperm(N, device=dev, generator=g)[:topx].to(torch.int32)
    return L


def batched_call(mod, L, x, y):
    getattr(mod, f"vecquant{L['bits']}matmul_spmv_hybrid_nuq_perchannel_batched")(
        L["rows"], L["cols"], L["vals"], x, L["full_rows"], L["fri"], y, L["N"], L["qweight"], L["lut"])


def time_ms(fn, n):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n


def rel(a, b):
    a, b = a.double(), b.double()
    den = torch.maximum(b.abs(), 1e-2 * b.abs().max())
    return float(((a - b).abs() / den).max())


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    ref = build_ref.load() if build_ref.have_ref_so() else None
    shapes, rows = (SHAPES[:2], [16, 512]) if quick else (SHAPES, ROWS)
    layer_ms = {}
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        for M in rows:
            x16 = torch.randn((M, K), device="cuda").half()
            x32 = x16.float()
            ys = {"ours_batched": torch.zeros((M, N), device="cuda"), "reference_batched": torch.zeros((M, N), device="cuda")}
            out = {}
            arms = {
                "ours_tc": lambda: out.__setitem__("ours_tc", qc.lutgemm_fused(x16, L["qweight"], L["lut"], bits, None, L["rows"],
                                                                                L["cols"], L["vals"], L["full_rows"], L["fri"])),
                "ours_batched": lambda: batched_call(qc, L, x32, ys["ours_batched"]),
            }
            if ref is not None:
                arms["reference_batched"] = lambda: batched_call(ref, L, x32, ys["reference_batched"])
            # outputs for the error check: one call each from zero
            for a, fn in arms.items():
                if a in ys:
                    ys[a].zero_()
                fn()
            torch.cuda.synchronize()
            got = {"ours_tc": out["ours_tc"].float(), **{a: ys[a].clone() for a in arms if a in ys}}
            t = {a: [] for a in arms}
            for a, fn in arms.items():  # warm-up, and size the loop to about 20 ms per measurement
                t0 = time_ms(fn, 1)
                t[a + "_n"] = max(1, min(50, int(20.0 / max(t0, 1e-3))))
            for _ in range(3 if quick else 5):
                for a, fn in arms.items():
                    t[a].append(time_ms(fn, t[a + "_n"]))
            rec = dict(kind="prefill", shape=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, M=M)
            for a in arms:
                ms = statistics.median(t[a])
                rec[a + "_ms"] = round(ms, 4)
                rec[a + "_tflops"] = round(2.0 * M * K * N / ms / 1e9, 2)
                if a != "ours_tc":
                    rec[a + "_max_rel_err_vs_tc"] = float(f"{rel(got[a], got['ours_tc']):.3e}")
            rec["tc_speedup_vs_ours_batched"] = round(rec["ours_batched_ms"] / rec["ours_tc_ms"], 2)
            print(json.dumps(rec), flush=True)
            if M == 2048 and name.startswith("7B"):
                layer_ms[name] = (rec["ours_tc_ms"], rec["ours_batched_ms"])
            del out, got, ys
    if len(layer_ms) == 4:
        tc_ms, b_ms = sum(v[0] for v in layer_ms.values()), sum(v[1] for v in layer_ms.values())
        print(json.dumps(dict(kind="7B-decoder-layer", M=2048, launches=list(layer_ms), ours_tc_ms=round(tc_ms, 3),
                              ours_batched_ms=round(b_ms, 3), ours_tc_tokens_per_s_per_layer=round(2048 / tc_ms * 1e3),
                              ours_batched_tokens_per_s_per_layer=round(2048 / b_ms * 1e3),
                              ours_tc_7B_prefill_tokens_per_s_32_layers=round(2048 / (32 * tc_ms) * 1e3))), flush=True)


if __name__ == "__main__":
    main()
