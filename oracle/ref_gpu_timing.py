#!/usr/bin/env python3
"""TEST / MEASUREMENT INFRASTRUCTURE (lives under oracle/ because it executes oracle/_ref).

Times, on one GPU, per LLaMA layer shape: our accumulate-mode symbols, our fused path, and the REFERENCE's
own CUDA kernels (oracle/_ref) as the only like-for-like GPU baseline (BASELINE.md section 4).  Weights rotate
through > 2x L2 of distinct copies so every launch streams from HBM; launches are replayed from a CUDA graph
(ours; the reference launches on the legacy stream and cannot be captured, so it is timed eagerly in a
back-to-back loop, which favours it).  Prints one JSON line per (shape, impl).

    gpurun -- 'python oracle/ref_gpu_timing.py > gpurun_out/ref_gpu_timing.jsonl'
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import build_ref  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

PEAK = 3350.0  # H100 SXM data-sheet HBM3 bandwidth (GB/s), unless a measured peak is present
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def synth(bits, K, N, sp, topx, copies, dev="cuda"):
    g = torch.Generator(device=dev).manual_seed(K * 31 + N)
    Ls = []
    nnz = int(round(sp * K * N))
    for _ in range(copies):
        L = dict(bits=bits, K=K, N=N)
        L["qweight"] = torch.randint(-2**31, 2**31 - 1, (K // 32 * bits, N), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
        L["lut"] = torch.sort(torch.randn((N, 2**bits), device=dev, generator=g) * 0.02, dim=1).values.contiguous()
        if nnz:
            r = torch.randint(0, N, (nnz,), device=dev, generator=g)
            counts = torch.bincount(r, minlength=N)
            rows = torch.zeros(N + 1, dtype=torch.int32, device=dev)
            rows[1:] = torch.cumsum(counts, 0).to(torch.int32)
            L["rows"] = rows
            L["cols"] = torch.randint(0, K, (nnz,), device=dev, generator=g).to(torch.int32)
            L["vals"] = torch.randn(nnz, device=dev, generator=g) * 0.1
        if topx:
            L["full_rows"] = torch.zeros((K, topx), device=dev)
            L["fri"] = torch.zeros(topx, dtype=torch.int32, device=dev)
        Ls.append(L)
    return Ls


def alg_bytes(bits, K, N, nnz, topx):
    b = K // 32 * bits * N * 4 + N * (2**bits) * 4 + K * 4 + N * 4
    if nnz:
        b += nnz * 8 + (N + 1) * 4
    if topx:
        b += K * topx * 4 + topx * 4
    return b


def call12(mod, L, x, y):
    b = L["bits"]
    if "rows" in L and "full_rows" in L:
        getattr(mod, f"vecquant{b}matmul_spmv_hybrid_nuq_perchannel")(L["rows"], L["cols"], L["vals"], x, L["full_rows"], L["fri"], y, L["N"], L["qweight"], L["lut"])
    elif "rows" in L:
        getattr(mod, f"vecquant{b}matmul_spmv_nuq_perchannel")(L["rows"], L["cols"], L["vals"], x, y, L["N"], L["qweight"], L["lut"])
    else:
        getattr(mod, f"vecquant{b}matmul_nuq_perchannel")(x, L["qweight"], y, L["lut"])


def time_loop(fn, n_iter, graph):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(n_iter):
            ev0.record(); g.replay(); ev1.record(); torch.cuda.synchronize()
            best = min(best, ev0.elapsed_time(ev1))
        return best
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(n_iter):
        ev0.record(); fn(); ev1.record(); torch.cuda.synchronize()
        best = min(best, ev0.elapsed_time(ev1))
    return best


def main():
    ref = build_ref.load() if build_ref.have_ref_so() else None
    shapes = [(4, 4096, 4096, 0.0, 0), (4, 4096, 11008, 0.0, 0), (4, 11008, 4096, 0.0, 0),
              (4, 4096, 4096, 0.0045, 10), (4, 4096, 11008, 0.0045, 10), (4, 11008, 4096, 0.0045, 10),
              (3, 4096, 4096, 0.0, 0), (3, 4096, 4096, 0.0045, 10), (3, 4096, 11008, 0.0045, 10), (3, 11008, 4096, 0.0045, 10),
              (4, 5120, 5120, 0.0005, 10), (4, 5120, 13824, 0.0005, 10), (3, 8192, 8192, 0.0045, 10)]
    if len(sys.argv) > 1 and sys.argv[1] == "--quick":
        shapes = shapes[:1] + shapes[3:4] + shapes[7:8]
    for bits, K, N, sp, topx in shapes:
        wbytes = K // 32 * bits * N * 4
        copies = max(2, int(2.2 * 128e6 / wbytes) + 1)
        Ls = synth(bits, K, N, sp, topx, copies)
        nnz = int(round(sp * K * N))
        B = alg_bytes(bits, K, N, nnz, topx)
        x32 = torch.randn(K, device="cuda").half().float()
        x16 = x32.half()
        ys = [torch.zeros(N, device="cuda") for _ in range(copies)]

        def ours_acc():
            for L, y in zip(Ls, ys):
                call12(qc, L, x32, y)

        def ours_fused():
            for L in Ls:
                qc.lutgemv_fused(x16, L["qweight"], L["lut"], bits, None, L.get("rows"), L.get("cols"), L.get("vals"), L.get("full_rows"), L.get("fri"))

        def theirs():
            for L, y in zip(Ls, ys):
                call12(ref, L, x32, y)

        def ours_fused_lut16():
            qc.set_lut_mode("fp16")
            try:
                ours_fused()
            finally:
                qc.set_lut_mode("exact")

        res = []
        for name, fn, graph in (("ours_accumulate", ours_acc, True), ("ours_fused_fp16", ours_fused, True), ("ours_fused_fp16_lut16", ours_fused_lut16, True),
                                ("reference_kernel", theirs, False)):
            if fn is theirs and (ref is None or K % 128 or N % 128):
                continue
            ms = time_loop(fn, 10, graph)
            us = ms * 1e3 / copies
            res.append(dict(impl=name, bits=bits, K=K, N=N, sparsity=sp, topX=topx, us_per_gemv=round(us, 3), alg_bytes=B,
                            gbs=round(B / us / 1e3, 1), frac_of_measured_peak=round(B / us / 1e3 / PEAK, 3), copies=copies))
            print(json.dumps(res[-1]), flush=True)


def batched():
    """The *_batched symbols (prefill-shaped inputs, SURVEY 8(f) row 3): ours (register-tiled LUT GEMM + batched outlier kernels)
    against the reference's own batched kernels on the same GPU, eager launches on both sides, B rows of a 4096 x 4096 layer."""
    ref = build_ref.load() if build_ref.have_ref_so() else None
    for bits, K, N, sp, topx in [(4, 4096, 4096, 0.0, 0), (4, 4096, 4096, 0.0045, 10), (3, 4096, 4096, 0.0045, 10)]:
        L = synth(bits, K, N, sp, topx, 1)[0]
        for B in (16, 64, 2048):
            x = torch.randn((B, K), device="cuda").half().float()
            out = {}
            for name, mod in (("ours_batched", qc), ("reference_batched", ref)):
                if mod is None:
                    continue
                y = torch.zeros((B, N), device="cuda")

                def fn():
                    b = L["bits"]
                    if "rows" in L and "full_rows" in L:
                        getattr(mod, f"vecquant{b}matmul_spmv_hybrid_nuq_perchannel_batched")(L["rows"], L["cols"], L["vals"], x, L["full_rows"], L["fri"], y, N, L["qweight"], L["lut"])
                    elif "rows" in L:
                        getattr(mod, f"vecquant{b}matmul_spmv_nuq_perchannel_batched")(L["rows"], L["cols"], L["vals"], x, y, N, L["qweight"], L["lut"])
                    else:
                        getattr(mod, f"vecquant{b}matmul_nuq_perchannel_batched")(x, L["qweight"], y, L["lut"])
                out[name] = time_loop(fn, 5, False)
            rec = dict(kind="batched", bits=bits, K=K, N=N, sparsity=sp, topX=topx, batch=B, ours_ms=round(out["ours_batched"], 4),
                       ours_tflops=round(2.0 * B * K * N / out["ours_batched"] / 1e9, 2))
            if "reference_batched" in out:
                rec.update(reference_ms=round(out["reference_batched"], 4), speedup=round(out["reference_batched"] / out["ours_batched"], 2))
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--batched":
        batched()
    else:
        main()
