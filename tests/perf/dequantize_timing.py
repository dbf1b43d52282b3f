#!/usr/bin/env python3
"""Dequantize timing on one GPU: W [out, in] of the LLaMA-7B layers as the model runs them (q/k/v and gate/up stacked; w4, 0.45 %
CSR outliers, 10 dense rows) and one 65B w3 layer, with fp16 and fp32 output.

Arms:
  kernel   quant_cuda.dequantize: one launch (decode, outlier fold, transpose through shared memory, 16-byte stores)
  torch    the same W from tensor ops: the indices unpacked with shifts and masks, the codebook gathered, the CSR entries added
           with index_put_(accumulate=True), the dense rows with index_add_, then one cast

Per (shape, dtype) one JSON line: ms of both arms (median of 5 alternating repetitions, CUDA events around many launches), the
algorithmic bytes (qweight, codebook, CSR and dense rows read, W written), the kernel's GB/s, that rate as a fraction of the H100 SXM
data-sheet bandwidth (3.35 TB/s: a data-sheet figure, not a reached one), and the largest difference between the arms.  The
first line names the card and its power limit (nvidia-smi, read-only query).

    python tests/perf/dequantize_timing.py [--quick]
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
from prefill_tc_timing import SHAPES, synth, time_ms  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

NAMES = ("7B-qkv", "7B-o", "7B-gate_up", "7B-down", "65B-qkvo-w3")
DATASHEET_BPS = 3.35e12


def torch_dequant(L, dtype):
    bits, K, N = L["bits"], L["K"], L["N"]
    q = L["qweight"].to(torch.int64) & 0xFFFFFFFF
    if bits == 4:
        sh = 4 * torch.arange(8, device=q.device)
        idx = ((q[:, None, :] >> sh[None, :, None]) & 15).reshape(K, N)
    else:
        w0, w1, w2 = q[0::3], q[1::3], q[2::3]
        s = 3 * torch.arange(10, device=q.device)[None, :, None]
        idx = torch.cat([(w0[:, None] >> s) & 7, ((w0 >> 30) | ((w1 & 1) << 2))[:, None], (w1[:, None] >> (s + 1)) & 7,
                         ((w1 >> 31) | ((w2 & 3) << 1))[:, None], (w2[:, None] >> (s + 2)) & 7], dim=1).reshape(K, N)
    W = L["lut"].gather(1, idx.t())
    r = torch.repeat_interleave(torch.arange(N, device=q.device), torch.diff(L["rows"]).to(torch.int64))
    W.index_put_((r, L["cols"].to(torch.int64)), L["vals"], accumulate=True)
    W.index_add_(0, L["fri"].to(torch.int64), L["full_rows"].t())
    return W.to(dtype)


def algo_bytes(L, dtype):
    K, N, bits, topx = L["K"], L["N"], L["bits"], L["full_rows"].shape[1]
    read = K // 32 * bits * N * 4 + N * 2 ** bits * 4 + (N + 1) * 4 + L["cols"].numel() * 8 + K * topx * 4 + topx * 4
    return read, N * K * torch.empty((), dtype=dtype).element_size()


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    shapes = [s for s in SHAPES if s[0] in NAMES][:2 if quick else None]
    reps, n = (2, 5) if quick else (5, 100)
    for name, bits, K, N, sp, topx in shapes:
        L = synth(bits, K, N, sp, topx)
        lay = (L["qweight"], L["lut"], bits, L["rows"], L["cols"], L["vals"], L["full_rows"], L["fri"])
        for dtype in (torch.float16, torch.float32):
            arms = {"kernel": lambda: qc.dequantize(*lay, dtype=dtype), "torch": lambda: torch_dequant(L, dtype)}
            diff = float((arms["kernel"]().float() - arms["torch"]().float()).abs().max())
            ms = {a: [] for a in arms}
            for _ in range(reps):
                for a, fn in arms.items():
                    time_ms(fn, 3)  # warm-up of this arm (allocator, caches)
                    ms[a].append(time_ms(fn, n))
            med = {a: statistics.median(v) for a, v in ms.items()}
            rd, wr = algo_bytes(L, dtype)
            gbps = (rd + wr) / (med["kernel"] * 1e-3) / 1e9
            print(json.dumps({"shape": name, "bits": bits, "K": K, "N": N, "nnz": L["cols"].numel(), "topX": topx,
                              "dtype": str(dtype).replace("torch.", ""), "kernel_ms": round(med["kernel"], 4),
                              "torch_ms": round(med["torch"], 4), "bytes_read": rd, "bytes_written": wr,
                              "kernel_GBps": round(gbps, 1), "frac_of_3.35TBps": round(gbps * 1e9 / DATASHEET_BPS, 3),
                              "speedup_vs_torch": round(med["torch"] / med["kernel"], 2), "max_abs_diff": diff}), flush=True)
            del arms


if __name__ == "__main__":
    main()
