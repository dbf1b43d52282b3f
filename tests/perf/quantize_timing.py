#!/usr/bin/env python3
"""Quantizer timing on one GPU: the exact weighted k-means (quant_cuda.kmeans1d) on whole LLaMA-7B weight matrices, against the
CPU pipeline it replaces (one sklearn KMeans per row, reference quantization/nuq.py:50-58, one thread as nuq.py runs it).

  * GPU: CUDA events around one whole-matrix call, after a warm-up call on the same shape; 4096-wide rows x {4096 (q/k/v/o),
    12288 (q/k/v stacked), 22016 (gate/up stacked)} and 11008-wide rows x 4096 (down), bits 3 and 4.  Synthetic rows: Student-t
    weights, squared log-normal-scaled Gaussian Fisher weights.  -> ms, rows/s, and the projected k-means time of a 7B, 13B and
    65B model (each layer's rows at the per-row time measured at the nearest width, scaled by n log2 n).
  * CPU: sklearn KMeans(n_clusters, random_state=0, n_init="auto", max_iter=50) on 64 of those rows with one thread -> ms per
    row, and the median ratio of the GPU's objective to sklearn's on the same rows (<= 1: the GPU result is the optimum).
The first line names the card and its power limit (nvidia-smi, read-only query).  Output: JSON lines on stdout, also written
to FILE with --out FILE.

    python tests/perf/quantize_timing.py [--quick] [--out FILE]
"""
import json
import math
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402

SHAPES = [(4096, 4096), (12288, 4096), (22016, 4096), (4096, 11008)]  # (rows, n)
MODELS = {  # (hidden, intermediate, layers): rows x width of every quantized matrix per layer
    "7B": (4096, 11008, 32), "13B": (5120, 13824, 40), "65B": (8192, 22016, 80)}


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    out.append(line)


def rows_of(R, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.distributions.StudentT(4.0).sample((R, n)).cuda() * 0.02
    s = (torch.exp(torch.randn(R, n, device="cuda", generator=g) * 1.5) * torch.randn(R, n, device="cuda", generator=g)) ** 2
    return w.float().contiguous(), s.float().contiguous()


def objective(w, s, c, lab):
    w, s = w.double(), s.double()
    return (s * (w - c.double().gather(1, lab.long())) ** 2).sum(1)


def main():
    quick = "--quick" in sys.argv
    out = []
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    emit({"card": card[torch.cuda.current_device()] if card else torch.cuda.get_device_name()}, out)
    per_row = {}
    for bits in (3, 4):
        k = 2 ** bits
        for R, n in SHAPES:
            if quick:
                R = 256
            w, s = rows_of(R, n, seed=R + n)
            qc.kmeans1d(w[:64].contiguous(), s[:64].contiguous(), k)  # warm-up: module load, sort kernels
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            c, lab = qc.kmeans1d(w, s, k)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            per_row.setdefault(bits, {})[n] = ms / R  # the last (largest) matrix of each width
            emit({"bits": bits, "rows": R, "n": n, "ms": round(ms, 2), "rows_per_s": round(R / ms * 1e3, 1),
                  "cost_evals_per_s": round(k * n * math.log2(n) * R / ms * 1e3 / 1e9, 2)}, out)
            del w, s, c, lab
        for name, (h, inter, layers) in MODELS.items():
            total = 0.0
            for R, n in [(h, h)] * 4 + [(inter, h)] * 2 + [(h, inter)]:
                ref = 4096 if n <= 8192 else 11008
                total += R * per_row[bits][ref] * (n * math.log2(n)) / (ref * math.log2(ref))
            emit({"bits": bits, "model": name, "projected_kmeans_s": round(total * layers / 1e3, 1)}, out)

    # sklearn on 64 rows per width, one thread, and the objective ratio on the same rows
    from sklearn.cluster import KMeans
    from threadpoolctl import threadpool_limits
    for bits in (3, 4):
        k = 2 ** bits
        for n in (4096, 11008):
            w, s = rows_of(64, n, seed=7 * n + bits)
            c, lab = qc.kmeans1d(w, s, k)
            ours = objective(w, s, c, lab).cpu().numpy()
            wn, sn = w.cpu().numpy(), s.cpu().numpy()
            sk = []
            t0 = time.perf_counter()
            with threadpool_limits(1), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                for r in range(wn.shape[0] if not quick else 8):
                    km = KMeans(n_clusters=k, random_state=0, n_init="auto", max_iter=50).fit(wn[r].reshape(-1, 1), sample_weight=sn[r])
                    cc = km.cluster_centers_.reshape(-1).astype(np.float32)
                    sk.append(float((sn[r].astype(np.float64) * (wn[r].astype(np.float64) - cc[km.labels_]) ** 2).sum()))
            dt = (time.perf_counter() - t0) / len(sk)
            ratio = ours[:len(sk)] / np.array(sk)
            emit({"bits": bits, "n": n, "sklearn_ms_per_row_1thread": round(dt * 1e3, 2),
                  "gpu_over_sklearn_objective_median": round(float(np.median(ratio)), 5),
                  "min": round(float(ratio.min()), 5), "max": round(float(ratio.max()), 5)}, out)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write("\n".join(out) + "\n")


if __name__ == "__main__":
    main()
