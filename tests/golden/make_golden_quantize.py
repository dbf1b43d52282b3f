#!/usr/bin/env python3
"""Golden data of the reference's quantization pipeline, for tests/test_quantize_*.py.  Run once on a host that has the
reference checkout and scikit-learn (neither is needed by the tests):

    python tests/golden/make_golden_quantize.py [/path/to/reference]

Writes tests/golden/quantize_kmeans.npz, quantize_outliers.npz and quantize_iqr.npz:

  * kmeans: seeded synthetic rows at n = 4096 and 11008, and sklearn's fit of each at bits 3 and 4, made exactly as
    quantization/nuq.py:50-58,169-176 makes it: KMeans(n_clusters=2^bits, random_state=0, n_init="auto", max_iter=50) on the
    row with sample_weight = fisher * (w != 0), all ones when that sums to 0.  nuq.py itself cannot be imported under
    NumPy 2 (np.cast, nuq.py:58), so its call is restated here.  Stored: w, s = fisher * (w != 0) (before the all-ones rule),
    sklearn's centers (fp32, its order), labels and the fp64 objective sum s (w - c[label])^2.
    Rows: Student-t and Gaussian values, masked zeros, an all-zero-Fisher row, a row of 5 distinct values, magnitudes
    x1e-3 and x1e2, Fisher weights spread over 1e-12 .. 1e2.
  * outliers: dense and outlier matrices of the reference's own squeezellm/outliers.py (remove_outliers) for threshold-only,
    sensitivity-only and combined cases, including Fisher values tied at the sensitivity cut.
  * iqr: the outlier threshold of quantization/generate_outlier_config.py:47-53 evaluated by numpy on fp32 arrays.
"""
import importlib.util
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("SQLLM_REFERENCE_DIR", "/root/reference")


def kmeans_rows(n, rng):
    rows, fish = [], []
    scale = lambda: np.exp(rng.normal(0.0, 1.5, n))
    rows.append(rng.standard_t(4, n) * 0.02); fish.append((scale() * rng.standard_normal(n)) ** 2)
    w = rng.standard_normal(n) * 0.02
    w[rng.random(n) < 0.1] = 0.0  # masked zeros: sample weight 0
    rows.append(w); fish.append((scale() * rng.standard_normal(n)) ** 2)
    rows.append(rng.standard_t(3, n) * 0.02); fish.append(np.zeros(n))  # all-zero Fisher: nuq.py weights it uniformly
    rows.append(rng.choice(np.array([-0.03, -0.01, 0.0, 0.01, 0.025]), n)); fish.append(rng.random(n))  # 5 distinct values
    rows.append(rng.standard_normal(n) * 1e-3); fish.append(10.0 ** rng.uniform(-12, 2, n))
    rows.append(rng.standard_t(5, n) * 1e2); fish.append((scale() * rng.standard_normal(n)) ** 2)
    return np.array(rows, dtype=np.float32), np.array(fish, dtype=np.float32)


def sklearn_fit(w, s, k):
    from sklearn.cluster import KMeans
    s_eff = s if s.sum() != 0 else np.ones_like(s)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # fewer distinct points than clusters
        km = KMeans(n_clusters=k, random_state=0, n_init="auto", max_iter=50).fit(w.reshape(-1, 1), sample_weight=s_eff)
    c = km.cluster_centers_.reshape(-1).astype(np.float32)
    lab = km.labels_.astype(np.uint8)
    sse = float((s_eff.astype(np.float64) * (w.astype(np.float64) - c[lab].astype(np.float64)) ** 2).sum())
    return c, lab, sse


def make_kmeans():
    rng = np.random.default_rng(20261016)
    out = {}
    for n in (4096, 11008):
        w, f = kmeans_rows(n, rng)
        s = (f * (w != 0)).astype(np.float32)
        out[f"w_{n}"], out[f"s_{n}"] = w, s
        for bits in (3, 4):
            fits = [sklearn_fit(w[r], s[r], 2 ** bits) for r in range(len(w))]
            out[f"centers_{n}_{bits}"] = np.stack([c for c, _, _ in fits])
            out[f"labels_{n}_{bits}"] = np.stack([lab for _, lab, _ in fits])
            out[f"sse_{n}_{bits}"] = np.array([e for _, _, e in fits])
    np.savez_compressed(os.path.join(HERE, "quantize_kmeans.npz"), **out)


def make_outliers():
    spec = importlib.util.spec_from_file_location("ref_outliers", os.path.join(REF, "squeezellm", "outliers.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rng = np.random.default_rng(7)
    w = (rng.standard_t(3, (48, 256)) * 0.02).astype(np.float32)
    g = ((np.exp(rng.normal(0, 1.5, w.shape)) * rng.standard_normal(w.shape)) ** 2).astype(np.float32)
    g_tied = np.round(g * 4) / 4  # many Fisher values equal at the sensitivity cut
    cases = [("thr", g, 0.05, 0.0), ("sens", g, None, 0.45), ("both", g, 0.05, 0.45), ("tied", g_tied, None, 5.0),
             ("tied_both", g_tied, 0.04, 2.0)]
    out = {"w": w}
    for name, fisher, thr, sens in cases:
        model = {"layer": torch.from_numpy(w.copy())}
        grads = {"layer": torch.from_numpy(fisher.astype(np.float32))}
        res = ref.remove_outliers(model=model, sensitivity=sens, outlier_config=None if thr is None else {"layer": thr},
                                  gradients=grads)
        out[f"{name}_fisher"] = fisher.astype(np.float32)
        out[f"{name}_params"] = np.array([np.nan if thr is None else thr, sens])
        out[f"{name}_dense"] = model["layer"].numpy()
        out[f"{name}_outliers"] = res[0][0].numpy()
    np.savez_compressed(os.path.join(HERE, "quantize_outliers.npz"), **out)


def make_iqr():
    rng = np.random.default_rng(11)
    out = {}
    for i, shape in enumerate([(64, 128), (33, 97), (1, 5), (128, 1024)]):
        a = (rng.standard_t(3, shape) * 0.02).astype(np.float32)
        out[f"a{i}"] = a
        for r in (1.5, 3.0, 10.0):  # generate_outlier_config.py:47-53
            q1, q3 = np.quantile(a, 0.25), np.quantile(a, 0.75)
            lo, hi = q1 - r * (q3 - q1), q3 + r * (q3 - q1)
            out[f"thr{i}_{r}"] = np.array(max(abs(lo), abs(hi)))
    np.savez_compressed(os.path.join(HERE, "quantize_iqr.npz"), **out)


if __name__ == "__main__":
    make_kmeans()
    make_outliers()
    make_iqr()
    print("wrote quantize_kmeans.npz, quantize_outliers.npz, quantize_iqr.npz")
