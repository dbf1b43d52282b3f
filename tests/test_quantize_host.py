"""CPU tests of the quantizer's checkers and host logic: the exact weighted 1-D k-means oracle against brute force and against
the reference's sklearn fits, and split_outliers / outlier_threshold against the reference's own outliers.py and
generate_outlier_config.py formula (tests/golden/make_golden_quantize.py)."""
import itertools
import os

import numpy as np
import pytest
import torch

import kmeans_oracle as kmo
from util import GOLDEN


def brute_dp(w, s, k):
    """O(k n^2) DP over the sorted row in fp64: the optimum of sum s (w - c)^2 with k clusters."""
    s = s if s.sum() > 0 else np.ones_like(s)
    o = np.argsort(w, kind="stable")
    w, s = w[o].astype(np.float64), s[o].astype(np.float64)
    n = len(w)

    def cost(i, j):
        W = s[i:j].sum()
        return 0.0 if W == 0 else float((s[i:j] * (w[i:j] - (s[i:j] * w[i:j]).sum() / W) ** 2).sum())

    C = np.array([[cost(i, j) if i < j else 0.0 for j in range(n + 1)] for i in range(n + 1)])
    D = C[0].copy()
    for m in range(2, k + 1):
        D = np.array([min(D[i] + C[i, j] for i in range(m - 1, j)) if j >= m else np.inf for j in range(n + 1)])
    return D[n]


def spread(w, s):
    """sum s (w - mu)^2: the scale of the absolute rounding error of the centred prefix sums."""
    w, s = np.asarray(w, np.float64), np.asarray(s, np.float64)
    s = s if s.sum() > 0 else np.ones_like(s)
    return float((s * (w - (s * w).sum() / s.sum()) ** 2).sum())


def rows(rng, n, kind):
    if kind == "gauss":
        return rng.standard_normal(n).astype(np.float32), rng.random(n).astype(np.float32)
    if kind == "dup":
        return rng.choice(np.array([-1.0, -0.5, 0.0, 0.5, 1.0], np.float32), n), (rng.random(n) < 0.7).astype(np.float32)
    if kind == "zeros":
        return (rng.standard_t(3, n) * 0.02).astype(np.float32), np.zeros(n, np.float32)
    return (rng.standard_t(3, n) * 1e-3).astype(np.float32), (10.0 ** rng.uniform(-12, 2, n)).astype(np.float32)


@pytest.mark.parametrize("n,k", [(40, 3), (96, 8), (200, 16), (512, 4)])
@pytest.mark.parametrize("kind", ["gauss", "dup", "zeros", "wide"])
def test_oracle_equals_brute_force_dp(n, k, kind):
    w, s = rows(np.random.default_rng(n * 31 + k), n, kind)
    if n > 200 and kind != "gauss":
        pytest.skip("one large case is enough for the O(k n^2) brute force")
    opt, cent, lab = kmo.kmeans1d(w, s, k)
    want = brute_dp(w, s, k)
    tol = 1e-9 * want + 1e-12 * spread(w, s)
    assert abs(opt[0] - want) <= tol, (opt[0], want)
    got = kmo.kmeans_objective(w, s, cent, lab)[0]
    assert abs(got - want) <= tol
    assert np.all(np.diff(cent[0]) >= 0)


@pytest.mark.parametrize("n", [2, 5, 8])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_oracle_equals_exhaustive_labelings(n, k):
    """Every assignment of n points to k clusters (not only contiguous ones), each cluster at its weighted mean."""
    if k > n:
        pytest.skip("k > n")
    rng = np.random.default_rng(100 * n + k)
    w = rng.standard_normal(n).astype(np.float32)
    s = rng.random(n).astype(np.float32) + 0.01
    best = np.inf
    for lab in itertools.product(range(k), repeat=n):
        lab = np.array(lab)
        tot = 0.0
        for c in range(k):
            m = lab == c
            if m.any():
                mu = (s[m].astype(np.float64) * w[m]).sum() / s[m].sum()
                tot += (s[m] * (w[m].astype(np.float64) - mu) ** 2).sum()
        best = min(best, tot)
    assert abs(kmo.kmeans1d(w, s, k)[0][0] - best) <= 1e-9 * best + 1e-12 * spread(w, s)


@pytest.mark.parametrize("n", [9, 12])
@pytest.mark.parametrize("k", [2, 4])
def test_oracle_equals_exhaustive_contiguous_partitions(n, k):
    rng = np.random.default_rng(7 * n + k)
    w = rng.standard_normal(n).astype(np.float32)
    s = (rng.random(n) * (rng.random(n) < 0.8)).astype(np.float32)
    o = np.argsort(w, kind="stable")
    ws, ss = w[o].astype(np.float64), s[o].astype(np.float64)

    def seg(i, j):
        W = ss[i:j].sum()
        return 0.0 if W == 0 else (ss[i:j] * (ws[i:j] - (ss[i:j] * ws[i:j]).sum() / W) ** 2).sum()

    best = min(sum(seg(a, b) for a, b in zip((0,) + cuts, cuts + (n,))) for cuts in itertools.combinations(range(1, n), k - 1))
    assert abs(kmo.kmeans1d(w, s, k)[0][0] - best) <= 1e-9 * best + 1e-12 * spread(w, s)


def test_oracle_is_never_worse_than_sklearn_on_the_golden_rows():
    g = np.load(os.path.join(GOLDEN, "quantize_kmeans.npz"))
    for n in (4096, 11008):
        w, s = g[f"w_{n}"], g[f"s_{n}"]
        for bits in (3, 4):
            opt, cent, lab = kmo.kmeans1d(w, s, 2 ** bits)
            sse = g[f"sse_{n}_{bits}"]
            tol = np.array([1e-12 * spread(w[r], s[r]) for r in range(len(w))])
            assert np.all(opt <= sse * (1 + 1e-9) + tol), (n, bits, opt / np.maximum(sse, 1e-300))
            sk = kmo.kmeans_objective(w, s, g[f"centers_{n}_{bits}"], g[f"labels_{n}_{bits}"])
            np.testing.assert_allclose(sk, sse, rtol=1e-12)


# ---- outliers (run on CPU tensors: the functions are plain torch) -------------------------------------------------------
from squeezellm_b200.quantize import outlier_threshold, split_outliers  # noqa: E402


@pytest.mark.parametrize("case", ["thr", "sens", "both", "tied", "tied_both"])
def test_split_outliers_matches_the_reference_masks(case):
    g = np.load(os.path.join(GOLDEN, "quantize_outliers.npz"))
    thr, sens = g[f"{case}_params"]
    dense, outl = split_outliers(torch.from_numpy(g["w"]), torch.from_numpy(g[f"{case}_fisher"]),
                                 threshold=None if np.isnan(thr) else float(thr), sensitivity=float(sens))
    assert np.array_equal(dense.numpy(), g[f"{case}_dense"])
    assert np.array_equal(outl.numpy(), g[f"{case}_outliers"])
    assert np.array_equal(dense.numpy() != 0, g[f"{case}_dense"] != 0)


def test_split_outliers_count_zero_takes_none():
    w = torch.randn(4, 64)
    dense, outl = split_outliers(w, torch.rand(4, 64), sensitivity=0.1)  # int(256 * 0.1 / 100) = 0
    assert torch.equal(dense, w) and not outl.any()


def test_outlier_threshold_matches_numpy():
    g = np.load(os.path.join(GOLDEN, "quantize_iqr.npz"))
    for i in range(4):
        for r in (1.5, 3.0, 10.0):
            assert outlier_threshold(torch.from_numpy(g[f"a{i}"]), r) == float(g[f"thr{i}_{r}"])
