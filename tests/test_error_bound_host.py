"""The per-element error bound of tests/util.py (bound_ratio) on the CPU: an fp32 execution of the reference's own summation order
passes it on every layer shape the route tests use, and each single fault below fails it on at least one element - including the
two that rel_err < TIGHT_TOL misses, because its floor is 1 % of the largest output of the whole array."""
import numpy as np
import pytest

from util import TIGHT_TOL, abs_sum, bound_ratio, make_activations, massive_channels, orc, rel_err

# the route tests' layers (tests/test_routes_gpu.py): K x N, bits
SHAPES = [(4096, 12288, 4), (4096, 4096, 3), (4096, 22016, 4), (11008, 4096, 3), (5120, 13824, 3), (13824, 5120, 4),
          (8192, 2752, 3), (22016, 1024, 4), (512, 132, 3), (512, 132, 4)]


def _layer(K, N, bits, seed):
    return orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=seed, nonzero_full_rows=True, bias=True)


@pytest.mark.parametrize("K,N,bits", SHAPES, ids=[f"w{b}_{k}x{n}" for k, n, b in SHAPES])
def test_fp32_blocked_order_within_bound(K, N, bits):
    """One legal fp32 execution of the reference kernels (128-input blocks, atomics onto the bias) is within the bound."""
    L = _layer(K, N, bits, seed=K + N)
    x = make_activations(K, 6, seed=K)
    want = orc.forward_f64(L, x, mul_init=L["bias"][None, :])
    got = orc.forward_f32_blocked(L, x, mul_init=L["bias"][None, :])
    ratio = bound_ratio(got, want, abs_sum(L, x, L["bias"]))
    print(f"forward_f32_blocked w{bits} {K}x{N}: max bound_ratio {ratio:.4f}")
    assert ratio <= 1.0
    assert np.array_equal(got[2], L["bias"])  # the all-zero row: exactly the bias


# ---- mutations ----------------------------------------------------------------------------------------------------------------
K, N, BITS, M = 4096, 1024, 4, 12


@pytest.fixture(scope="module")
def case():
    L = _layer(K, N, BITS, seed=77)
    x = make_activations(K, M, seed=77)
    typical = np.median(np.abs(x), axis=1)
    assert typical[0] < 1e-3 and typical[1] > 50  # rows span 1e-3 .. 1e2
    bias = L["bias"][None, :]
    want = orc.forward_f64(L, x, mul_init=bias)
    S = abs_sum(L, x, L["bias"])
    good = orc.forward_f32_blocked(L, x, mul_init=bias)
    assert bound_ratio(good, want, S) <= 1.0
    return L, x, want, S, good


def _blocked(L, x):
    return orc.forward_f32_blocked(L, x, mul_init=L["bias"][None, :])


def _neighbour_centroid(L, x, good):
    idx = orc.unpack(L["qweight"], BITS)
    b = 1
    k = int(np.nonzero(np.abs(x[b]) >= 1.0)[0][0])
    c = 17
    idx[k, c] = idx[k, c] + 1 if idx[k, c] < 2 ** BITS - 1 else idx[k, c] - 1
    return _blocked(dict(L, qweight=orc.pack(idx, BITS)), x)


def _csr_dropped(L, x, good):
    # the entry on the first massive channel (a large x), else the largest value
    hit = np.nonzero(np.isin(L["cols"], massive_channels(K)))[0]
    i = int(hit[0]) if hit.size else int(np.abs(L["vals"]).argmax())
    c = int(np.searchsorted(L["rows"], i, side="right") - 1)
    rows = L["rows"].copy()
    rows[c + 1:] -= 1
    return _blocked(dict(L, rows=rows, cols=np.delete(L["cols"], i), vals=np.delete(L["vals"], i)), x)


def _dense_row_twice(L, x, good):
    j = 3
    fr = np.ascontiguousarray(np.concatenate([L["full_rows"], L["full_rows"][:, j:j + 1]], axis=1))
    fri = np.concatenate([L["full_row_indices"], L["full_row_indices"][j:j + 1]]).astype(np.int32)
    return _blocked(dict(L, full_rows=fr, full_row_indices=fri), x)


def _last_row_copies_previous(L, x, good):
    bad = good.copy()
    bad[M - 1] = good[M - 2]
    return bad


def _lo_part_missing(L, x, good):
    """Column c computed from the hi half of the tensor-core path's hi/lo split only (DESIGN.md 3.6: s_c = 2^(e-15) with 2^e above
    max|lut_c| + the CSR values of row c + the dense-row maxima of column c; hi = fp16(w / s_c))."""
    c = 40
    w = orc.dequant_f32(L["qweight"], L["lookup_table"], BITS)[:, c].astype(np.float64)
    e0, e1 = L["rows"][c], L["rows"][c + 1]
    w[L["cols"][e0:e1]] += L["vals"][e0:e1]
    dense = np.nonzero(L["full_row_indices"] == c)[0]
    w += L["full_rows"][:, dense].sum(axis=1)
    bound = np.abs(L["lookup_table"][c]).max() + np.abs(L["vals"][e0:e1]).sum() + np.abs(L["full_rows"][:, dense]).max(axis=0).sum()
    s = 2.0 ** (np.floor(np.log2(bound)) + 1 - 15)
    hi = (w / s).astype(np.float16).astype(np.float64) * s
    bad = good.copy()
    bad[:, c] -= (x.astype(np.float64) @ (w - hi)).astype(np.float32)
    return bad


def _bias_twice(L, x, good):
    return good + L["bias"][None, :]


def _small_row_2_percent_off(L, x, good):
    bad = good.copy()
    bad[0] += 0.02 * (good[0] - L["bias"])  # row 0 is the 1e-3 row; its x.W part 2 % off
    return bad


def _subnormals_flushed(L, x, good):
    xf = np.where(np.abs(x) < 2.0 ** -14, 0.0, x).astype(np.float32)
    assert (xf != x).sum() > 100
    return _blocked(L, xf)


MUTATIONS = [_neighbour_centroid, _csr_dropped, _dense_row_twice, _last_row_copies_previous, _lo_part_missing, _bias_twice,
             _small_row_2_percent_off, _subnormals_flushed]
OLD_METRIC_MISSES = {_small_row_2_percent_off, _subnormals_flushed}


@pytest.mark.parametrize("mutate", MUTATIONS, ids=[f.__name__.strip("_") for f in MUTATIONS])
def test_single_fault_fails_the_bound(case, mutate):
    L, x, want, S, good = case
    bad = mutate(L, x, good)
    assert not np.array_equal(bad, good)
    ratio, old = bound_ratio(bad, want, S), rel_err(bad, want)
    print(f"{mutate.__name__.strip('_')}: bound_ratio {ratio:.3g}, rel_err {old:.3g}")
    assert ratio > 1.0
    if mutate in OLD_METRIC_MISSES:
        assert old < TIGHT_TOL  # what the old metric lets through
