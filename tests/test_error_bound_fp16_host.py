"""The per-element error bound of tests/util.py with fp16 output, on the CPU: an fp32 execution of the reference's own summation order,
rounded to the nearest fp16 once with the bias inside the sum, passes it on every layer shape the route tests use, and each single fault
below fails it - including an output rounded toward zero, which rel_err < REL_TOL lets through.  For the fp16 pair table (the codebook
rounded to fp16, round-to-nearest-even) the truth is the oracle on the rounded codebook, and a table rounded any other way fails."""
import numpy as np
import pytest

from test_error_bound_host import SHAPES, _layer
from util import OUT_ROUNDING, REL_TOL, abs_sum, bound_ratio, make_activations, orc, rel_err

R16, ETA16 = OUT_ROUNDING["float16"]


def fp16(a):
    """fp32 / fp64 -> the nearest fp16 (ties to even), as fp64."""
    return np.asarray(a, dtype=np.float32).astype(np.float16).astype(np.float64)


def toward_zero(a):
    """fp32 -> fp16 rounded toward zero, as fp64: the nearest fp16, moved one step back toward zero where it came out larger."""
    a = np.asarray(a, dtype=np.float32)
    h = a.astype(np.float16)
    over = np.abs(h.astype(np.float32)) > np.abs(a)
    return np.where(over, np.nextafter(h, np.float16(0)), h).astype(np.float64)


def _rows(K, seed):
    """The 1e-3 row (fp16 subnormals), the 1e2 row, a one-entry row and an ordinary one (make_activations rows 0, 1, 3, 5)."""
    return make_activations(K, 6, seed=seed)[[0, 1, 3, 5]]


@pytest.mark.parametrize("K,N,bits", SHAPES, ids=[f"w{b}_{k}x{n}" for k, n, b in SHAPES])
def test_fp32_blocked_order_rounded_to_fp16_within_bound(K, N, bits):
    L = _layer(K, N, bits, seed=K + N)
    x = _rows(K, seed=K)
    bias = L["bias"][None, :]
    want = orc.forward_f64(L, x, mul_init=bias)
    got = fp16(orc.forward_f32_blocked(L, x, mul_init=bias))
    assert np.isfinite(got).all()
    ratio = bound_ratio(got, want, abs_sum(L, x, L["bias"]), want, R16, eta=ETA16)
    print(f"forward_f32_blocked -> fp16 w{bits} {K}x{N}: max bound_ratio {ratio:.4f}")
    assert ratio <= 1.0


# ---- faults of the fp16 output --------------------------------------------------------------------------------------------------
K, N, BITS = 4096, 4096, 4


@pytest.fixture(scope="module")
def case():
    L = orc.make_layer(BITS, K, N, sparsity=0.0045, topX=10, seed=5, nonzero_full_rows=True, bias=True)
    x = _rows(K, seed=11)
    bias = L["bias"][None, :]
    want = orc.forward_f64(L, x, mul_init=bias)
    S = abs_sum(L, x, L["bias"])
    f32 = orc.forward_f32_blocked(L, x, mul_init=bias)
    assert bound_ratio(fp16(f32), want, S, want, R16, eta=ETA16) <= 1.0
    return L, x, want, S, f32


def _toward_zero(L, x, f32):
    return toward_zero(f32)


def _bias_after_rounding(L, x, f32):
    """The sum rounded to fp16 first, then the fp16 bias added and rounded again."""
    bias = L["bias"][None, :]
    return fp16(fp16(f32 - bias) + fp16(bias))


def _dense_row_dropped(L, x, f32):
    fr = L["full_rows"].copy()
    fr[:, 3] = 0.0
    return fp16(orc.forward_f32_blocked(dict(L, full_rows=fr), x, mul_init=L["bias"][None, :]))


def _subnormals_flushed(L, x, f32):
    xf = np.where(np.abs(x) < 2.0 ** -14, 0.0, x).astype(np.float32)
    assert (xf != x).sum() > 100
    return fp16(orc.forward_f32_blocked(L, xf, mul_init=L["bias"][None, :]))


FAULTS = [_toward_zero, _bias_after_rounding, _dense_row_dropped, _subnormals_flushed]
OLD_METRIC_MISSES = {_toward_zero}


@pytest.mark.parametrize("fault", FAULTS, ids=[f.__name__.strip("_") for f in FAULTS])
def test_single_fault_fails_the_fp16_bound(case, fault):
    L, x, want, S, f32 = case
    bad = fault(L, x, f32)
    assert not np.array_equal(bad, fp16(f32))
    ratio, old = bound_ratio(bad, want, S, want, R16, eta=ETA16), rel_err(bad, want)
    print(f"{fault.__name__.strip('_')}: bound_ratio {ratio:.3g}, rel_err {old:.3g}")
    assert ratio > 1.0
    if fault in OLD_METRIC_MISSES:
        assert old < REL_TOL  # what the per-vector metric with its 1 % floor lets through


# ---- the fp16 pair table's codebook ---------------------------------------------------------------------------------------------
def halfway_codebook(lut):
    """Every centroid moved to the exact midpoint of the two fp16 values around it (fp32 holds it exactly): the rounding of the
    table build decides each one, ties to even."""
    h = np.asarray(lut, dtype=np.float32).astype(np.float16)
    up = np.nextafter(h, np.float16(np.inf))
    mid = (h.astype(np.float64) + up.astype(np.float64)) / 2
    assert np.array_equal(mid.astype(np.float32).astype(np.float64), mid)
    return mid.astype(np.float32)


def ties_away(lut):
    """fp32 -> fp16 with ties rounded away from zero (fp32 numpy)."""
    lut = np.asarray(lut, dtype=np.float32)
    h = lut.astype(np.float16)
    lo = np.where(np.abs(h.astype(np.float32)) > np.abs(lut), np.nextafter(h, np.float16(0)), h)
    hi = np.nextafter(lo, np.copysign(np.float16(np.inf), lo))
    tie = np.abs(hi.astype(np.float64) - lut) == np.abs(lut - lo.astype(np.float64))
    return np.where(tie, hi, h).astype(np.float32)


@pytest.mark.parametrize("codebook", ["random", "halfway"])
def test_pair_table_codebook_rounding(codebook):
    """Against the oracle on the codebook rounded to nearest even: that table passes; the exact codebook, a table rounded toward zero
    and (halfway centroids) a table with ties away from zero fail."""
    L = orc.make_layer(BITS, K, N, sparsity=0.0045, topX=10, seed=5, nonzero_full_rows=True, bias=True)
    if codebook == "halfway":
        L["lookup_table"] = halfway_codebook(L["lookup_table"])
    x = _rows(K, seed=11)
    bias = L["bias"][None, :]
    lut = L["lookup_table"]
    L16 = dict(L, lookup_table=lut.astype(np.float16).astype(np.float32))
    want, S = orc.forward_f64(L16, x, mul_init=bias), abs_sum(L16, x, L["bias"])
    tables = {"nearest even": L16["lookup_table"], "exact": lut, "toward zero": toward_zero(lut).astype(np.float32)}
    if codebook == "halfway":
        tables["ties away"] = ties_away(lut)
    ratios = {}
    for name, t in tables.items():
        ratios[name] = bound_ratio(orc.forward_f32_blocked(dict(L, lookup_table=t), x, mul_init=bias), want, S)
        print(f"{codebook} codebook, {name} table: bound_ratio {ratios[name]:.3g}")
    assert ratios.pop("nearest even") <= 1.0
    assert all(r > 1.0 for r in ratios.values()), ratios
