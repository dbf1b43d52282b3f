"""The fp64 input-gradient truth (tests/backward_ref.py) on the CPU: against an element-by-element restatement of the semantics,
and against the C forward oracle through the adjoint identity <dy, x W> = <dy W^T, x>, on small shapes with duplicate and
out-of-range outlier indices."""
import numpy as np
import pytest

from backward_ref import backward_abs_sum, backward_f64, dense_w_f64
from util import orc


def _layer(bits, K, N, seed, dup=True, oor=True):
    L = orc.make_layer(bits, K, N, sparsity=0.05, topX=5, seed=seed, nonzero_full_rows=True)
    if dup:  # dense rows on one channel twice, and on channel 0
        L["full_row_indices"][1] = L["full_row_indices"][0]
        L["full_row_indices"][2] = 0
    if oor:  # out-of-range channels / columns: ignored
        L["full_row_indices"][3] = N + 2
        L["full_row_indices"][4] = -1
        L["cols"] = L["cols"].copy()
        L["cols"][0] = K + 5
        L["cols"][-1] = -3
    if dup:  # two CSR entries of one row on the same column: they add up
        rows = L["rows"]
        c = int(np.argmax(np.diff(rows)))
        assert rows[c + 1] - rows[c] >= 2
        L["cols"][rows[c] + 1] = L["cols"][rows[c]]
    return L


def _loop_truth(L, dy):
    """dx from the definition, one element at a time, in Python floats (fp64)."""
    K, N, bits = L["infeatures"], L["outfeatures"], L["bits"]
    idx = orc.unpack_np(L["qweight"], bits)
    lut, rows, cols, vals = L["lookup_table"], L["rows"], L["cols"], L["vals"]
    fr, fri = L["full_rows"], L["full_row_indices"]
    W = [[float(lut[c][idx[k][c]]) for c in range(N)] for k in range(K)]
    for c in range(N):
        for e in range(rows[c], rows[c + 1]):
            if 0 <= cols[e] < K:
                W[cols[e]][c] += float(vals[e])
    for j in range(len(fri)):
        if 0 <= fri[j] < N:
            for k in range(K):
                W[k][fri[j]] += float(fr[k][j])
    M = dy.shape[0]
    return np.array([[sum(float(dy[m][c]) * W[k][c] for c in range(N)) for k in range(K)] for m in range(M)])


@pytest.mark.parametrize("bits", [3, 4])
def test_matches_elementwise_definition(bits):
    L = _layer(bits, 64, 12, seed=bits)
    dy = np.random.default_rng(1).standard_normal((3, 12)).astype(np.float32)
    got = backward_f64(L, dy)
    want = _loop_truth(L, dy)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("bits", [3, 4])
def test_adjoint_of_the_forward_oracle(bits):
    """<dy, forward(x)> == <backward(dy), x> with the C forward oracle (valid indices only: it does not filter)."""
    K, N = 256, 72
    L = _layer(bits, K, N, seed=10 + bits, oor=False)
    rng = np.random.default_rng(2)
    x = rng.standard_normal((4, K)).astype(np.float32)
    dy = rng.standard_normal((4, N)).astype(np.float32)
    lhs = float((dy.astype(np.float64) * orc.forward_f64(L, x)).sum())
    rhs = float((backward_f64(L, dy) * x.astype(np.float64)).sum())
    assert abs(lhs - rhs) <= 1e-10 * max(1.0, abs(lhs))


def test_column_blocks_and_abs_sum():
    """Column-blocked product equals the one-block product; the condition S bounds |dx| and is the product of absolute values."""
    import backward_ref
    L = _layer(4, 128, 300, seed=5)
    dy = np.random.default_rng(3).standard_normal((5, 300))
    old = backward_ref.COL_BLOCK
    try:
        backward_ref.COL_BLOCK = 64
        blocked = backward_f64(L, dy)
    finally:
        backward_ref.COL_BLOCK = old
    whole = dy @ dense_w_f64(L).T
    np.testing.assert_allclose(blocked, whole, rtol=1e-12, atol=1e-13)
    S = backward_abs_sum(L, dy)
    assert (S >= np.abs(whole) - 1e-12).all()
    W = dense_w_f64(L)
    assert (np.abs(W) <= dense_w_f64(dict(L, lookup_table=np.abs(L["lookup_table"]), vals=np.abs(L["vals"]),
                                          full_rows=np.abs(L["full_rows"]))) + 1e-15).all()
