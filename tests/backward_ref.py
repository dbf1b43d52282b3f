"""fp64 truth of the input gradient dx = dy . W^T of a QuantLinearLUT layer (test infrastructure).

    dx[m][k] = sum_c dy[m][c] W[k][c],   W[k][c] = LUT[c][idx(k,c)] + CSR(c,k) + sum_j full_rows[k][j] [fri[j] == c]

W is built as a dense fp64 matrix from the C oracle's exact dequantisation (oracle.dequant_f32) plus the CSR entries and the dense
rows, with the kernels' rules: entries on the same (k, c) add up, CSR columns outside [0, K) and dense-row channels outside
[0, N) are ignored.  The product runs in fp64 (BLAS): its rounding, at most about N 2^-53 of sum_c |dy| |w|, is far below the
2^-20 the GPU bound allows.  Wide layers are done in column blocks so that no more than a few hundred MB are alive at once.
"""
import numpy as np

from util import abs_layer, orc

COL_BLOCK = 2048


def dense_w_f64(L, c0=0, c1=None):
    """W[:, c0:c1] in fp64 (the outlier terms included)."""
    K, N, bits = L["infeatures"], L["outfeatures"], L["bits"]
    c1 = N if c1 is None else c1
    W = orc.dequant_f32(np.ascontiguousarray(L["qweight"][:, c0:c1]), np.ascontiguousarray(L["lookup_table"][c0:c1]),
                        bits).astype(np.float64)
    if L.get("rows") is not None:
        rows = np.asarray(L["rows"], dtype=np.int64)
        e0, e1 = int(rows[c0]), int(rows[c1])
        ch = np.repeat(np.arange(c0, c1), np.diff(rows[c0:c1 + 1]))
        k = np.asarray(L["cols"][e0:e1], dtype=np.int64)
        ok = (k >= 0) & (k < K)
        np.add.at(W, (k[ok], ch[ok] - c0), np.asarray(L["vals"][e0:e1], dtype=np.float64)[ok])
    if L.get("full_rows") is not None:
        fri = np.asarray(L["full_row_indices"], dtype=np.int64)
        for j in np.nonzero((fri >= c0) & (fri < c1))[0]:
            W[:, fri[j] - c0] += L["full_rows"][:, j].astype(np.float64)
    return W


def backward_f64(L, dy):
    """dx [M, K] in fp64 for dy [M, N]."""
    dy = np.asarray(dy, dtype=np.float64).reshape(-1, L["outfeatures"])
    dx = np.zeros((dy.shape[0], L["infeatures"]), dtype=np.float64)
    for c0 in range(0, L["outfeatures"], COL_BLOCK):
        c1 = min(L["outfeatures"], c0 + COL_BLOCK)
        dx += dy[:, c0:c1] @ dense_w_f64(L, c0, c1).T
    return dx


def backward_abs_sum(L, dy):
    """S [M, K] = sum_c |dy| |w| (|lut + csr + dense| <= |lut| + |csr| + |dense|): the condition of every dx element."""
    return backward_f64(abs_layer(L), np.abs(np.asarray(dy, dtype=np.float64)))


def backward_and_abs_sum(L, dy):
    """(backward_f64(L, dy), backward_abs_sum(L, dy)) with one pass over the column blocks."""
    dy = np.asarray(dy, dtype=np.float64).reshape(-1, L["outfeatures"])
    A = abs_layer(L)
    dx = np.zeros((dy.shape[0], L["infeatures"]), dtype=np.float64)
    S = np.zeros_like(dx)
    ady = np.abs(dy)
    for c0 in range(0, L["outfeatures"], COL_BLOCK):
        c1 = min(L["outfeatures"], c0 + COL_BLOCK)
        dx += dy[:, c0:c1] @ dense_w_f64(L, c0, c1).T
        S += ady[:, c0:c1] @ dense_w_f64(A, c0, c1).T
    return dx, S
