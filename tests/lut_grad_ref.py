"""fp64 truth of the codebook, CSR-value and dense-row gradients of a QuantLinearLUT layer (test infrastructure).

    G[k][c]          = sum_m x[m][k] dy[m][c]
    dlut[c][v]       = sum_{k : idx(k,c) = v} G[k][c]
    dvals[e]         = G[cols[e]][c]  for e in CSR row c with 0 <= cols[e] < K, else 0
    dfull_rows[k][j] = G[k][fri[j]]   if 0 <= fri[j] < N, else 0

G is an fp64 product, bucketed by the indices oracle.unpack_np decodes.  The condition S of every output is the same bucketing
applied to |x|^T |dy|: |dlut[c][v]| <= S_lut[c][v], and the GPU kernels' error is bounded by e * S (tests/util.py, bound_ratio).
The arithmetic is torch fp64 on `device` (the GPU tests run it on the GPU: fp64 products of 2048 rows of a 4096 x 22016 layer
take milliseconds there, minutes in numpy); its rounding, at most about (M + K) 2^-53 of S, is far below the 2^-20 the bound
allows.  Wide layers are done in column blocks so that no more than a few hundred MB are alive at once.

dense_w_torch restates the forward's weight W(LUT, vals, full_rows) with differentiable torch operations: torch's autograd through
it (fp64) is the independent statement of the gradient that the truth is checked against.
"""
import numpy as np
import torch

from util import orc

COL_BLOCK = 2048


def lut_grad_f64(L, x, dy, device="cpu"):
    """({"lookup_table", "vals", "full_rows"} -> fp64 gradient, same keys -> its condition S), numpy, for x [M, K] and dy [M, N]
    (numpy or torch; the exact values the kernels see); a key is absent when the layer has no such tensor."""
    K, N, bits = L["infeatures"], L["outfeatures"], L["bits"]
    nv = 1 << bits
    f64 = dict(dtype=torch.float64, device=device)
    x = torch.as_tensor(x).to(**f64).reshape(-1, K)
    dy = torch.as_tensor(dy).to(**f64).reshape(-1, N)
    ax, ady = x.abs(), dy.abs()
    g = {"lookup_table": torch.zeros((N, nv), **f64)}
    s = {"lookup_table": torch.zeros((N, nv), **f64)}
    has_csr = L.get("rows") is not None
    if has_csr:
        rows = np.asarray(L["rows"], dtype=np.int64)
        cols = np.asarray(L["cols"], dtype=np.int64)
        g["vals"], s["vals"] = torch.zeros(len(cols), **f64), torch.zeros(len(cols), **f64)
    has_full = L.get("full_rows") is not None
    if has_full:
        fri = np.asarray(L["full_row_indices"], dtype=np.int64)
        g["full_rows"], s["full_rows"] = torch.zeros((K, len(fri)), **f64), torch.zeros((K, len(fri)), **f64)
    for c0 in range(0, N, COL_BLOCK):
        c1 = min(N, c0 + COL_BLOCK)
        G = x.t() @ dy[:, c0:c1]
        A = ax.t() @ ady[:, c0:c1]
        idx = torch.from_numpy(orc.unpack_np(np.ascontiguousarray(L["qweight"][:, c0:c1]), bits).astype(np.int64)).to(device)
        key = (torch.arange(c1 - c0, device=device)[None, :] * nv + idx).reshape(-1)
        g["lookup_table"][c0:c1] = torch.zeros((c1 - c0) * nv, **f64).scatter_add_(0, key, G.reshape(-1)).reshape(-1, nv)
        s["lookup_table"][c0:c1] = torch.zeros((c1 - c0) * nv, **f64).scatter_add_(0, key, A.reshape(-1)).reshape(-1, nv)
        if has_csr:
            e0, e1 = int(rows[c0]), int(rows[c1])
            ch = np.repeat(np.arange(c0, c1), np.diff(rows[c0:c1 + 1]))
            k = cols[e0:e1]
            ok = (k >= 0) & (k < K)
            e = torch.from_numpy(np.arange(e0, e1)[ok]).to(device)
            kk, cc = torch.from_numpy(k[ok]).to(device), torch.from_numpy(ch[ok] - c0).to(device)
            g["vals"][e] = G[kk, cc]
            s["vals"][e] = A[kk, cc]
        if has_full:
            for j in np.nonzero((fri >= c0) & (fri < c1))[0]:
                g["full_rows"][:, j] = G[:, fri[j] - c0]
                s["full_rows"][:, j] = A[:, fri[j] - c0]
    return ({k: v.cpu().numpy() for k, v in g.items()}, {k: v.cpu().numpy() for k, v in s.items()})


def dense_w_torch(L, lut, vals=None, full_rows=None):
    """W [K, N] = LUT[c][idx(k,c)] + CSR entries + dense rows from the torch tensors lut [N, 2^bits], vals [nnz], full_rows [K, topX]
    (any dtype and device; differentiable in all three), with the kernels' rules: entries on one (k, c) add up, CSR columns
    outside [0, K) and dense-row channels outside [0, N) are ignored."""
    K, N, bits = L["infeatures"], L["outfeatures"], L["bits"]
    dev = lut.device
    idx = torch.from_numpy(orc.unpack_np(L["qweight"], bits).astype(np.int64)).to(dev)
    W = torch.gather(lut, 1, idx.t().contiguous()).t()
    if vals is not None:
        rows = torch.from_numpy(np.asarray(L["rows"], dtype=np.int64)).to(dev)
        cols = torch.from_numpy(np.asarray(L["cols"], dtype=np.int64)).to(dev)
        ch = torch.repeat_interleave(torch.arange(N, device=dev), rows[1:] - rows[:-1])
        ok = (cols >= 0) & (cols < K)
        W = W.index_put((cols[ok], ch[ok]), vals[ok], accumulate=True)
    if full_rows is not None:
        fri = torch.from_numpy(np.asarray(L["full_row_indices"], dtype=np.int64)).to(dev)
        ok = (fri >= 0) & (fri < N)
        W = W.index_add(1, fri[ok], full_rows[:, ok])
    return W
