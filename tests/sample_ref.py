"""The contract of sqllm_sample (include/sqllm_b200.h) in numpy: Philox4x32-10, the Gumbel noise of a row at a position, and a row's
kept set (temperature, then top-k, then top-p) with the mass above each token in fp64.

`philox` is pinned to the Random123 known-answer vectors (test_sample_host.py).  `row(x, t, k, p)` gives what the kernel's draw is
checked against: z in fp32 as the kernel computes it, the top-k mask (exact: it compares fp32 values), and M_i, the fp64 softmax mass
of the top-k tokens whose z is strictly above z_i; a token survives top-p iff M_i < top_p.  `scores(z, V, pos, seed)` gives the fp64
z_i + g_i of the draw, with u_i exact and g_i = -log(-log(u_i)) in fp64."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
LO = np.uint64(0xFFFFFFFF)


def philox(ctr, key):
    """Philox4x32-10 of counters ctr uint32 [..., 4] under keys key uint32 [..., 2] (broadcast): uint32 [..., 4]."""
    ctr, key = np.asarray(ctr, dtype=np.uint64), np.asarray(key, dtype=np.uint64)
    c = [ctr[..., j] for j in range(4)]
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & LO, (k1 + W1) & LO
        p0, p1 = M0 * c[0], M1 * c[2]  # < 2^64: exact
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & LO, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & LO]
    return np.stack(np.broadcast_arrays(*c), -1).astype(np.uint32)


def words(V, pos, seed):
    """The Philox word of token i < V at position(s) pos (an int or an int array [P]): uint32 [V] or [P, V]."""
    seed = int(seed)
    pos = np.asarray(pos, dtype=np.int64)
    Q = (V + 3) // 4
    ctr = np.zeros(pos.shape + (Q, 4), dtype=np.uint64)
    ctr[..., 0] = np.arange(Q, dtype=np.uint64)
    ctr[..., 1] = (pos.astype(np.uint64) & LO)[..., None]
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64)
    return philox(ctr, key).reshape(pos.shape + (4 * Q,))[..., :V]


def uniform(w):
    """u = ((w >> 9) + 1/2) 2^-23: exact in fp32 (and fp64), in (0, 1)."""
    return ((w >> 9).astype(np.float64) + 0.5) * 2.0 ** -23


def gumbel(V, pos, seed):
    """fp64 g_i = -log(-log(u_i)) of the row's tokens at position(s) pos."""
    return -np.log(-np.log(uniform(words(V, pos, seed))))


def greedy(x, t):
    """True when the row takes the greedy rule: t <= 0 or NaN, a NaN logit, or a z maximum that is not finite."""
    x = np.asarray(x, dtype=np.float32)
    t = np.float32(t)
    if not t > 0 or np.isnan(x).any():
        return True
    with np.errstate(over="ignore"):
        return not np.isfinite(x.max() / t)


def zvals(x, t):
    with np.errstate(over="ignore", divide="ignore"):
        return np.asarray(x, dtype=np.float32) / np.float32(t)


def row(x, t, top_k, top_p):
    """(z fp32 [V], top-k mask [V], M fp64 [V]) of a row that does not take the greedy rule.  M_i: the softmax mass (over the top-k
    tokens) of the top-k tokens with z strictly above z_i, np.inf for tokens top-k drops."""
    z = zvals(x, t)
    V = z.size
    z64 = z.astype(np.float64)
    topk = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(z)[::-1][top_k - 1]
        topk = z >= kth
    zmax = z64.max()
    m = np.where(topk, np.exp(z64 - zmax), 0.0)
    m /= m.sum()
    order = np.argsort(-z64, kind="stable")
    zs, ms = z64[order], m[order]
    before = np.concatenate([[0.0], np.cumsum(ms)[:-1]])
    first = np.searchsorted(-zs, -zs, side="left")  # first position of each value's tie group
    M = np.empty(V)
    M[order] = before[first]
    M[~topk] = np.inf
    return z, topk, M


def kept(M, z, top_p, slack=0.0):
    """The kept set of a row from row()'s M, with the top-p boundary moved by `slack` (of mass): top_p <= 0 keeps the maximum alone,
    top_p >= 1 or NaN keeps every top-k token."""
    if not top_p < 1:
        return np.isfinite(M)
    if top_p <= 0:
        return np.isfinite(M) & (z == z.max())
    return M < top_p + slack


def scores(z, pos, seed):
    """fp64 z_i + g_i of the draw at position pos."""
    return z.astype(np.float64) + gumbel(z.size, pos, seed)


def draw(x, t, top_k, top_p, pos, seed):
    """The contract's token in exact arithmetic: the kept token of largest fp64 score (greedy rows: np.argmax, first of ties)."""
    x = np.asarray(x, dtype=np.float32)
    if greedy(x, t):
        return int(np.argmax(x))
    z, _, M = row(x, t, top_k, top_p)
    s = np.where(kept(M, z, top_p), scores(z, pos, seed), -np.inf)
    return int(np.argmax(s))


def probs(x, t, top_k, top_p):
    """fp64 probabilities of the filtered softmax (the distribution the draw samples)."""
    z, _, M = row(x, t, top_k, top_p)
    k = kept(M, z, top_p)
    m = np.where(k, np.exp(z.astype(np.float64) - z.max()), 0.0)
    return m / m.sum()
