"""Shared helpers for the test-suite (oracle access, tolerances, ctypes view of the C ABI)."""
import ctypes
import glob
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import oracle as orc  # noqa: E402  (tests are allowed to use the oracle)

GOLDEN = os.path.join(ROOT, "tests", "golden")
LIB = os.path.join(ROOT, "squeezellm_b200", "libsqllm_b200.so")
HEADER = os.path.join(ROOT, "include", "sqllm_b200.h")

# north_star: outputs match the reference to <= 1e-3 max relative error.  Relative error needs an absolute
# floor for outputs that cancel to ~0 (SURVEY.md 8(c)); defined once, here:
#     err = max_i |a_i - b_i| / max(|b_i|, FLOOR * max_j |b_j|)
REL_TOL = 1e-3
FLOOR = 1e-2
# our kernels accumulate in fp32 with a fixed order; against the fp64 truth they must be far inside REL_TOL
TIGHT_TOL = 5e-5


def rel_err(a, b, b_absmax=None):
    """b_absmax: max|b| over the whole vector when a and b are a sample of it (the floor stays that of the whole vector)."""
    a = np.asarray(a, dtype=np.float64).ravel()
    b = np.asarray(b, dtype=np.float64).ravel()
    assert a.shape == b.shape
    den = np.maximum(np.abs(b), FLOOR * max(np.abs(b).max() if b_absmax is None else b_absmax, 1e-30))
    return float((np.abs(a - b) / den).max())


"""Per-element, condition-aware error bound.  rel_err's floor is 1 % of the largest output of the whole array, so an output far
below the largest (a token whose activations are 1e-3 of another's) can be off by percents and still pass.  This bound scales with
each element's own condition instead:

    |got_i - want_i| <= r * |rounded_i| + eta + (1 + r) * e * S_i,      S_i = sum_k |x_k| |w_kc| + |bias_c|

  * S: the oracle on abs_layer(L) and |x| (|lut + csr + dense| <= |lut| + |csr| + |dense|), with |bias| as one more term.
  * r, eta: the final rounding to the output dtype (OUT_ROUNDING: relative unit roundoff and half the smallest subnormal);
    `rounded` is the value that was rounded: the whole output when the bias is inside the sum, the sum without the bias where the
    module rounds first and adds the bias afterwards.  The (1 + r) factor covers rounding a value that already carries e * S.
  * e = E_ACC = 2^-20 = 16 u (u = 2^-24, fp32): every route forms each output from fp32 products that are exact (tensor cores) or
    rounded once (CUDA cores: <= u * S together) and fp32 sums (DESIGN.md 3.1-3.6).  The tensor-core path also rounds the outlier
    fold (lut + csr + dense, <= 2 u of each |w| with distinct dense rows) and keeps 22 bits of each folded weight in its hi/lo
    split (<= 4 u of each |w|).  Additions: sums of terms of either sign keep their partial sums near sqrt(j) terms, so their
    rounding errors total about u * S, not the worst case of (number of additions) * u * S (Higham & Mary, SIAM J. Sci. Comput.
    41(5), 2019).  That is at most about 7 u; 16 u leaves a factor of two.
"""
U32 = 2.0 ** -24
E_ACC = 2.0 ** -20
OUT_ROUNDING = {"float32": (0.0, 0.0), "float16": (2.0 ** -11, 2.0 ** -25), "bfloat16": (2.0 ** -8, 2.0 ** -134)}


def abs_layer(L):
    """Copy of the layer dict with lookup_table, vals and full_rows replaced by their absolute values."""
    A = dict(L)
    for k in ("lookup_table", "vals", "full_rows"):
        if A.get(k) is not None:
            A[k] = np.abs(A[k])
    return A


def abs_sum(L, x, bias=None):
    """S [rows, N] = sum_k |x_k| |w_kc| (+ |bias_c|) in fp64: the condition of every output."""
    return orc.forward_f64(abs_layer(L), np.abs(x), mul_init=None if bias is None else np.abs(bias)[None, :])


def bound_ratio(got, want, S, rounded=None, r=0.0, e=E_ACC, eta=0.0):
    """max_i |got_i - want_i| / (r |rounded_i| + eta + (1 + r) e S_i); <= 1 passes.  rounded defaults to want.  An element whose
    allowance is 0 (an all-zero row without bias) must be exact: any difference there gives inf, a NaN gives NaN."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape == np.shape(S), (got.shape, want.shape, np.shape(S))
    rounded = want if rounded is None else np.asarray(rounded, dtype=np.float64)
    err = np.abs(got - want)
    den = r * np.abs(rounded) + eta + (1.0 + r) * e * np.asarray(S, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / den)
    return float(q.max()) if q.size else 0.0


MASSIVE_SCALE = 100.0


def massive_channels(K):
    """The three fixed input channels that carry "massive activations" in make_activations."""
    return np.array([5, K // 2 + 3, K - 7])


def make_activations(K, M, seed=0):
    """Prefill-like fp16-exact activations [M, K] (fp32 array): rows of N(0, 1), each scaled by 10^U(-3, 2), with row 0 scaled by
    exactly 1e-3 and row 1 by 1e2; the massive_channels x100 in every row; row 2 all zero and row 3 a single non-zero entry.  A
    1e-3 row holds fp16 subnormals (|x| < 2^-14) in about 5 % of its entries."""
    rng = np.random.default_rng(seed + 4242)
    scale = 10.0 ** rng.uniform(-3.0, 2.0, size=M)
    scale[:2] = (1e-3, 1e2)[:M]
    x = rng.standard_normal((M, K)) * scale[:, None]
    x[:, massive_channels(K)] *= MASSIVE_SCALE
    x = np.clip(x, -60000.0, 60000.0).astype(np.float16).astype(np.float32)
    if M > 2:
        x[2] = 0.0
    if M > 3:
        x[3] = 0.0
        x[3, K // 3] = 1.5
    return x


def sample_idx(n, cap=2048):
    """The output positions kept in golden data of large outputs: all of them up to `cap`, else `cap` positions spread over
    the vector by a prime stride (7919 divides none of the sizes used)."""
    if n <= cap:
        return np.arange(n)
    assert n % 7919
    return (np.arange(cap, dtype=np.int64) * 7919 + 13) % n


def golden_files(prefix):
    return sorted(glob.glob(os.path.join(GOLDEN, prefix + "*.npz")))


def header_symbols():
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(sqllm_\w+)\s*\(", txt)))


def load_lib():
    lib = ctypes.CDLL(LIB)
    lib.sqllm_last_error.restype = ctypes.c_char_p
    lib.sqllm_workspace_bytes.restype = ctypes.c_size_t
    return lib


class Args(ctypes.Structure):  # mirrors sqllm_lutgemv_args
    _fields_ = [("bits", ctypes.c_int), ("in_features", ctypes.c_int), ("out_features", ctypes.c_int),
                ("batch", ctypes.c_int), ("qweight", ctypes.c_void_p), ("lookup_table", ctypes.c_void_p),
                ("vec", ctypes.c_void_p), ("mul", ctypes.c_void_p), ("rows", ctypes.c_void_p),
                ("cols", ctypes.c_void_p), ("vals", ctypes.c_void_p), ("full_rows", ctypes.c_void_p),
                ("full_row_indices", ctypes.c_void_p), ("topX", ctypes.c_int)]


def late_owned_strips(bits, K, N, sm, first=8):
    """Strips that are the (first+1)-th or later strip owned by some CTA of the one-CTA-per-SM kernels (lutgemv_v2.cuh, lutgemv_seq.cuh):
    the [strip][unit] space (R units per 64-column strip) is cut into chunks of 2*ceil(T / (2*sm)) units, and a strip is owned by the CTA
    in whose chunk it starts.  Their finishers keep `first` = 8 owned strips in shared memory; the sums of later ones go through the
    global accumulator."""
    R = K // 8 if bits == 4 else K // 32
    strips = (N + 63) // 64
    T = strips * R
    chunk = max(2, 2 * ((T + 2 * sm - 1) // (2 * sm)))
    out = []
    for b in range((T + chunk - 1) // chunk):
        so0, so1 = (b * chunk + R - 1) // R, (min(T, (b + 1) * chunk) + R - 1) // R
        out.extend(range(so0 + first, so1))
    return np.asarray(out, dtype=np.int64)


def quant_layer(layer, **override):
    """The QuantLinearLUT (CPU buffers) of an oracle layer dict (oracle.make_layer), through QuantLinearLUT.from_buffers on copies
    of its arrays; `override` replaces entries first (bias=None: a layer without a bias)."""
    import torch
    from squeezellm_b200.quant import QuantLinearLUT
    d = dict(layer, **override)
    return QuantLinearLUT.from_buffers(d["bits"], {k: torch.tensor(v) for k, v in d.items() if isinstance(v, np.ndarray)})


def layer_as_read(m):
    """The oracle layer dict of what QuantLinearLUT m's own forward reads (CPU buffers): its packed words and LUT rows, and the
    outliers that m._sparse_args() gives it; no bias."""
    rows, cols, vals, fr, fri = (t.numpy() if t is not None else None for t in m._sparse_args())
    return dict(bits=m.bits, infeatures=m.infeatures, outfeatures=m.outfeatures, qweight=m.qweight.contiguous().numpy(),
                lookup_table=m.lookup_table.contiguous().numpy(), bias=None, rows=rows, cols=cols, vals=vals, full_rows=fr,
                full_row_indices=fri)


def to_torch(layer, device="cuda"):
    """numpy layer dict (oracle.make_layer) -> dict of torch tensors on `device`."""
    import torch
    out = {}
    for k, v in layer.items():
        out[k] = torch.from_numpy(v).to(device) if isinstance(v, np.ndarray) else v
    return out
