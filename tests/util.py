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


def to_torch(layer, device="cuda"):
    """numpy layer dict (oracle.make_layer) -> dict of torch tensors on `device`."""
    import torch
    out = {}
    for k, v in layer.items():
        out[k] = torch.from_numpy(v).to(device) if isinstance(v, np.ndarray) else v
    return out
