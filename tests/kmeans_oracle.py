"""TEST INFRASTRUCTURE ONLY - Python face of tests/kmeans_oracle.c, the exact weighted 1-D k-means that checks the GPU quantizer.

The C source is compiled once per process into a temporary directory (removed at exit), so running the tests writes nothing into
the tree.  Independent of the CUDA code: qsort by (w, index), long double prefix sums, a depth-first divide-and-conquer DP per
level, OpenMP over rows.
"""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "kmeans_oracle.c")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="sqllm_kmeans_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libkmeans_oracle.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "gcc")
        subprocess.check_call([cc, "-O2", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=c11", "-shared", "-o", so, _SRC])
        _LIB = ctypes.CDLL(so)
    return _LIB


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def kmeans1d(w, s, k):
    """Exact weighted 1-D k-means of each row of w [rows, n] with sample weights s (long double DP).
    -> (optimum fp64 [rows], centroids fp64 [rows, k], labels uint8 [rows, n] = each element's segment)."""
    w = np.ascontiguousarray(np.atleast_2d(w), dtype=np.float32)
    s = np.ascontiguousarray(np.atleast_2d(s), dtype=np.float32)
    assert w.shape == s.shape and 1 <= k <= min(256, w.shape[1])
    rows, n = w.shape
    opt = np.empty(rows, dtype=np.float64)
    cent = np.empty((rows, k), dtype=np.float64)
    labels = np.empty((rows, n), dtype=np.uint8)
    _lib().sq_kmeans1d(_p(w), _p(s), ctypes.c_int(rows), ctypes.c_int(n), ctypes.c_int(k), _p(opt), _p(cent), _p(labels))
    return opt, cent, labels


def kmeans_objective(w, s, centroids, labels):
    """fp64 sum s (w - centroids[label])^2 per row, with all-zero weight rows weighted uniformly (as the quantizer does)."""
    w = np.atleast_2d(np.asarray(w, dtype=np.float64))
    s = np.atleast_2d(np.asarray(s, dtype=np.float64)).copy()
    s[s.sum(1) == 0] = 1.0
    c = np.take_along_axis(np.atleast_2d(np.asarray(centroids, dtype=np.float64)), np.atleast_2d(labels).astype(np.int64), 1)
    return (s * (w - c) ** 2).sum(1)
