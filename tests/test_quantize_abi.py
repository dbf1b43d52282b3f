"""CPU tests of the quantizer's C ABI argument checks (sqllm_kmeans1d_workspace_bytes, sqllm_kmeans1d, sqllm_pack_indices): bad
arguments are rejected with SQLLM_EINVAL (or SQLLM_EWORKSPACE) and a message before anything touches a device."""
import ctypes

import pytest

from util import header_symbols, load_lib

V, I, S = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t


def _lib():
    lib = load_lib()
    lib.sqllm_kmeans1d_workspace_bytes.argtypes = [I, I, I, ctypes.POINTER(S)]
    lib.sqllm_kmeans1d.argtypes = [V, V, I, I, I, V, V, V, S, V]
    lib.sqllm_pack_indices.argtypes = [I, V, I, I, V, V]
    return lib


@pytest.mark.parametrize("rows,n,k,frag", [
    (0, 64, 8, b"rows=0 must be >= 1"), (-2, 64, 8, b"rows=-2 must be >= 1"),
    (4, 64, 1, b"k=1 must be in [2, 16]"), (4, 64, 32, b"k=32 must be in [2, 16]"),
    (4, 7, 8, b"n=7 must be in [k=8, 65535]"), (4, 65536, 16, b"n=65536 must be in [k=16, 65535]")])
def test_kmeans_rejects_bad_shapes(rows, n, k, frag):
    lib = _lib()
    out = S(0)
    assert lib.sqllm_kmeans1d_workspace_bytes(rows, n, k, ctypes.byref(out)) == -1
    assert frag in lib.sqllm_last_error()
    assert lib.sqllm_kmeans1d(16, 16, rows, n, k, 16, 16, 256, 1 << 30, None) == -1
    assert frag in lib.sqllm_last_error()


def test_kmeans_workspace_bytes_rejects_null_out():
    lib = _lib()
    assert lib.sqllm_kmeans1d_workspace_bytes(4, 64, 8, None) == -1
    assert b"bytes must not be null" in lib.sqllm_last_error()


@pytest.mark.parametrize("ptrs,rc,frag", [
    (dict(w=0), -1, b"w / s / centroids / labels must not be null"), (dict(s=0), -1, b"must not be null"),
    (dict(c=0), -1, b"must not be null"), (dict(lab=0), -1, b"must not be null"),
    (dict(w=18), -1, b"4-byte aligned"), (dict(s=17), -1, b"4-byte aligned"), (dict(c=2), -1, b"4-byte aligned"),
    (dict(ws=0), -3, b"workspace must not be null"), (dict(ws=128), -1, b"workspace must be 256-byte aligned")])
def test_kmeans_rejects_bad_pointers(ptrs, rc, frag):
    lib = _lib()
    p = dict(w=16, s=16, c=16, lab=16, ws=256)
    p.update(ptrs)
    assert lib.sqllm_kmeans1d(p["w"] or None, p["s"] or None, 4, 64, 8, p["c"] or None, p["lab"] or None, p["ws"] or None,
                              1 << 30, None) == rc
    assert frag in lib.sqllm_last_error()


@pytest.mark.parametrize("args,frag", [
    (dict(bits=2), b"bits=2 must be 3 or 4"), (dict(bits=8), b"bits=8 must be 3 or 4"),
    (dict(K=0), b"in_features=0 must be a positive multiple of 32"), (dict(K=100), b"in_features=100 must be a positive multiple of 32"),
    (dict(N=0), b"out_features=0 must be >= 1"), (dict(N=-1), b"out_features=-1 must be >= 1"),
    (dict(lab=0), b"labels / qweight must not be null"), (dict(q=0), b"labels / qweight must not be null"),
    (dict(q=18), b"qweight must be 4-byte aligned")])
def test_pack_rejects_bad_arguments(args, frag):
    lib = _lib()
    a = dict(bits=4, lab=16, K=128, N=64, q=16)
    a.update(args)
    assert lib.sqllm_pack_indices(a["bits"], a["lab"] or None, a["K"], a["N"], a["q"] or None, None) == -1
    assert frag in lib.sqllm_last_error()


def test_declared_in_the_header_and_the_version_unchanged():
    syms = header_symbols()
    for name in ("sqllm_kmeans1d_workspace_bytes", "sqllm_kmeans1d", "sqllm_pack_indices"):
        assert name in syms
    assert load_lib().sqllm_abi_version() == 4
