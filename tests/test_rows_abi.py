"""CPU tests of sqllm_lutgemv_rows's argument validation: bad arguments are rejected with SQLLM_EINVAL and a message before
anything touches a device."""
import ctypes

import pytest

from util import Args, load_lib


def _call(a, x=16, y=16, bias=None):
    lib = load_lib()
    lib.sqllm_lutgemv_rows.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_lutgemv_rows(None if a is None else ctypes.byref(a), x, y, 1, bias, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=128, batch=7, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change,frag", [
    (dict(bits=2), b"bits must be 3 or 4"), (dict(bits=8), b"bits must be 3 or 4"),
    (dict(in_features=100), b"in_features=100 must be a positive multiple of 32"),
    (dict(in_features=0), b"in_features=0 must be a positive multiple of 32"),
    (dict(in_features=49184), b"in_features=49184 exceeds 49152"),
    (dict(out_features=0), b"out_features=0 must be a positive multiple of 4"),
    (dict(out_features=130), b"out_features=130 must be a positive multiple of 4"),
    (dict(out_features=65536 * 64), b"out_features=4194304 exceeds"),
    (dict(batch=0), b"batch"), (dict(batch=-3), b"batch"),
    (dict(qweight=0), b"qweight / lookup_table must not be null"), (dict(lookup_table=0), b"qweight / lookup_table must not be null"),
    (dict(qweight=18), b"4-byte aligned"), (dict(lookup_table=17), b"4-byte aligned"),
    (dict(topX=-1), b"topX < 0"), (dict(full_rows=16, topX=4), b"full_rows given without full_row_indices")])
def test_rejects_bad_descriptor(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("ptrs,frag", [(dict(x=0), b"x / y must not be null"), (dict(y=0), b"x / y must not be null"),
                                       (dict(x=24), b"x must be 16-byte aligned"), (dict(y=40), b"y must be 16-byte aligned"),
                                       (dict(bias=18), b"4-byte aligned")])
def test_rejects_null_and_misaligned_pointers(ptrs, frag):
    rc, msg = _call(_args(), **ptrs)
    assert rc == -1 and frag in msg, msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null args" in msg


def test_declared_in_the_header_and_the_version_unchanged():
    from util import header_symbols
    assert "sqllm_lutgemv_rows" in header_symbols()
    lib = load_lib()
    assert lib.sqllm_abi_version() == 4
