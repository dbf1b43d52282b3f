"""CPU tests of the argument checks of sqllm_lutgemv_fused_dt and sqllm_lutgemv_rows_dt: every dtype pair either entry point does
not take, and the checks they share with sqllm_lutgemv_fused / sqllm_lutgemv_rows, come back as SQLLM_EINVAL (or SQLLM_EWORKSPACE)
with a message naming the argument, before anything touches a device."""
import ctypes

import pytest

from util import Args, load_lib

F32, F16, BF16 = 0, 1, 2
CODES = [F32, F16, BF16, -1, 3, 99]
FUSED_OK = {(F32, F32), (F32, F16), (F16, F32), (F16, F16), (BF16, F32), (BF16, BF16)}
ROWS_OK = {(F16, F32), (F16, F16), (BF16, F32), (BF16, BF16)}


def _lib():
    lib = load_lib()
    lib.sqllm_lutgemv_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.sqllm_lutgemv_rows_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _fused(a, x=16, y=16, bias=None, x_dtype=BF16, y_dtype=F32, ws=16, ws_bytes=1 << 30):
    lib = _lib()
    rc = lib.sqllm_lutgemv_fused_dt(None if a is None else ctypes.byref(a), x, x_dtype, y, y_dtype, bias, ws, ws_bytes, None)
    return rc, lib.sqllm_last_error()


def _rows(a, x=16, y=16, bias=None, x_dtype=BF16, y_dtype=F32):
    lib = _lib()
    rc = lib.sqllm_lutgemv_rows_dt(None if a is None else ctypes.byref(a), x, x_dtype, y, y_dtype, bias, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=256, out_features=128, batch=9, qweight=16, lookup_table=16, vec=16, mul=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("x_dtype,y_dtype", [(x, y) for x in CODES for y in CODES if (x, y) not in FUSED_OK])
def test_fused_rejects_dtype_pair(x_dtype, y_dtype):
    rc, msg = _fused(_args(), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and f"x_dtype={x_dtype}, y_dtype={y_dtype}".encode() in msg, msg


@pytest.mark.parametrize("x_dtype,y_dtype", [(x, y) for x in CODES for y in CODES if (x, y) not in ROWS_OK])
def test_rows_rejects_dtype_pair(x_dtype, y_dtype):
    rc, msg = _rows(_args(), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and f"x_dtype={x_dtype}, y_dtype={y_dtype}".encode() in msg, msg


@pytest.mark.parametrize("x_dtype,y_dtype", sorted(FUSED_OK))
@pytest.mark.parametrize("change,frag", [(dict(bits=2), b"bits"), (dict(in_features=100), b"in_features"),
                                         (dict(in_features=0), b"in_features"), (dict(out_features=0), b"out_features"),
                                         (dict(qweight=0), b"null"), (dict(lookup_table=0), b"null"),
                                         (dict(qweight=24), b"qweight must be 16-byte aligned"),
                                         (dict(lookup_table=40), b"lookup_table must be 16-byte aligned"),
                                         (dict(topX=-1), b"topX"), (dict(full_rows=16, topX=4), b"full_row_indices"),
                                         (dict(full_rows=16, full_row_indices=16, topX=129), b"topX <= 128")])
def test_fused_rejects_bad_descriptor(change, frag, x_dtype, y_dtype):
    rc, msg = _fused(_args(**change), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("x_dtype", [BF16, F16, F32])
@pytest.mark.parametrize("ptrs,frag", [(dict(x=0), b"null"), (dict(y=0), b"null"), (dict(x=24), b"x must be 16-byte aligned"),
                                       (dict(x=16 + 2), b"x must be 16-byte aligned"), (dict(y=40), b"y and bias must be 16-byte aligned"),
                                       (dict(bias=20), b"y and bias must be 16-byte aligned")])
def test_fused_rejects_null_and_misaligned_pointers(ptrs, frag, x_dtype):
    rc, msg = _fused(_args(), x_dtype=x_dtype, **ptrs)
    assert rc == -1 and frag in msg, msg


def test_fused_rejects_a_missing_or_small_workspace():
    for ws, n in ((0, 1 << 30), (16, 1024)):
        rc, msg = _fused(_args(), ws=ws, ws_bytes=n)
        assert rc == -3 and b"workspace too small" in msg, msg


@pytest.mark.parametrize("x_dtype,y_dtype", sorted(ROWS_OK))
@pytest.mark.parametrize("change,frag", [(dict(bits=2), b"bits"), (dict(in_features=100), b"in_features"),
                                         (dict(in_features=49152 + 32), b"exceeds 49152"),
                                         (dict(out_features=130), b"multiple of 4"), (dict(out_features=0), b"out_features"),
                                         (dict(out_features=65536 * 64), b"out_features"),
                                         (dict(batch=0), b"batch"), (dict(qweight=0), b"null"), (dict(lookup_table=0), b"null"),
                                         (dict(qweight=18), b"aligned"), (dict(topX=-1), b"topX"),
                                         (dict(full_rows=16, topX=4), b"full_row_indices")])
def test_rows_rejects_bad_descriptor(change, frag, x_dtype, y_dtype):
    rc, msg = _rows(_args(**change), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("x_dtype", [BF16, F16])
@pytest.mark.parametrize("ptrs,frag", [(dict(x=0), b"null"), (dict(y=0), b"null"), (dict(x=24), b"x must be 16-byte aligned"),
                                       (dict(y=40), b"y must be 16-byte aligned"), (dict(bias=18), b"aligned")])
def test_rows_rejects_null_and_misaligned_pointers(ptrs, frag, x_dtype):
    rc, msg = _rows(_args(), x_dtype=x_dtype, **ptrs)
    assert rc == -1 and frag in msg, msg


def test_null_descriptor():
    for call in (_fused, _rows):
        rc, msg = call(None)
        assert rc == -1 and b"null" in msg, msg


def test_header_declares_the_entry_points():
    from util import HEADER, header_symbols
    syms = header_symbols()
    txt = open(HEADER).read()
    later = txt.split("#define SQLLM_ABI_VERSION")[1].split("*/")[0]  # the "later +" list
    for name in ("sqllm_lutgemv_fused_dt", "sqllm_lutgemv_rows_dt"):
        assert name in syms and name in later
    assert load_lib().sqllm_abi_version() == 4
