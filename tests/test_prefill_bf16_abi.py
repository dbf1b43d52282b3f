"""CPU tests of sqllm_lutgemm_fused_dt's argument validation: every rejection of sqllm_lutgemm_fused, and bad dtype codes, come
back as SQLLM_EINVAL with a message naming the argument, before anything touches a device."""
import ctypes

import pytest

from util import Args, load_lib

F32, F16, BF16 = 0, 1, 2


def _call(a, x=16, y=16, bias=None, x_dtype=BF16, y_dtype=F32):
    lib = load_lib()
    lib.sqllm_lutgemm_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_lutgemm_fused_dt(None if a is None else ctypes.byref(a), x, x_dtype, y, y_dtype, bias, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=128, batch=17, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("x_dtype,y_dtype", [(BF16, F32), (BF16, BF16), (F16, F32), (F16, F16)])
@pytest.mark.parametrize("change,frag", [(dict(bits=2), b"bits"), (dict(bits=8), b"bits"), (dict(in_features=100), b"in_features"),
                                         (dict(in_features=0), b"in_features"), (dict(out_features=0), b"out_features"),
                                         (dict(out_features=65536 * 128), b"out_features"),
                                         (dict(batch=0), b"batch"), (dict(batch=-3), b"batch"),
                                         (dict(qweight=0), b"null"), (dict(lookup_table=0), b"null"),
                                         (dict(qweight=18), b"aligned"), (dict(lookup_table=20 + 2), b"aligned"),
                                         (dict(topX=-1), b"topX"), (dict(full_rows=16, topX=4), b"full_row_indices")])
def test_rejects_bad_descriptor(change, frag, x_dtype, y_dtype):
    rc, msg = _call(_args(**change), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("x_dtype", [BF16, F16])
@pytest.mark.parametrize("ptrs,frag", [(dict(x=0), b"null"), (dict(y=0), b"null"), (dict(x=24), b"x must be 16-byte aligned"),
                                       (dict(x=16 + 2), b"x must be 16-byte aligned"), (dict(y=40), b"y must be 16-byte aligned"),
                                       (dict(bias=18), b"aligned")])
def test_rejects_null_and_misaligned_pointers(ptrs, frag, x_dtype):
    rc, msg = _call(_args(), x_dtype=x_dtype, **ptrs)
    assert rc == -1 and frag in msg, msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null" in msg


@pytest.mark.parametrize("x_dtype", [F32, -1, 3, 99])
def test_rejects_x_dtype(x_dtype):
    """fp32 x (not exact in a 16-bit operand) and unknown codes."""
    rc, msg = _call(_args(), x_dtype=x_dtype, y_dtype=F32)
    assert rc == -1 and b"x_dtype" in msg and b"SQLLM_DT_F16" in msg and b"SQLLM_DT_BF16" in msg, msg


@pytest.mark.parametrize("x_dtype,y_dtype", [(BF16, F16), (F16, BF16), (BF16, -1), (F16, 3), (BF16, 7)])
def test_rejects_y_dtype(x_dtype, y_dtype):
    """y is fp32 or x's own dtype."""
    rc, msg = _call(_args(), x_dtype=x_dtype, y_dtype=y_dtype)
    assert rc == -1 and b"y_dtype" in msg and b"x's dtype" in msg, msg


def test_header_declares_the_entry_point():
    from util import HEADER, header_symbols
    assert "sqllm_lutgemm_fused_dt" in header_symbols()
    txt = open(HEADER).read()
    assert "sqllm_lutgemm_fused_dt" in txt.split("#define SQLLM_ABI_VERSION")[1].split("*/")[0]  # in the "later +" list
    assert load_lib().sqllm_abi_version() == 4
