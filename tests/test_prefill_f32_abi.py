"""CPU tests of sqllm_lutgemm_fused_f32's argument validation: every rejection of sqllm_lutgemm_fused_dt comes back as SQLLM_EINVAL with
a message naming the argument, before anything touches a device."""
import ctypes

import pytest

from util import Args, load_lib


def _call(a, x=16, y=16, bias=None):
    lib = load_lib()
    lib.sqllm_lutgemm_fused_f32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_lutgemm_fused_f32(None if a is None else ctypes.byref(a), x, y, bias, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=128, batch=17, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change,frag", [(dict(bits=2), b"bits"), (dict(bits=8), b"bits"), (dict(in_features=100), b"in_features"),
                                         (dict(in_features=0), b"in_features"), (dict(in_features=-32), b"in_features"),
                                         (dict(out_features=0), b"out_features"), (dict(out_features=65536 * 128), b"out_features"),
                                         (dict(batch=0), b"batch"), (dict(batch=-3), b"batch"),
                                         (dict(qweight=0), b"null"), (dict(lookup_table=0), b"null"),
                                         (dict(qweight=18), b"aligned"), (dict(lookup_table=20 + 2), b"aligned"),
                                         (dict(topX=-1), b"topX"), (dict(full_rows=16, topX=4), b"full_row_indices")])
def test_rejects_bad_descriptor(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


def test_out_features_limit_is_that_of_the_dtype_entry():
    """65535 N-tiles of 128 columns: the last accepted width passes the checks up to the device set-up."""
    rc, msg = _call(_args(out_features=65536 * 128))
    assert rc == -1 and b"out_features=8388608 exceeds 8388480" in msg, msg


@pytest.mark.parametrize("ptrs,frag", [(dict(x=0), b"x / y must not be null"), (dict(y=0), b"x / y must not be null"),
                                       (dict(x=24), b"x must be 16-byte aligned"), (dict(x=16 + 4), b"x must be 16-byte aligned"),
                                       (dict(y=40), b"y must be 16-byte aligned"), (dict(y=16 + 8), b"y must be 16-byte aligned"),
                                       (dict(bias=18), b"aligned")])
def test_rejects_null_and_misaligned_pointers(ptrs, frag):
    rc, msg = _call(_args(), **ptrs)
    assert rc == -1 and frag in msg, msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null" in msg


def test_checks_run_in_the_dtype_entry_order():
    """A descriptor fault is reported before a null x, and a null x before a misaligned one: the same order as
    sqllm_lutgemm_fused_dt."""
    rc, msg = _call(_args(bits=5), x=0)
    assert rc == -1 and b"bits" in msg, msg
    rc, msg = _call(_args(batch=0), x=0)
    assert rc == -1 and b"batch" in msg, msg
    rc, msg = _call(_args(), x=0, y=40)
    assert rc == -1 and b"null" in msg, msg


def test_header_declares_the_entry_point():
    from util import HEADER, header_symbols
    assert "sqllm_lutgemm_fused_f32" in header_symbols()
    txt = open(HEADER).read()
    assert "sqllm_lutgemm_fused_f32" in txt.split("#define SQLLM_ABI_VERSION")[1].split("*/")[0]  # in the "later +" list
    assert load_lib().sqllm_abi_version() == 4


def test_dtype_entry_still_rejects_fp32_x():
    """fp32 x has an entry point of its own; sqllm_lutgemm_fused_dt keeps taking fp16 and bf16 only."""
    lib = load_lib()
    lib.sqllm_lutgemm_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_lutgemm_fused_dt(ctypes.byref(_args()), 16, 0, 16, 0, None, None)
    assert rc == -1 and b"x_dtype" in lib.sqllm_last_error()
