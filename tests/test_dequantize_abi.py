"""CPU tests of sqllm_dequantize's argument validation: bad arguments are rejected with SQLLM_EINVAL and a message before anything
touches a device.  The checks of quant_cuda.dequantize that need CUDA tensors are in test_dequantize_gpu.py."""
import ctypes
import re

import pytest

from util import HEADER, Args, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


def _call(a, col0=0, ncols=132, w=16, w_dt=F16):
    lib = load_lib()
    lib.sqllm_dequantize.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    rc = lib.sqllm_dequantize(None if a is None else ctypes.byref(a), col0, ncols, w, w_dt, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=132, batch=0, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change,frag", [
    (dict(bits=2), b"bits must be 3 or 4"), (dict(bits=8), b"bits must be 3 or 4"),
    (dict(in_features=100), b"in_features=100 must be a positive multiple of 32"),
    (dict(in_features=0), b"in_features=0 must be a positive multiple of 32"),
    (dict(in_features=65536 * 128), b"in_features=8388608 exceeds 8388480"),
    (dict(out_features=0), b"out_features=0 must be positive"), (dict(out_features=-4), b"out_features=-4 must be positive"),
    (dict(qweight=0), b"qweight / lookup_table must not be null"), (dict(lookup_table=0), b"qweight / lookup_table must not be null"),
    (dict(qweight=18), b"qweight and lookup_table must be 4-byte aligned"),
    (dict(lookup_table=17), b"qweight and lookup_table must be 4-byte aligned"),
    (dict(topX=-1), b"topX < 0"), (dict(full_rows=16, topX=4), b"full_rows given without full_row_indices")])
def test_rejects_bad_descriptor(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("col0,ncols", [(-1, 4), (0, 0), (0, -1), (0, 133), (130, 3), (132, 1), (1, 132), (2**31 - 1, 2)])
def test_rejects_bad_column_range(col0, ncols):
    rc, msg = _call(_args(), col0=col0, ncols=ncols)
    assert rc == -1, msg
    assert f"column range col0={col0}, ncols={ncols} must be non-empty and lie in [0, out_features=132)".encode() in msg, msg


@pytest.mark.parametrize("kw,frag", [
    (dict(w=0), b"w must not be null"),
    (dict(w_dt=3), b"w_dtype=3 is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16"), (dict(w_dt=-1), b"w_dtype=-1 is not"),
    (dict(w=24), b"w must be 16-byte aligned"), (dict(w=20, w_dt=F32), b"w must be 16-byte aligned"),
    (dict(w=18, w_dt=BF16), b"w must be 16-byte aligned")])
def test_rejects_bad_output(kw, frag):
    rc, msg = _call(_args(), **kw)
    assert rc == -1 and frag in msg, msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null args" in msg


def test_module_rejects_a_cpu_qweight():
    torch = pytest.importorskip("torch")
    from squeezellm_b200.quant import quant_cuda
    with pytest.raises(RuntimeError, match="dequantize: qweight must be a contiguous CUDA tensor"):
        quant_cuda.dequantize(torch.zeros(20, 8, dtype=torch.int32), torch.zeros(8, 16), 4)


def test_declared_in_the_header_and_the_version_unchanged():
    assert "sqllm_dequantize" in header_symbols()
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_dequantize\(const sqllm_lutgemv_args \*args, int col0, int ncols, void \*w, int w_dtype, "
                     r"void \*stream\);", txt)
    assert "sqllm_dequantize" in txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert load_lib().sqllm_abi_version() == 4
