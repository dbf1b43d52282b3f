"""CPU tests of sqllm_lutgemm_t's argument validation: bad arguments are rejected with SQLLM_EINVAL and a message before anything
touches a device."""
import ctypes
import re

import pytest

from util import HEADER, Args, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


def _call(a, dy=16, dy_dt=F16, dx=16, dx_dt=F32, path=0):
    lib = load_lib()
    lib.sqllm_lutgemm_t.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_void_p]
    rc = lib.sqllm_lutgemm_t(None if a is None else ctypes.byref(a), dy, dy_dt, dx, dx_dt, path, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=132, batch=7, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change,frag", [
    (dict(bits=2), b"bits must be 3 or 4"), (dict(bits=8), b"bits must be 3 or 4"),
    (dict(in_features=100), b"in_features=100 must be a positive multiple of 32"),
    (dict(in_features=0), b"in_features=0 must be a positive multiple of 32"),
    (dict(in_features=65536 * 128), b"in_features=8388608 exceeds"),
    (dict(out_features=0), b"out_features=0 must be positive"),
    (dict(batch=0), b"batch (rows of dy) must be >= 1"), (dict(batch=-3), b"batch (rows of dy) must be >= 1"),
    (dict(qweight=0), b"qweight / lookup_table must not be null"), (dict(lookup_table=0), b"qweight / lookup_table must not be null"),
    (dict(qweight=18), b"4-byte aligned"), (dict(lookup_table=17), b"4-byte aligned"),
    (dict(topX=-1), b"topX < 0"), (dict(full_rows=16, topX=4), b"full_rows given without full_row_indices")])
def test_rejects_bad_descriptor(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("kw,frag", [
    (dict(dy=0), b"dy / dx must not be null"), (dict(dx=0), b"dy / dx must not be null"),
    (dict(dy_dt=3), b"dy_dtype=3 is not"), (dict(dy_dt=-1), b"dy_dtype=-1 is not"),
    (dict(dy_dt=F16, dx_dt=BF16), b"dx_dtype=2 must be SQLLM_DT_F32 or dy's dtype (1)"),
    (dict(dy_dt=F32, dx_dt=F16), b"dx_dtype=1 must be SQLLM_DT_F32 or dy's dtype (0)"),
    (dict(dx_dt=7), b"dx_dtype=7"),
    (dict(path=3), b"path=3 must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)"), (dict(path=-1), b"path=-1 must be"),
    (dict(path=1, dy_dt=F32), b"path=1 (tensor cores) takes fp16 or bf16 dy, not fp32"),
    (dict(dy=17, dy_dt=F16), b"dy must be aligned to its element size"),
    (dict(dy=18, dy_dt=F32), b"dy must be aligned to its element size"),
    (dict(dx=24), b"dx must be 16-byte aligned")])
def test_rejects_bad_pointers_dtypes_and_paths(kw, frag):
    rc, msg = _call(_args(), **kw)
    assert rc == -1 and frag in msg, msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null args" in msg


def test_declared_in_the_header_and_the_version_unchanged():
    assert "sqllm_lutgemm_t" in header_symbols()
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_lutgemm_t\(const sqllm_lutgemv_args \*args, const void \*dy, int dy_dtype, void \*dx, int dx_dtype, "
                     r"int path,\s+void \*stream\);", txt)
    for name, v in (("SQLLM_DT_F32", 0), ("SQLLM_DT_F16", 1), ("SQLLM_DT_BF16", 2), ("SQLLM_BWD_TC_MIN_ROWS", 96)):
        assert re.search(rf"#define {name} {v}\b", txt)
    assert load_lib().sqllm_abi_version() == 4
