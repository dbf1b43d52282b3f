"""CPU tests of the argument checks of sqllm_sequence_create_dt and sqllm_lutgemv_fused_exchange_dt: a dtype code either entry point
does not take comes back as SQLLM_EINVAL with a message naming the code, and the checks they share with sqllm_sequence_create /
sqllm_lutgemv_fused_exchange still apply, all before anything touches a device."""
import ctypes

import pytest

from test_sequence_host import SeqItem, SeqOptions, _item
from util import Args, load_lib

F32, F16, BF16 = 0, 1, 2
CODES = [F32, F16, BF16, -1, 3, 99]
FUSED_OK = {(F32, F32), (F32, F16), (F16, F32), (F16, F16), (BF16, F32), (BF16, BF16)}


class Exchange(ctypes.Structure):  # mirrors sqllm_exchange
    _fields_ = [("world", ctypes.c_int), ("rank", ctypes.c_int), ("members", ctypes.c_int), ("out_features_full", ctypes.c_int),
                ("peer_base", ctypes.c_void_p), ("out_offset", ctypes.c_size_t), ("flag_offset", ctypes.c_size_t),
                ("state_offset", ctypes.c_size_t), ("error_offset", ctypes.c_size_t)]


def _lib():
    lib = load_lib()
    lib.sqllm_sequence_create_dt.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.sqllm_lutgemv_fused_exchange_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _create(items, dtype, **opt):
    lib = _lib()
    arr = (SeqItem * len(items))(*items) if items else None
    o = SeqOptions(lut_mode=opt.get("lut_mode", 0), world=opt.get("world", 1), rank=opt.get("rank", 0))
    if "exports" in opt:
        its, dsts = zip(*opt["exports"])
        ei, ed = (ctypes.c_int * len(its))(*its), (ctypes.c_void_p * len(dsts))(*dsts)
        o.n_export, o.export_items, o.export_dst = len(its), ctypes.cast(ei, ctypes.c_void_p), ctypes.cast(ed, ctypes.c_void_p)
    h = ctypes.c_void_p()
    rc = lib.sqllm_sequence_create_dt(arr, len(items), ctypes.byref(o), dtype, ctypes.byref(h))
    return rc, lib.sqllm_last_error().decode()


def _exchange(a, dtypes, x=16, xc=True, ws=16, ws_bytes=1 << 30, **kw):
    lib = _lib()
    e = Exchange(world=kw.get("world", 1), rank=kw.get("rank", 0), members=kw.get("members", 1), out_features_full=kw.get("nfull", 128),
                 peer_base=16, out_offset=4096, flag_offset=0, state_offset=64, error_offset=128)
    rc = lib.sqllm_lutgemv_fused_exchange_dt(None if a is None else ctypes.byref(a), x, dtypes[0], dtypes[1], None, ws, ws_bytes,
                                             ctypes.byref(e) if xc else None, None)
    return rc, lib.sqllm_last_error().decode()


def _args(**kw):
    a = Args(bits=4, in_features=256, out_features=128, batch=1, qweight=16, lookup_table=16, vec=0, mul=0)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("dtype", [F32, -1, 3, 99])
def test_sequence_create_dt_rejects_dtype(dtype):
    rc, msg = _create([_item()], dtype)
    assert rc == -1 and f"dtype={dtype}" in msg, msg


def test_sequence_create_dt_checks_the_dtype_first():
    rc, msg = _create([], F32)   # null items too: the dtype is named
    assert rc == -1 and "dtype=0" in msg, msg


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("items,kw,needle", [
    ([], {}, "null / empty"),
    ([_item(), _item(bits=3, x_from=0)], {}, "one sequence, one width"),
    ([_item(), _item(x_from=1)], {}, "must name an earlier item"),
    ([_item(N=256), _item(K=256, x_from=0, x_offset=2)], {}, "reads ["),
    ([_item(N=256), _item(K=512, x_from=0)], {}, "reads ["),
    ([_item(N=32)], {}, "out_features=32 <"),
    ([_item(N=256, members=3)], {}, "members of a multiple of 4"),
    ([_item()], {"world": 2, "rank": 0}, "peer-visible arena"),
    ([_item()], {"world": 2, "rank": 5}, "bad world / rank"),
    ([_item()], {"exports": [(1, 16)]}, "export 0: bad item 1"),
    ([_item()], {"exports": [(0, 20)]}, "export 0: bad item 0"),
    ([_item()], {"lut_mode": 1, "world": 2, "rank": 2}, "bad world / rank"),
])
def test_sequence_create_dt_keeps_the_sequence_checks(items, kw, needle, dtype):
    rc, msg = _create(items, dtype, **kw)
    assert rc == -1 and needle in msg, (rc, msg)


@pytest.mark.parametrize("dtype,name", [(F16, "fp16"), (BF16, "bf16")])
def test_sequence_messages_name_the_dtype(dtype, name):
    it = _item()
    it.x_ext = 16 + 8   # misaligned
    rc, msg = _create([it], dtype)
    assert rc == -1 and f"x_ext must be a 16-byte aligned {name} vector" in msg, msg
    rc, msg = _create([_item()], dtype, exports=[(0, 12)])
    assert rc == -1 and f"8-byte aligned {name} vector" in msg, msg


@pytest.mark.parametrize("x_dtype,y_dtype", [(x, y) for x in CODES for y in CODES if (x, y) not in FUSED_OK])
def test_exchange_dt_rejects_dtype_pair(x_dtype, y_dtype):
    rc, msg = _exchange(_args(), (x_dtype, y_dtype))
    assert rc == -1 and f"x_dtype={x_dtype}, y_dtype={y_dtype}" in msg, msg


@pytest.mark.parametrize("dtypes", sorted(FUSED_OK))
@pytest.mark.parametrize("change,kw,frag", [
    (dict(bits=2), {}, "bits"), (dict(in_features=100), {}, "in_features"), (dict(qweight=0), {}, "null"),
    (dict(qweight=24), {}, "qweight must be 16-byte aligned"),
    ({}, {"xc": False}, "exchange descriptor must not be null"),
    ({}, {"x": 0}, "must not be null"),
    ({}, {"x": 24}, "x must be 16-byte aligned"),
    ({}, {"rank": 1}, "bad world / rank"),
    ({}, {"members": 3}, "equal members"),
    ({}, {"nfull": 64}, "out_features_full=64"),
    ({}, {"ws": 0}, "workspace too small"),
])
def test_exchange_dt_keeps_the_exchange_checks(change, kw, frag, dtypes):
    rc, msg = _exchange(_args(**change), dtypes, **kw)
    assert rc in (-1, -3) and frag in msg, (rc, msg)


def test_exchange_dt_null_descriptor():
    rc, msg = _exchange(None, (BF16, BF16))
    assert rc == -1 and "null" in msg, msg


def test_header_declares_and_library_exports_the_entry_points():
    from util import HEADER, header_symbols
    syms = header_symbols()
    txt = open(HEADER).read()
    later = txt.split("#define SQLLM_ABI_VERSION")[1].split("*/")[0]  # the "later +" list
    lib = load_lib()
    for name in ("sqllm_sequence_create_dt", "sqllm_lutgemv_fused_exchange_dt"):
        assert name in syms and name in later
        assert hasattr(lib, name)
    assert lib.sqllm_abi_version() == 4
