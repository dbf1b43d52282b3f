"""CPU tests of the argument checks of sqllm_attn_decode_paged / sqllm_attn_extend_paged and of their quant_cuda bindings: every bad
argument is rejected (SQLLM_EINVAL, or RuntimeError in Python) with a message naming the field, before anything touches a device."""
import ctypes
import math
import re

import pytest
import torch

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2
P = ctypes.c_void_p


class DecodeArgs(ctypes.Structure):  # mirrors sqllm_attn_decode_paged_args
    _fields_ = [("dtype", ctypes.c_int), ("batch", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int),
                ("head_dim", ctypes.c_int), ("capacity", ctypes.c_int), ("scale", ctypes.c_float), ("qkv", P), ("pos", P),
                ("rope_cos", P), ("rope_sin", P), ("k_pages", P), ("v_pages", P), ("n_pages", ctypes.c_int), ("block_table", P),
                ("table_width", ctypes.c_int), ("out", P)]


class ExtendArgs(ctypes.Structure):  # mirrors sqllm_attn_extend_paged_args
    _fields_ = [("dtype", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int), ("head_dim", ctypes.c_int),
                ("capacity", ctypes.c_int), ("start", ctypes.c_int), ("n_tokens", ctypes.c_int), ("scale", ctypes.c_float), ("qkv", P),
                ("rope_cos", P), ("rope_sin", P), ("k_pages", P), ("v_pages", P), ("n_pages", ctypes.c_int), ("block_table", P),
                ("table_width", ctypes.c_int), ("out", P)]


def _decode(**kw):
    a = DecodeArgs(dtype=F16, batch=8, n_heads=32, n_kv=8, head_dim=128, capacity=4096, scale=0.0884, qkv=0x1000, pos=0x2000,
                   rope_cos=0x3000, rope_sin=0x4000, k_pages=0x5000, v_pages=0x6000, n_pages=100, block_table=0x7004, table_width=64,
                   out=0x8000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _extend(**kw):
    a = ExtendArgs(dtype=F16, n_heads=32, n_kv=8, head_dim=128, capacity=4096, start=100, n_tokens=300, scale=0.0884, qkv=0x1000,
                   rope_cos=0x3000, rope_sin=0x4000, k_pages=0x5000, v_pages=0x6000, n_pages=100, block_table=0x7004, table_width=64,
                   out=0x8000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(fn, a):
    lib = load_lib()
    f = getattr(lib, fn)
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = f(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


PAGE_BAD = [
    (dict(n_pages=0), "n_pages=0 must be >= 1"),
    (dict(n_pages=-3), "n_pages=-3 must be >= 1"),
    (dict(table_width=63), "table_width=63 must be ceil(capacity=4096 / 64) = 64"),
    (dict(table_width=65), "table_width=65 must be ceil(capacity=4096 / 64) = 64"),
    (dict(capacity=4097), "table_width=64 must be ceil(capacity=4097 / 64) = 65"),
    (dict(block_table=0), "block_table must be a non-null 4-byte aligned pointer"),
    (dict(block_table=0x7002), "block_table must be a non-null 4-byte aligned pointer"),
] + [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("k_pages", "v_pages") for v in (0, 0x5008)]
SHARED_BAD = [
    (dict(dtype=F32), "dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(n_heads=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (dict(head_dim=96), "head_dim=96 is not 64 or 128"),
    (dict(capacity=0), "capacity=0 must be >= 1"),
    (dict(scale=math.nan), "scale=nan must be finite and > 0"),
]
DECODE_BAD = SHARED_BAD + PAGE_BAD + [
    (dict(batch=0), "batch=0 must be in [1, 65535]"),
    (dict(batch=65536), "batch=65536 must be in [1, 65535]"),
] + [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("qkv", "pos", "rope_cos", "rope_sin", "out")
     for v in (0, 0x1008)]
EXTEND_BAD = SHARED_BAD + PAGE_BAD + [
    (dict(n_tokens=0), "n_tokens=0 must be >= 1"),
    (dict(start=-1), "start=-1 must be >= 0"),
    (dict(start=4000, n_tokens=97), "start=4000 + n_tokens=97 must be <= capacity=4096"),
] + [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("qkv", "rope_cos", "rope_sin", "out")
     for v in (0, 0x1008)]


def _id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


@pytest.mark.parametrize("change,frag", DECODE_BAD, ids=[_id(c) for c, _ in DECODE_BAD])
def test_decode_rejects(change, frag):
    rc, msg = _call("sqllm_attn_decode_paged", _decode(**change))
    assert rc != 0 and frag in msg, msg


@pytest.mark.parametrize("change,frag", EXTEND_BAD, ids=[_id(c) for c, _ in EXTEND_BAD])
def test_extend_rejects(change, frag):
    rc, msg = _call("sqllm_attn_extend_paged", _extend(**change))
    assert rc != 0 and frag in msg, msg


@pytest.mark.parametrize("fn", ["sqllm_attn_decode_paged", "sqllm_attn_extend_paged"])
def test_null_args(fn):
    rc, msg = _call(fn, None)
    assert rc != 0 and "null args" in msg


def test_header_lists_the_symbols_and_the_abi_stays_4():
    syms = header_symbols()
    for s in ("sqllm_attn_decode_paged", "sqllm_attn_extend_paged"):
        assert s in syms
    later = re.search(r"later \+(.*?)\*/", open(HEADER).read(), re.S).group(1)
    assert "sqllm_attn_decode_paged" in later and "sqllm_attn_extend_paged" in later
    from squeezellm_b200.quant import quant_cuda
    assert quant_cuda.abi_version() == 4


# the bindings, on CPU tensors: every rejection below comes before the device checks
NH, NKV, D, CAP, NP, B = 8, 2, 64, 200, 6, 3
W = (CAP + 63) // 64


def _t(*shape, dt=torch.float16):
    return torch.zeros(*shape, dtype=dt)


def _decode_inputs(**kw):
    a = dict(qkv=_t(B, (NH + 2 * NKV) * D), pos=_t(B, dt=torch.int32), rope_cos=_t(CAP, D // 2, dt=torch.float32),
             rope_sin=_t(CAP, D // 2, dt=torch.float32), k_pages=_t(NP, NKV, 64, D), v_pages=_t(NP, NKV, 64, D),
             block_table=_t(B, W, dt=torch.int32), out=_t(B, NH * D), n_heads=NH, n_kv=NKV, scale=0.125)
    a.update(kw)
    return a


def _extend_inputs(**kw):
    a = dict(qkv=_t(5, (NH + 2 * NKV) * D), start=10, rope_cos=_t(CAP, D // 2, dt=torch.float32),
             rope_sin=_t(CAP, D // 2, dt=torch.float32), k_pages=_t(NP, NKV, 64, D), v_pages=_t(NP, NKV, 64, D),
             block_table_row=_t(W, dt=torch.int32), out=_t(5, NH * D), n_heads=NH, n_kv=NKV, scale=0.125)
    a.update(kw)
    return a


BIND_BAD = [
    (dict(k_pages=_t(NP, NKV, 32, D)), "k_pages must be [n_pages, n_kv=2, 64, head_dim]"),
    (dict(k_pages=_t(NP, 4, 64, D)), "k_pages must be [n_pages, n_kv=2, 64, head_dim]"),
    (dict(k_pages=_t(NKV, 64, D)), "k_pages must be [n_pages, n_kv=2, 64, head_dim]"),
    (dict(k_pages=_t(0, NKV, 64, D), v_pages=_t(0, NKV, 64, D)), "k_pages must be [n_pages"),
    (dict(v_pages=_t(NP + 1, NKV, 64, D)), "v_cache must have k_cache's shape"),
    (dict(k_pages=_t(NP, NKV, 64, 96), v_pages=_t(NP, NKV, 64, 96)), "head_dim=96 is not 64 or 128"),
    (dict(scale=0.0), "scale=0 must be finite and > 0"),
]


@pytest.mark.parametrize("change,frag", BIND_BAD + [
    (dict(block_table=_t(B, W + 1, dt=torch.int32)), "block_table must be [batch, ceil(capacity=200 / 64)=4]"),
    (dict(block_table=_t(B * W, dt=torch.int32)), "block_table must be [batch, ceil(capacity=200 / 64)=4]"),
    (dict(block_table=_t(B, W, dt=torch.int64)), "block_table must be a contiguous int32 tensor"),
    (dict(block_table=_t(W, B, dt=torch.int32).t()), "block_table must be a contiguous int32 tensor"),
    (dict(block_table=_t(B * W + 1, dt=torch.int32)[1:].view(B, W)), None),   # 4-byte aligned is enough: on to the device check
    (dict(pos=_t(B + 1, dt=torch.int32)), "pos must be int32 [batch=3]"),
    (dict(qkv=_t(B + 1, (NH + 2 * NKV) * D)), "qkv must be [batch=3"),
])
def test_decode_binding_rejects(change, frag):
    from squeezellm_b200.quant import quant_cuda
    with pytest.raises(RuntimeError, match=re.escape(frag) if frag else "must be a CUDA tensor"):
        quant_cuda.attn_decode_paged(**_decode_inputs(**change))


@pytest.mark.parametrize("change,frag", BIND_BAD + [
    (dict(block_table_row=_t(W + 1, dt=torch.int32)), "block_table must be [ceil(capacity=200 / 64)=4]"),
    (dict(block_table_row=_t(B, W, dt=torch.int32)), "block_table must be [ceil(capacity=200 / 64)=4]"),
    (dict(block_table_row=_t(W, dt=torch.float32)), "block_table must be a contiguous int32 tensor"),
    (dict(start=196), "start=196 + T=5 must be <= capacity=200"),
    (dict(start=-1), "start=-1 must be >= 0"),
])
def test_extend_binding_rejects(change, frag):
    from squeezellm_b200.quant import quant_cuda
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        quant_cuda.attn_extend_paged(**_extend_inputs(**change))
