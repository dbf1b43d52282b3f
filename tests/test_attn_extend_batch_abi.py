"""CPU tests of the argument checks of sqllm_attn_extend_batch / sqllm_attn_extend_batch_paged and of their quant_cuda bindings: every
bad argument is rejected (SQLLM_EINVAL, or RuntimeError in Python) with a message naming the field, before anything touches a device."""
import ctypes
import math
import re

import pytest
import torch

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2
P = ctypes.c_void_p
I32P = ctypes.POINTER(ctypes.c_int32)

COMMON = [("dtype", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int), ("head_dim", ctypes.c_int),
          ("capacity", ctypes.c_int), ("scale", ctypes.c_float), ("n_segments", ctypes.c_int), ("slots", I32P), ("starts", I32P),
          ("n_tokens", I32P), ("n_slots", ctypes.c_int), ("qkv", P), ("rope_cos", P), ("rope_sin", P)]


class BatchArgs(ctypes.Structure):  # mirrors sqllm_attn_extend_batch_args
    _fields_ = COMMON + [("k_cache", P), ("v_cache", P), ("out", P)]


class PagedArgs(ctypes.Structure):  # mirrors sqllm_attn_extend_batch_paged_args
    _fields_ = COMMON + [("k_pages", P), ("v_pages", P), ("n_pages", ctypes.c_int), ("block_table", P), ("table_width", ctypes.c_int),
                         ("out", P)]


def _ints(v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def _args(paged, slots=(3, 0, 5), starts=(100, 0, 4000), n_tokens=(300, 17, 8), **kw):
    keep = [_ints(slots), _ints(starts), _ints(n_tokens)]
    common = dict(dtype=F16, n_heads=32, n_kv=8, head_dim=128, capacity=4096, scale=0.0884, n_segments=len(slots),
                  slots=ctypes.cast(keep[0], I32P), starts=ctypes.cast(keep[1], I32P), n_tokens=ctypes.cast(keep[2], I32P), n_slots=8,
                  qkv=0x1000, rope_cos=0x3000, rope_sin=0x4000, out=0x8000)
    if paged:
        a = PagedArgs(k_pages=0x5000, v_pages=0x6000, n_pages=100, block_table=0x7004, table_width=64, **common)
    else:
        a = BatchArgs(k_cache=0x5000, v_cache=0x6000, **common)
    for k, v in kw.items():
        setattr(a, k, v)
    a._keep = keep
    return a


def _call(fn, a):
    lib = load_lib()
    f = getattr(lib, fn)
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = f(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


NULL = ctypes.cast(None, I32P)
SEGMENT_BAD = [
    (dict(n_segments=0), "n_segments=0 must be in [1, 128]"),
    (dict(slots=list(range(129)), starts=[0] * 129, n_tokens=[1] * 129, n_slots=200), "n_segments=129 must be in [1, 128]"),
    (dict(n_slots=0), "n_slots=0 must be >= 1"),
    (dict(slots=(3, 8, 5)), "slots[1]=8 must be in [0, n_slots=8)"),
    (dict(slots=(3, -1, 5)), "slots[1]=-1 must be in [0, n_slots=8)"),
    (dict(slots=(3, 0, 3)), "slots[2]=3 repeats slots[0]"),
    (dict(n_tokens=(300, 0, 8)), "n_tokens[1]=0 must be >= 1"),
    (dict(starts=(100, -1, 4000)), "starts[1]=-1 must be >= 0"),
    (dict(starts=(100, 0, 4089)), "starts[2]=4089 + n_tokens[2]=8 must be <= capacity=4096"),
    # 2 x 4096 tokens x 1024 heads per KV head = 131072 tiles of 64 rows; each segment alone would fit
    (dict(n_heads=1024, n_kv=1, capacity=8192, slots=(0, 1), starts=(0, 4096), n_tokens=(4096, 4096)),
     "the segments need 131072 query tiles of 64 per KV head, more than 65535"),
]
SHARED_BAD = [
    (dict(dtype=F32), "dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(n_heads=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (dict(head_dim=96), "head_dim=96 is not 64 or 128"),
    (dict(capacity=0), "capacity=0 must be >= 1"),
    (dict(scale=math.nan), "scale=nan must be finite and > 0"),
]
PTR_BAD = [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("qkv", "rope_cos", "rope_sin", "out")
           for v in (0, 0x1008)]
CACHE_BAD = [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("k_cache", "v_cache") for v in (0, 0x5008)]
PAGE_BAD = [
    (dict(n_pages=0), "n_pages=0 must be >= 1"),
    (dict(table_width=63), "table_width=63 must be ceil(capacity=4096 / 64) = 64"),
    (dict(capacity=4097), "table_width=64 must be ceil(capacity=4097 / 64) = 65"),
    (dict(block_table=0), "block_table must be a non-null 4-byte aligned pointer"),
    (dict(block_table=0x7002), "block_table must be a non-null 4-byte aligned pointer"),
] + [(dict(**{f: v}), f"{f} must be a non-null 16-byte aligned pointer") for f in ("k_pages", "v_pages") for v in (0, 0x5008)]


def _id(c):
    return "-".join(f"{k}={v if not isinstance(v, (list, tuple)) or len(v) < 5 else len(v)}" for k, v in c.items())


def _build(paged, change):
    lists = {k: change[k] for k in ("slots", "starts", "n_tokens") if k in change}
    rest = {k: v for k, v in change.items() if k not in lists}
    return _args(paged, **lists, **rest)


@pytest.mark.parametrize("change,frag", SEGMENT_BAD + SHARED_BAD + PTR_BAD + CACHE_BAD, ids=lambda x: _id(x) if isinstance(x, dict) else None)
def test_batch_rejects(change, frag):
    rc, msg = _call("sqllm_attn_extend_batch", _build(False, change))
    assert rc != 0 and frag in msg, msg


@pytest.mark.parametrize("change,frag", SEGMENT_BAD + SHARED_BAD + PTR_BAD + PAGE_BAD, ids=lambda x: _id(x) if isinstance(x, dict) else None)
def test_batch_paged_rejects(change, frag):
    rc, msg = _call("sqllm_attn_extend_batch_paged", _build(True, change))
    assert rc != 0 and frag in msg, msg


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("field", ["slots", "starts", "n_tokens"])
def test_null_lists(paged, field):
    a = _args(paged)
    setattr(a, field, NULL)
    rc, msg = _call("sqllm_attn_extend_batch_paged" if paged else "sqllm_attn_extend_batch", a)
    assert rc != 0 and "slots, starts and n_tokens must be non-null host arrays" in msg, msg


@pytest.mark.parametrize("fn", ["sqllm_attn_extend_batch", "sqllm_attn_extend_batch_paged"])
def test_null_args(fn):
    rc, msg = _call(fn, None)
    assert rc != 0 and "null args" in msg


def test_header_lists_the_symbols_and_the_abi_stays_4():
    syms = header_symbols()
    for s in ("sqllm_attn_extend_batch", "sqllm_attn_extend_batch_paged"):
        assert s in syms
    text = open(HEADER).read()
    later = re.search(r"later \+(.*?)\*/", text, re.S).group(1)
    assert "sqllm_attn_extend_batch," in later and "sqllm_attn_extend_batch_paged" in later
    assert re.search(r"#define SQLLM_ATTN_EXTEND_MAX_SEGMENTS 128\b", text)
    from squeezellm_b200.quant import quant_cuda
    assert quant_cuda.abi_version() == 4


# the bindings, on CPU tensors: every rejection below comes before the device checks
NH, NKV, D, CAP, NP, NS = 8, 2, 64, 200, 6, 4
W = (CAP + 63) // 64


def _t(*shape, dt=torch.float16):
    return torch.zeros(*shape, dtype=dt)


def _inputs(paged, rows=7, **kw):
    a = dict(qkv=_t(rows, (NH + 2 * NKV) * D), slots=[2, 0], starts=[10, 0], n_tokens=[5, 2],
             rope_cos=_t(CAP, D // 2, dt=torch.float32), rope_sin=_t(CAP, D // 2, dt=torch.float32), out=_t(rows, NH * D), n_heads=NH,
             n_kv=NKV, scale=0.125)
    if paged:
        a.update(k_pages=_t(NP, NKV, 64, D), v_pages=_t(NP, NKV, 64, D), block_table=_t(NS, W, dt=torch.int32))
    else:
        a.update(k_cache=_t(NS, NKV, CAP, D), v_cache=_t(NS, NKV, CAP, D))
    a.update(kw)
    return a


BIND_SEGMENT_BAD = [
    (dict(slots=[], starts=[], n_tokens=[]), "n_segments=0 must be in [1, 128]"),
    (dict(slots=list(range(129)), starts=[0] * 129, n_tokens=[1] * 129), "n_segments=129 must be in [1, 128]"),
    (dict(starts=[10]), "slots, starts and n_tokens must have one length"),
    (dict(n_tokens=[5, 2, 1]), "slots, starts and n_tokens must have one length"),
    (dict(slots=[2, 4]), "slots[1]=4 must be in [0, n_slots=4)"),
    (dict(slots=[-1, 0]), "slots[0]=-1 must be in [0, n_slots=4)"),
    (dict(slots=[2, 2]), "slots[1]=2 repeats slots[0]"),
    (dict(n_tokens=[7, 0]), "n_tokens[1]=0 must be >= 1"),
    (dict(starts=[-1, 0]), "starts[0]=-1 must be >= 0"),
    (dict(starts=[196, 0]), "starts[0]=196 + n_tokens[0]=5 must be <= capacity=200"),
    (dict(qkv=_t(8, (NH + 2 * NKV) * D)), "qkv must be [sum n_tokens=7"),
    (dict(out=_t(8, NH * D)), "out must be [sum n_tokens=7"),
    (dict(scale=0.0), "scale=0 must be finite and > 0"),
]


def _many_tiles(paged):
    """2 segments of 2048 tokens x 1024 query heads of one KV head: 32768 query tiles each, 65536 together.  The tile check comes
    before the shapes of qkv and out, so they stay small."""
    nh, d, cap = 1024, 64, 2048
    pool = (dict(k_pages=_t(2, 1, 64, d), v_pages=_t(2, 1, 64, d), block_table=_t(2, cap // 64, dt=torch.int32)) if paged
            else dict(k_cache=_t(2, 1, cap, d), v_cache=_t(2, 1, cap, d)))
    return dict(qkv=_t(1, 8), slots=[0, 1], starts=[0, 0], n_tokens=[2048, 2048], rope_cos=_t(cap, d // 2, dt=torch.float32),
                rope_sin=_t(cap, d // 2, dt=torch.float32), out=_t(1, 8), n_heads=nh, n_kv=1, scale=0.125, **pool)


@pytest.mark.parametrize("change,frag", BIND_SEGMENT_BAD + [
    (dict(k_cache=_t(NKV, CAP, D)), "k_cache must be [batch, n_kv=2, capacity, head_dim]"),
    (dict(v_cache=_t(NS + 1, NKV, CAP, D)), "v_cache must have k_cache's shape"),
    (dict(k_cache=_t(NS, NKV, CAP, 96), v_cache=_t(NS, NKV, CAP, 96)), "head_dim=96 is not 64 or 128"),
    (dict(qkv=_t(7, (NH + 2 * NKV) * D, dt=torch.float32)), "dtype of qkv must be torch.float16 or torch.bfloat16"),
    (dict(k_cache=_t(NS, NKV, CAP, D + 8)[..., :D]), "k_cache must be a contiguous tensor"),
    (dict(qkv=torch.zeros(7 * (NH + 2 * NKV) * D + 1, dtype=torch.float16)[1:].view(7, -1)), "qkv must be 16-byte aligned"),
    ({}, "must be a CUDA tensor"),
])
def test_batch_binding_rejects(change, frag):
    from squeezellm_b200.quant import quant_cuda
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        quant_cuda.attn_extend_batch(**_inputs(False, **change))


@pytest.mark.parametrize("change,frag", BIND_SEGMENT_BAD + [
    (dict(k_pages=_t(NP, NKV, 32, D)), "k_pages must be [n_pages, n_kv=2, 64, head_dim]"),
    (dict(v_pages=_t(NP + 1, NKV, 64, D)), "v_cache must have k_cache's shape"),
    (dict(block_table=_t(NS, W + 1, dt=torch.int32)), "block_table must be [batch, ceil(capacity=200 / 64)=4]"),
    (dict(block_table=_t(NS * W, dt=torch.int32)), "block_table must be [batch, ceil(capacity=200 / 64)=4]"),
    (dict(block_table=_t(NS, W, dt=torch.int64)), "block_table must be a contiguous int32 tensor"),
    (dict(slots=[2, 4]), "slots[1]=4 must be in [0, n_slots=4)"),
    ({}, "must be a CUDA tensor"),
])
def test_batch_paged_binding_rejects(change, frag):
    from squeezellm_b200.quant import quant_cuda
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        quant_cuda.attn_extend_batch_paged(**_inputs(True, **change))


@pytest.mark.parametrize("paged", [False, True])
def test_binding_rejects_too_many_tiles(paged):
    from squeezellm_b200.quant import quant_cuda
    fn = quant_cuda.attn_extend_batch_paged if paged else quant_cuda.attn_extend_batch
    with pytest.raises(RuntimeError, match=re.escape("the segments need 65536 query tiles of 64 per KV head, more than 65535")):
        fn(**_many_tiles(paged))
