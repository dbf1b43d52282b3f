"""CPU tests of the argument checks of sqllm_attn_decode_batch and quant_cuda.attn_decode_batch: every bad argument is rejected
(SQLLM_EINVAL, or RuntimeError in Python) with a message naming the field, before anything touches a device; and the split rule of
sqllm_attn_decode_batch_splits."""
import ctypes
import math
import re

import pytest

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


class BatchArgs(ctypes.Structure):  # mirrors sqllm_attn_decode_batch_args
    _fields_ = [("dtype", ctypes.c_int), ("batch", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int),
                ("head_dim", ctypes.c_int), ("capacity", ctypes.c_int), ("scale", ctypes.c_float), ("qkv", ctypes.c_void_p),
                ("pos", ctypes.c_void_p), ("rope_cos", ctypes.c_void_p), ("rope_sin", ctypes.c_void_p), ("k_cache", ctypes.c_void_p),
                ("v_cache", ctypes.c_void_p), ("out", ctypes.c_void_p)]


def _args(**kw):
    a = BatchArgs(dtype=F16, batch=8, n_heads=32, n_kv=8, head_dim=128, capacity=4096, scale=0.0884, qkv=0x1000, pos=0x2000,
                  rope_cos=0x3000, rope_sin=0x4000, k_cache=0x5000, v_cache=0x6000, out=0x7000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a):
    lib = load_lib()
    lib.sqllm_attn_decode_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_attn_decode_batch(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


BAD = [
    (dict(dtype=F32), "dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(dtype=3), "dtype=3 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(batch=0), "batch=0 must be in [1, 65535]"),
    (dict(batch=-2), "batch=-2 must be in [1, 65535]"),
    (dict(batch=65536), "batch=65536 must be in [1, 65535]"),
    (dict(n_heads=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (dict(n_kv=0), "n_heads=32 must be a positive multiple of n_kv=0"),
    (dict(n_heads=0), "n_heads=0 must be a positive multiple of n_kv=8"),
    (dict(n_heads=4), "n_heads=4 must be a positive multiple of n_kv=8"),
    (dict(head_dim=96), "head_dim=96 is not 64 or 128"),
    (dict(capacity=0), "capacity=0 must be >= 1"),
    (dict(capacity=-5), "capacity=-5 must be >= 1"),
    (dict(scale=0.0), "scale=0 must be finite and > 0"),
    (dict(scale=-0.1), "must be finite and > 0"),
    (dict(scale=math.inf), "scale=inf must be finite and > 0"),
    (dict(scale=math.nan), "scale=nan must be finite and > 0"),
] + [(dict(**{f: 0}), f"{f} must be a non-null 16-byte aligned pointer")
     for f in ("qkv", "pos", "rope_cos", "rope_sin", "k_cache", "v_cache", "out")] \
  + [(dict(**{f: 0x1008}), f"{f} must be a non-null 16-byte aligned pointer")
     for f in ("qkv", "pos", "rope_cos", "rope_sin", "k_cache", "v_cache", "out")]


@pytest.mark.parametrize("change,frag", BAD, ids=[f"{next(iter(c))}={next(iter(c.values()))}" for c, _ in BAD])
def test_rejects(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


def test_rejects_null_args():
    rc, msg = _call(None)
    assert rc == -1 and "null args" in msg


# min(8, max(1, SMs / (batch n_kv ceil(n_heads / n_kv / 8)))), 0 for invalid arguments
@pytest.mark.parametrize("nh,nkv,B,sm,want", [(32, 32, 1, 132, 4), (32, 32, 2, 132, 2), (32, 32, 8, 132, 1), (32, 8, 2, 132, 8),
                                              (32, 8, 4, 132, 4), (32, 8, 16, 132, 1), (8, 2, 5, 132, 8), (8, 2, 63, 132, 1),
                                              (4, 4, 8, 132, 4), (64, 8, 2, 132, 8), (128, 2, 1, 132, 8), (128, 2, 4, 132, 2), (128, 2, 8, 132, 1),
                                              (32, 32, 65535, 132, 1), (32, 32, 0, 132, 0), (32, 32, 65536, 132, 0),
                                              (30, 8, 2, 132, 0), (8, 0, 2, 132, 0), (8, 2, 2, 0, 0),
                                              (71, 1, 5, 132, 2),   # ceil(71 / 8) = 9 clusters per sequence, 45 in all: 132 / 45 = 2
                                              (48, 4, 4, 132, 4)])  # B 4 x n_kv 4 x ceil(12 / 8) = 32 clusters: 132 / 32 = 4
def test_splits(nh, nkv, B, sm, want):
    assert load_lib().sqllm_attn_decode_batch_splits(nh, nkv, B, sm) == want


@pytest.mark.parametrize("nh,nkv", [(32, 32), (32, 8), (8, 2), (4, 4), (128, 2)])
def test_batch_one_splits_like_the_single_row_kernel(nh, nkv):
    lib = load_lib()
    for sm in (16, 66, 132):
        assert lib.sqllm_attn_decode_batch_splits(nh, nkv, 1, sm) == lib.sqllm_attn_decode_splits(nh, nkv, sm)


def test_declared_in_the_header_and_the_version_unchanged():
    assert {"sqllm_attn_decode_batch", "sqllm_attn_decode_batch_splits"} <= set(header_symbols())
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_attn_decode_batch\(const sqllm_attn_decode_batch_args \*args, void \*stream\);", txt)
    versions = txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert "sqllm_attn_decode_batch" in versions and "sqllm_attn_decode_batch_splits" in versions
    assert load_lib().sqllm_abi_version() == 4


# ---- the same through quant_cuda, on CPU tensors (the checks run before the device check) ----
torch = pytest.importorskip("torch")


def _tensors(B=4, nh=32, nkv=8, d=128, cap=64, dt=None):
    dt = dt or torch.float16
    return dict(qkv=torch.zeros(B, (nh + 2 * nkv) * d, dtype=dt), pos=torch.zeros(B, dtype=torch.int32),
                rope_cos=torch.zeros(cap, d // 2), rope_sin=torch.zeros(cap, d // 2), k_cache=torch.zeros(B, nkv, cap, d, dtype=dt),
                v_cache=torch.zeros(B, nkv, cap, d, dtype=dt), out=torch.zeros(B, nh * d, dtype=dt))


def _module_call(nh=32, nkv=8, scale=0.0884, **t):
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.attn_decode_batch(t["qkv"], t["pos"], t["rope_cos"], t["rope_sin"], t["k_cache"], t["v_cache"], t["out"], nh, nkv, scale)


MODULE_BAD = [
    (lambda: _tensors(dt=torch.float32), {}, "dtype of qkv must be torch.float16 or torch.bfloat16"),
    (lambda: _tensors(), dict(nh=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (lambda: _tensors(), dict(nkv=0), "n_heads=32 must be a positive multiple of n_kv=0"),
    (lambda: _tensors(nh=8, nkv=2, d=96), dict(nh=8, nkv=2), "head_dim=96 is not 64 or 128"),
    (lambda: _tensors(cap=0), {}, "capacity=0 must be >= 1"),
    (lambda: _tensors(B=0), {}, "batch=0 must be in [1, 65535]"),
    (lambda: _tensors(), dict(scale=0.0), "scale=0 must be finite and > 0"),
    (lambda: _tensors(), dict(scale=math.inf), "scale=inf must be finite and > 0"),
    (lambda: _tensors(), dict(scale=math.nan), "scale=nan must be finite and > 0"),
    (lambda: _tensors(), dict(scale=1e39), "must be finite and > 0"),
    (lambda: dict(_tensors(), qkv=torch.zeros(4 * 48 * 128 + 1, dtype=torch.float16)[1:].view(4, 48 * 128)), {},
     "qkv must be 16-byte aligned"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(4, 8, 128, 64, dtype=torch.float16).transpose(2, 3)), {},
     "k_cache must be a contiguous tensor"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(8, 64, 128, dtype=torch.float16)), {}, "k_cache must be [batch, n_kv=8"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(4, 4, 64, 128, dtype=torch.float16)), {}, "k_cache must be [batch, n_kv=8"),
    (lambda: dict(_tensors(), v_cache=torch.zeros(4, 8, 32, 128, dtype=torch.float16)), {}, "v_cache must have k_cache's shape"),
    (lambda: dict(_tensors(), qkv=torch.zeros(3, 48 * 128, dtype=torch.float16)), {}, "qkv must be [batch=4"),
    (lambda: dict(_tensors(), qkv=torch.zeros(4 * 48 * 128, dtype=torch.float16)), {}, "qkv must be [batch=4"),
    (lambda: dict(_tensors(), out=torch.zeros(4, 32 * 128 + 8, dtype=torch.float16)), {}, "out must be [batch=4"),
    (lambda: dict(_tensors(), out=torch.zeros(5, 32 * 128, dtype=torch.float16)), {}, "out must be [batch=4"),
    (lambda: dict(_tensors(), pos=torch.zeros(4, dtype=torch.int64)), {}, "pos must be int32 [batch=4]"),
    (lambda: dict(_tensors(), pos=torch.zeros(3, dtype=torch.int32)), {}, "pos must be int32 [batch=4]"),
    (lambda: dict(_tensors(), rope_sin=torch.zeros(64, 128)), {}, "rope_cos / rope_sin must be fp32 [capacity=64, head_dim/2=64]"),
    (lambda: _tensors(), {}, "qkv must be a CUDA tensor"),
]


@pytest.mark.parametrize("make,kw,frag", MODULE_BAD, ids=[str(i) for i in range(len(MODULE_BAD))])
def test_module_rejects(make, kw, frag):
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        _module_call(**kw, **make())
