"""CPU tests of the argument checks of sqllm_attn_verify and quant_cuda.attn_verify: every bad argument is rejected (SQLLM_EINVAL, or
RuntimeError in Python) with a message naming the field, before anything touches a device; the split rule; the header entries."""
import ctypes
import math
import re

import pytest

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


class VerifyArgs(ctypes.Structure):  # mirrors sqllm_attn_verify_args
    _fields_ = [("dtype", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int), ("head_dim", ctypes.c_int),
                ("capacity", ctypes.c_int), ("n_tokens", ctypes.c_int), ("scale", ctypes.c_float), ("qkv", ctypes.c_void_p),
                ("pos", ctypes.c_void_p), ("rope_cos", ctypes.c_void_p), ("rope_sin", ctypes.c_void_p), ("k_cache", ctypes.c_void_p),
                ("v_cache", ctypes.c_void_p), ("out", ctypes.c_void_p)]


def _args(**kw):
    a = VerifyArgs(dtype=F16, n_heads=32, n_kv=8, head_dim=128, capacity=4096, n_tokens=4, scale=0.0884, qkv=0x1000, pos=0x2000,
                   rope_cos=0x3000, rope_sin=0x4000, k_cache=0x5000, v_cache=0x6000, out=0x7000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a):
    lib = load_lib()
    lib.sqllm_attn_verify.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_attn_verify(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


BAD = [
    (dict(dtype=F32), "dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(dtype=3), "dtype=3 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(n_heads=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (dict(n_kv=0), "n_heads=32 must be a positive multiple of n_kv=0"),
    (dict(n_heads=4), "n_heads=4 must be a positive multiple of n_kv=8"),
    (dict(head_dim=96), "head_dim=96 is not 64 or 128"),
    (dict(capacity=0), "capacity=0 must be >= 1"),
    (dict(scale=0.0), "scale=0 must be finite and > 0"),
    (dict(scale=math.nan), "scale=nan must be finite and > 0"),
    (dict(n_tokens=0), "n_tokens=0 must be in [1, 16]"),
    (dict(n_tokens=17), "n_tokens=17 must be in [1, 16]"),
    (dict(n_tokens=-2), "n_tokens=-2 must be in [1, 16]"),
    (dict(n_heads=65536, n_kv=65536), "n_kv=65536 x 1 clusters per KV head exceeds 65535"),
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


@pytest.mark.parametrize("nh,nkv,T,sm,want", [
    (32, 32, 8, 132, 4),     # 32 clusters (one chunk of 8 rows per KV head)
    (32, 32, 16, 132, 2),    # 64 clusters
    (32, 8, 8, 132, 4),      # 8 x ceil(32 / 8)
    (32, 8, 16, 132, 2),     # 8 x 8
    (8, 2, 1, 132, 8), (4, 4, 16, 132, 8), (4, 4, 2, 132, 8),
    (64, 8, 16, 132, 1),     # 8 x 16 clusters
    (32, 32, 1, 16, 1),
    (71, 1, 16, 132, 1),     # 1 x ceil(16 x 71 / 8) = 142 clusters: 132 / 142 = 0, at least 1
    (28, 4, 3, 132, 8),      # 4 x ceil(3 x 7 / 8) = 12 clusters: 132 / 12 = 11, at most 8
    (30, 8, 4, 132, 0), (8, 0, 4, 132, 0), (8, 2, 4, 0, 0), (8, 2, 0, 132, 0), (8, 2, 17, 132, 0), (65536, 65536, 1, 132, 0),
])
def test_splits(nh, nkv, T, sm, want):
    assert load_lib().sqllm_attn_verify_splits(nh, nkv, T, sm) == want


@pytest.mark.parametrize("nh,nkv", [(32, 32), (32, 8), (8, 2), (4, 4), (64, 8), (128, 2)])
def test_one_token_splits_as_decode(nh, nkv):
    lib = load_lib()
    assert lib.sqllm_attn_verify_splits(nh, nkv, 1, 132) == lib.sqllm_attn_decode_splits(nh, nkv, 132)


@pytest.mark.parametrize("args", [(F32, 32, 8, 128, 4), (F16, 30, 8, 128, 4), (F16, 32, 8, 96, 4), (BF16, 32, 8, 128, 0),
                                  (BF16, 32, 8, 128, 17), (F16, 65536, 65536, 128, 1)])
def test_launch_splits_reject_what_the_launch_rejects(args):
    assert load_lib().sqllm_attn_verify_launch_splits(*args) == 0


def test_declared_in_the_header_and_the_version_unchanged():
    assert {"sqllm_attn_verify", "sqllm_attn_verify_splits", "sqllm_attn_verify_launch_splits"} <= set(header_symbols())
    assert re.search(r"int sqllm_attn_verify_launch_splits\(int dtype, int n_heads, int n_kv, int head_dim, int n_tokens\);",
                     open(HEADER).read())
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_attn_verify\(const sqllm_attn_verify_args \*args, void \*stream\);", txt)
    assert re.search(r"int sqllm_attn_verify_splits\(int n_heads, int n_kv, int n_tokens, int sm_count\);", txt)
    abi = txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert "sqllm_attn_verify," in abi and "sqllm_attn_verify_splits," in abi and "sqllm_attn_verify_launch_splits" in abi
    assert load_lib().sqllm_abi_version() == 4


# ---- the same through quant_cuda, on CPU tensors (the checks run before the device check) ----
torch = pytest.importorskip("torch")


def _tensors(nh=32, nkv=8, d=128, cap=64, T=4, dt=None):
    dt = dt or torch.float16
    return dict(qkv=torch.zeros(T, (nh + 2 * nkv) * d, dtype=dt), pos=torch.zeros(1, dtype=torch.int32),
                rope_cos=torch.zeros(cap, d // 2), rope_sin=torch.zeros(cap, d // 2), k_cache=torch.zeros(nkv, cap, d, dtype=dt),
                v_cache=torch.zeros(nkv, cap, d, dtype=dt), out=torch.zeros(T, nh * d, dtype=dt))


def _module_call(nh=32, nkv=8, scale=0.0884, **t):
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.attn_verify(t["qkv"], t["pos"], t["rope_cos"], t["rope_sin"], t["k_cache"], t["v_cache"], t["out"], nh, nkv, scale)


MODULE_BAD = [
    (lambda: _tensors(dt=torch.float32), {}, "attn_verify: dtype of qkv must be torch.float16 or torch.bfloat16"),
    (lambda: _tensors(), dict(nh=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (lambda: _tensors(nh=8, nkv=2, d=96), dict(nh=8, nkv=2), "head_dim=96 is not 64 or 128"),
    (lambda: _tensors(cap=0), {}, "capacity=0 must be >= 1"),
    (lambda: _tensors(), dict(scale=math.inf), "scale=inf must be finite and > 0"),
    (lambda: _tensors(T=17), {}, "attn_verify: qkv has 17 rows, want T in [1, 16]"),
    (lambda: _tensors(T=0), {}, "attn_verify: qkv has 0 rows, want T in [1, 16]"),
    (lambda: dict(_tensors(), qkv=torch.zeros(4 * 48 * 128, dtype=torch.float16)), {}, "attn_verify: qkv must be [T, (n_heads + 2 n_kv)"),
    (lambda: dict(_tensors(), qkv=torch.zeros(4, 48 * 128 + 8, dtype=torch.float16)), {}, "attn_verify: qkv must be [T,"),
    (lambda: dict(_tensors(), out=torch.zeros(3, 32 * 128, dtype=torch.float16)), {}, "attn_verify: out must be [T=4, n_heads head_dim=4096]"),
    (lambda: dict(_tensors(), out=torch.zeros(4 * 32 * 128, dtype=torch.float16)), {}, "attn_verify: out must be [T=4"),
    (lambda: dict(_tensors(), qkv=torch.zeros(4 * 48 * 128 + 1, dtype=torch.float16)[1:].view(4, -1)), {},
     "attn_verify: qkv must be 16-byte aligned"),
    (lambda: dict(_tensors(), qkv=torch.zeros(48 * 128, 4, dtype=torch.float16).t()), {}, "attn_verify: qkv must be a contiguous tensor"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(8, 128, 64, dtype=torch.float16).transpose(1, 2)), {},
     "k_cache must be a contiguous tensor"),
    (lambda: dict(_tensors(), v_cache=torch.zeros(8, 32, 128, dtype=torch.float16)), {}, "v_cache must have k_cache's shape"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(4, 64, 128, dtype=torch.float16)), {}, "k_cache must be [n_kv=8"),
    (lambda: dict(_tensors(), pos=torch.zeros(1, dtype=torch.int64)), {}, "attn_verify: pos must be one int32 element"),
    (lambda: dict(_tensors(), pos=torch.zeros(2, dtype=torch.int32)), {}, "attn_verify: pos must be one int32 element"),
    (lambda: dict(_tensors(), rope_sin=torch.zeros(64, 128)), {}, "rope_cos / rope_sin must be fp32 [capacity=64, head_dim/2=64]"),
    (lambda: _tensors(), {}, "attn_verify: qkv must be a CUDA tensor"),
]


@pytest.mark.parametrize("make,kw,frag", MODULE_BAD, ids=[str(i) for i in range(len(MODULE_BAD))])
def test_module_rejects(make, kw, frag):
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        _module_call(**kw, **make())
