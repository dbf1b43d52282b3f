"""CPU tests of the argument checks of sqllm_attn_extend and quant_cuda.attn_extend: every bad argument is rejected (SQLLM_EINVAL, or
RuntimeError in Python) with a message naming the field, before anything touches a device; and the split rule of
sqllm_attn_extend_splits."""
import ctypes
import math
import re

import pytest

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


class ExtendArgs(ctypes.Structure):  # mirrors sqllm_attn_extend_args
    _fields_ = [("dtype", ctypes.c_int), ("n_heads", ctypes.c_int), ("n_kv", ctypes.c_int), ("head_dim", ctypes.c_int),
                ("capacity", ctypes.c_int), ("start", ctypes.c_int), ("n_tokens", ctypes.c_int), ("scale", ctypes.c_float),
                ("qkv", ctypes.c_void_p), ("rope_cos", ctypes.c_void_p), ("rope_sin", ctypes.c_void_p), ("k_cache", ctypes.c_void_p),
                ("v_cache", ctypes.c_void_p), ("out", ctypes.c_void_p)]


def _args(**kw):
    a = ExtendArgs(dtype=F16, n_heads=32, n_kv=8, head_dim=128, capacity=4096, start=100, n_tokens=300, scale=0.0884, qkv=0x1000,
                   rope_cos=0x3000, rope_sin=0x4000, k_cache=0x5000, v_cache=0x6000, out=0x7000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a):
    lib = load_lib()
    lib.sqllm_attn_extend.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_attn_extend(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


BAD = [
    (dict(dtype=F32), "dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(dtype=3), "dtype=3 is not SQLLM_DT_F16 or SQLLM_DT_BF16"),
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
    (dict(n_tokens=0), "n_tokens=0 must be >= 1"),
    (dict(n_tokens=-3), "n_tokens=-3 must be >= 1"),
    (dict(start=-1), "start=-1 must be >= 0"),
    (dict(start=3797), "start=3797 + n_tokens=300 must be <= capacity=4096"),
    (dict(start=2**31 - 100, n_tokens=200, capacity=2**31 - 1), "start=2147483548 + n_tokens=200 must be <= capacity=2147483647"),
    (dict(start=0, n_tokens=1048561, n_heads=32, n_kv=8, capacity=2**31 - 1), "needs more than 65535 query tiles of 64"),
    (dict(n_heads=70000, n_kv=70000), "n_kv=70000 > 65535"),
] + [(dict(**{f: 0}), f"{f} must be a non-null 16-byte aligned pointer")
     for f in ("qkv", "rope_cos", "rope_sin", "k_cache", "v_cache", "out")] \
  + [(dict(**{f: 0x1008}), f"{f} must be a non-null 16-byte aligned pointer")
     for f in ("qkv", "rope_cos", "rope_sin", "k_cache", "v_cache", "out")]


@pytest.mark.parametrize("change,frag", BAD, ids=[f"{next(iter(c))}={next(iter(c.values()))}" for c, _ in BAD])
def test_rejects(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


def test_rejects_null_args():
    rc, msg = _call(None)
    assert rc == -1 and "null args" in msg


def test_largest_grid_passes_the_checks():
    """64 * 65535 rows of one group is the last chunk the grid holds: the tile check passes and the pointer checks after it reject the
    (deliberately misaligned) out; one token more is rejected by the tile check."""
    rc, msg = _call(_args(start=0, n_tokens=64 * 65535 // 4, n_heads=32, n_kv=8, capacity=2**31 - 1, out=0x1008))
    assert rc == -1 and "out must be a non-null 16-byte aligned pointer" in msg, msg
    rc, msg = _call(_args(start=0, n_tokens=64 * 65535 // 4 + 1, n_heads=32, n_kv=8, capacity=2**31 - 1))
    assert rc == -1 and "query tiles" in msg


# max(1, min(8, SMs / (n_kv ceil(T g / 64)), ceil((start + T) / 64))), 0 for invalid arguments
@pytest.mark.parametrize("nh,nkv,T,start,sm,want", [
    (32, 8, 8, 4000, 132, 8),      # 8 tiles, 63 key blocks: 8 CTAs per tile
    (32, 8, 1, 0, 132, 1),         # one key block
    (32, 8, 1, 64, 132, 2),        # two key blocks
    (32, 32, 17, 0, 132, 1),       # 32 tiles, one block
    (32, 32, 64, 64, 132, 2),      # 32 tiles, 2 blocks
    (32, 32, 300, 100, 132, 1),    # 160 tiles fill the SMs
    (8, 2, 300, 100, 132, 3),      # 2 x 19 tiles: 132 / 38 = 3
    (4, 4, 5, 4091, 132, 8),
    (4, 4, 2048, 0, 132, 1),       # 128 tiles: 132 / 128 = 1
    (32, 8, 2048, 0, 132, 1),      # 1024 tiles fill the SMs
    (32, 8, 64, 4096, 132, 4),     # 32 tiles: 132 / 32 = 4
    (32, 8, 64, 4096, 66, 2),      # on 66 SMs: 66 / 32 = 2
    (128, 2, 1, 0, 16, 1),
    (32, 8, 0, 0, 132, 0), (32, 8, 8, -1, 132, 0), (30, 8, 8, 0, 132, 0), (8, 0, 8, 0, 132, 0), (8, 2, 8, 0, 0, 0),
    (8, 2, 100, 2**31 - 50, 132, 0), (32, 8, 1048561, 0, 132, 0)])
def test_splits(nh, nkv, T, start, sm, want):
    assert load_lib().sqllm_attn_extend_splits(nh, nkv, T, start, sm) == want


def test_declared_in_the_header_and_the_version_unchanged():
    assert {"sqllm_attn_extend", "sqllm_attn_extend_splits"} <= set(header_symbols())
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_attn_extend\(const sqllm_attn_extend_args \*args, void \*stream\);", txt)
    versions = txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert "sqllm_attn_extend" in versions and "sqllm_attn_extend_splits" in versions
    assert load_lib().sqllm_abi_version() == 4


# ---- the same through quant_cuda, on CPU tensors (the checks run before the device check) ----
torch = pytest.importorskip("torch")


def _tensors(T=5, nh=32, nkv=8, d=128, cap=64, dt=None):
    dt = dt or torch.float16
    return dict(qkv=torch.zeros(T, (nh + 2 * nkv) * d, dtype=dt), rope_cos=torch.zeros(cap, d // 2), rope_sin=torch.zeros(cap, d // 2),
                k_cache=torch.zeros(nkv, cap, d, dtype=dt), v_cache=torch.zeros(nkv, cap, d, dtype=dt), out=torch.zeros(T, nh * d, dtype=dt))


def _module_call(nh=32, nkv=8, scale=0.0884, start=3, **t):
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.attn_extend(t["qkv"], start, t["rope_cos"], t["rope_sin"], t["k_cache"], t["v_cache"], t["out"], nh, nkv, scale)


MODULE_BAD = [
    (lambda: _tensors(dt=torch.float32), {}, "dtype of qkv must be torch.float16 or torch.bfloat16"),
    (lambda: _tensors(), dict(nh=30), "n_heads=30 must be a positive multiple of n_kv=8"),
    (lambda: _tensors(), dict(nkv=0), "n_heads=32 must be a positive multiple of n_kv=0"),
    (lambda: _tensors(nh=8, nkv=2, d=96), dict(nh=8, nkv=2), "head_dim=96 is not 64 or 128"),
    (lambda: _tensors(cap=0), {}, "capacity=0 must be >= 1"),
    (lambda: _tensors(), dict(scale=0.0), "scale=0 must be finite and > 0"),
    (lambda: _tensors(), dict(scale=math.inf), "scale=inf must be finite and > 0"),
    (lambda: _tensors(), dict(scale=math.nan), "scale=nan must be finite and > 0"),
    (lambda: _tensors(), dict(scale=1e39), "must be finite and > 0"),
    (lambda: _tensors(T=0), {}, "qkv has no rows (T=0)"),
    (lambda: _tensors(), dict(start=-1), "start=-1 must be >= 0"),
    (lambda: _tensors(), dict(start=60), "start=60 + T=5 must be <= capacity=64"),
    (lambda: dict(_tensors(), qkv=torch.zeros(5 * 48 * 128 + 1, dtype=torch.float16)[1:].view(5, 48 * 128)), {},
     "qkv must be 16-byte aligned"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(8, 128, 64, dtype=torch.float16).transpose(1, 2)), {},
     "k_cache must be a contiguous tensor"),
    (lambda: dict(_tensors(), k_cache=torch.zeros(4, 64, 128, dtype=torch.float16)), {}, "k_cache must be [n_kv=8"),
    (lambda: dict(_tensors(), v_cache=torch.zeros(8, 32, 128, dtype=torch.float16)), {}, "v_cache must have k_cache's shape"),
    (lambda: dict(_tensors(), qkv=torch.zeros(5 * 48 * 128, dtype=torch.float16)), {}, "qkv must be [T, (n_heads + 2 n_kv) head_dim=6144]"),
    (lambda: dict(_tensors(), qkv=torch.zeros(5, 48 * 128 + 8, dtype=torch.float16)), {}, "qkv must be [T, (n_heads + 2 n_kv) head_dim=6144]"),
    (lambda: dict(_tensors(), out=torch.zeros(5, 32 * 128 + 8, dtype=torch.float16)), {}, "out must be [T=5"),
    (lambda: dict(_tensors(), out=torch.zeros(4, 32 * 128, dtype=torch.float16)), {}, "out must be [T=5"),
    (lambda: dict(_tensors(), out=torch.zeros(5, 32 * 128, dtype=torch.bfloat16)), {}, "k_cache, v_cache and out must have qkv's dtype"),
    (lambda: dict(_tensors(), rope_sin=torch.zeros(64, 128)), {}, "rope_cos / rope_sin must be fp32 [capacity=64, head_dim/2=64]"),
    (lambda: _tensors(), {}, "qkv must be a CUDA tensor"),
]


@pytest.mark.parametrize("make,kw,frag", MODULE_BAD, ids=[str(i) for i in range(len(MODULE_BAD))])
def test_module_rejects(make, kw, frag):
    with pytest.raises(RuntimeError, match=re.escape(frag)):
        _module_call(**kw, **make())
