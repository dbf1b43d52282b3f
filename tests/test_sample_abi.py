"""CPU tests of the argument checks of sqllm_sample and quant_cuda.sample: every bad argument is rejected (SQLLM_EINVAL, or RuntimeError
in Python) with a message naming the field, before anything touches a device."""
import ctypes
import re

import pytest

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


class SampleArgs(ctypes.Structure):  # mirrors sqllm_sample_args
    _fields_ = [("dtype", ctypes.c_int), ("rows", ctypes.c_int), ("vocab", ctypes.c_int), ("row_stride", ctypes.c_int64),
                ("logits", ctypes.c_void_p), ("pos", ctypes.c_void_p), ("temperature", ctypes.c_void_p), ("top_k", ctypes.c_void_p),
                ("top_p", ctypes.c_void_p), ("seed", ctypes.c_void_p), ("out", ctypes.c_void_p)]


def _args(**kw):
    a = SampleArgs(dtype=F16, rows=8, vocab=32000, row_stride=32000, logits=0x1000, pos=0x2000, temperature=0x3000, top_k=0x4000,
                   top_p=0x5000, seed=0x6000, out=0x7000)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _call(a):
    lib = load_lib()
    lib.sqllm_sample.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_sample(None if a is None else ctypes.byref(a), None)
    return rc, lib.sqllm_last_error().decode()


ALIGN = {"logits": 2, "pos": 4, "temperature": 4, "top_k": 4, "top_p": 4, "seed": 8, "out": 8}
BAD = [
    (dict(dtype=3), "dtype=3 is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(dtype=-1), "dtype=-1 is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16"),
    (dict(rows=0), "rows=0 must be in [1, 65535]"),
    (dict(rows=65536), "rows=65536 must be in [1, 65535]"),
    (dict(vocab=0), "vocab=0 must be in [1, 262144]"),
    (dict(vocab=262145, row_stride=300000), "vocab=262145 must be in [1, 262144]"),
    (dict(row_stride=31999), "row_stride=31999 must be >= vocab=32000"),
    (dict(row_stride=-1), "row_stride=-1 must be >= vocab=32000"),
    (dict(dtype=F32, logits=0x1002), "logits must be a non-null pointer aligned to 4 bytes"),
    (dict(dtype=BF16, logits=0x1001), "logits must be a non-null pointer aligned to 2 bytes"),
] + [(dict(**{f: 0}), f"{f} must be a non-null pointer aligned to {n} bytes") for f, n in ALIGN.items()] \
  + [(dict(**{f: 0x1001}), f"{f} must be a non-null pointer aligned to {n} bytes") for f, n in ALIGN.items()]


@pytest.mark.parametrize("change,frag", BAD, ids=[f"{next(iter(c))}={next(iter(c.values()))}" for c, _ in BAD])
def test_rejects(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


def test_rejects_null_args():
    rc, msg = _call(None)
    assert rc == -1 and "null args" in msg


def test_declared_in_the_header_and_the_version_unchanged():
    assert "sqllm_sample" in set(header_symbols())
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_sample\(const sqllm_sample_args \*args, void \*stream\);", txt)
    versions = txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert "sqllm_sample" in versions
    assert load_lib().sqllm_abi_version() == 4


# ---- the same through quant_cuda, on CPU tensors (the checks run before the device check) ----
torch = pytest.importorskip("torch")


def _tensors(R=4, V=100, dt=None):
    return dict(logits=torch.zeros(R, V, dtype=dt or torch.float16), pos=torch.zeros(R, dtype=torch.int32),
                temperature=torch.ones(R), top_k=torch.zeros(R, dtype=torch.int32), top_p=torch.ones(R),
                seed=torch.zeros(R, dtype=torch.int64), out=torch.zeros(R, dtype=torch.int64))


def _module_call(**t):
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.sample(t["logits"], t["pos"], t["temperature"], t["top_k"], t["top_p"], t["seed"], t["out"])


MODULE_BAD = [
    (lambda: _tensors(dt=torch.float64), "dtype of logits must be torch.float32, torch.float16 or torch.bfloat16"),
    (lambda: _tensors(dt=torch.int32), "dtype of logits must be torch.float32, torch.float16 or torch.bfloat16"),
    (lambda: dict(_tensors(), logits=torch.zeros(100, dtype=torch.float16)), "logits must be [rows, vocab]"),
    (lambda: dict(_tensors(), logits=torch.zeros(4, 0, dtype=torch.float16)), "logits must be [rows, vocab]"),
    (lambda: _tensors(R=65536, V=1), "rows=65536 must be in [1, 65535]"),
    (lambda: _tensors(R=1, V=262145), "vocab=262145 must be in [1, 262144]"),
    (lambda: dict(_tensors(), logits=torch.zeros(100, 4, dtype=torch.float16).t()), "logits must have unit last stride"),
    (lambda: dict(_tensors(), logits=torch.zeros(1, 100, dtype=torch.float16).expand(4, 100)), "logits' row stride 0 must be >= vocab=100"),
    (lambda: dict(_tensors(), pos=torch.zeros(4, dtype=torch.int64)), "pos must be a contiguous Int vector of rows=4"),
    (lambda: dict(_tensors(), pos=torch.zeros(3, dtype=torch.int32)), "pos must be a contiguous Int vector of rows=4"),
    (lambda: dict(_tensors(), temperature=torch.ones(4, dtype=torch.float64)), "temperature must be a contiguous Float vector of rows=4"),
    (lambda: dict(_tensors(), top_k=torch.zeros(4, 1, dtype=torch.int32)), "top_k must be a contiguous Int vector of rows=4"),
    (lambda: dict(_tensors(), top_p=torch.ones(8)[::2]), "top_p must be a contiguous Float vector of rows=4"),
    (lambda: dict(_tensors(), seed=torch.zeros(4, dtype=torch.int32)), "seed must be a contiguous Long vector of rows=4"),
    (lambda: dict(_tensors(), out=torch.zeros(4, dtype=torch.int32)), "out must be a contiguous Long vector of rows=4"),
    (lambda: dict(_tensors(), out=None), "out is undefined"),
    (lambda: _tensors(), "logits must be a CUDA tensor"),
    (lambda: _tensors(dt=torch.float32), "logits must be a CUDA tensor"),
]


@pytest.mark.parametrize("make,frag", MODULE_BAD, ids=[str(i) for i in range(len(MODULE_BAD))])
def test_module_rejects(make, frag):
    with pytest.raises((RuntimeError, TypeError), match=re.escape(frag) if "undefined" not in frag else None):
        _module_call(**make())


@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")
def test_module_rejects_mixed_devices():
    t = _tensors()
    t["logits"] = t["logits"].cuda()
    with pytest.raises(RuntimeError, match="pos must be a CUDA tensor, on the device of logits"):
        _module_call(**t)
