"""CPU tests of sqllm_fisher_accumulate's argument validation: bad arguments are rejected with SQLLM_EINVAL and a message before
anything touches a device.  The checks of quant_cuda.fisher_accumulate that need CUDA tensors are in test_fisher_gpu.py."""
import ctypes
import re

import pytest

from util import HEADER, header_symbols, load_lib

F32, F16, BF16 = 0, 1, 2


def _call(x=16, dy=32, dtype=F16, rows=128, seq_len=64, in_features=64, out_features=136, fisher=48):
    lib = load_lib()
    lib.sqllm_fisher_accumulate.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.sqllm_fisher_accumulate(x, dy, dtype, rows, seq_len, in_features, out_features, fisher, None)
    return rc, lib.sqllm_last_error()


@pytest.mark.parametrize("kw,frag", [
    (dict(dtype=F32), b"dtype=0 is not SQLLM_DT_F16 or SQLLM_DT_BF16"), (dict(dtype=3), b"dtype=3 is not"),
    (dict(dtype=-1), b"dtype=-1 is not"),
    (dict(rows=0), b"rows=0 must be >= 1"), (dict(rows=-64), b"rows=-64 must be >= 1"),
    (dict(seq_len=0), b"seq_len=0 must be >= 1"), (dict(seq_len=-2), b"seq_len=-2 must be >= 1"),
    (dict(rows=100, seq_len=64), b"rows=100 must be a multiple of seq_len=64"),
    (dict(rows=63, seq_len=2), b"rows=63 must be a multiple of seq_len=2"),
    (dict(in_features=0), b"in_features=0 must be a positive multiple of 8"),
    (dict(in_features=60), b"in_features=60 must be a positive multiple of 8"),
    (dict(in_features=-8), b"in_features=-8 must be a positive multiple of 8"),
    (dict(out_features=0), b"out_features=0 must be a positive multiple of 8"),
    (dict(out_features=132), b"out_features=132 must be a positive multiple of 8"),
    (dict(out_features=65536 * 128), b"out_features=8388608 exceeds 8388480"),
    (dict(x=0), b"x / dy / fisher must not be null"), (dict(dy=0), b"x / dy / fisher must not be null"),
    (dict(fisher=0), b"x / dy / fisher must not be null"),
    (dict(x=24), b"x / dy / fisher must be 16-byte aligned"), (dict(dy=34), b"x / dy / fisher must be 16-byte aligned"),
    (dict(fisher=52), b"x / dy / fisher must be 16-byte aligned"),
    (dict(dtype=BF16, fisher=8), b"x / dy / fisher must be 16-byte aligned")])
def test_rejects_bad_arguments(kw, frag):
    rc, msg = _call(**kw)
    assert rc == -1 and b"fisher_accumulate: " + frag in msg, msg


def test_module_rejects_cpu_tensors():
    torch = pytest.importorskip("torch")
    from squeezellm_b200.quant import quant_cuda
    x = torch.zeros(4, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="fisher_accumulate: x must be a contiguous CUDA tensor"):
        quant_cuda.fisher_accumulate(x, torch.zeros(4, 8, dtype=torch.float16), torch.zeros(8, 8), 2)


def test_declared_in_the_header_and_the_version_unchanged():
    assert "sqllm_fisher_accumulate" in header_symbols()
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_fisher_accumulate\(const void \*x, const void \*dy, int dtype, int rows, int seq_len, int in_features, "
                     r"int out_features,\s+float \*fisher, void \*stream\);", txt)
    assert "sqllm_fisher_accumulate" in txt[txt.index("#define SQLLM_ABI_VERSION"):txt.index("int sqllm_abi_version")]
    assert load_lib().sqllm_abi_version() == 4
