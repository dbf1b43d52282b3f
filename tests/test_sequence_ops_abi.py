"""CPU tests of the argument checks of sqllm_sequence_create_ops and of quant_cuda.sequence_create(ops=...): every bad op comes back
as SQLLM_EINVAL (RuntimeError in Python) with a message naming the item, before anything touches a device; ops = NULL / None and a
list of ops that do nothing keep the checks and messages of sqllm_sequence_create_dt."""
import ctypes
import math
import re

import pytest

from test_sequence_host import SeqItem, SeqOptions, _item
from util import HEADER, header_symbols, load_lib

F16, BF16 = 1, 2
PLAIN, RMSNORM, SILU = 0, 1, 2


class SeqOp(ctypes.Structure):  # mirrors sqllm_seq_op
    _fields_ = [("x_op", ctypes.c_int), ("norm_weight", ctypes.c_void_p), ("eps", ctypes.c_float), ("x2_from", ctypes.c_int),
                ("x2_offset", ctypes.c_int), ("res_from", ctypes.c_int), ("res_offset", ctypes.c_int), ("res_ext", ctypes.c_void_p)]


def _op(x_op=PLAIN, w=None, eps=1e-6, x2=(-1, 0), res=(-1, 0), res_ext=None):
    return SeqOp(x_op=x_op, norm_weight=w, eps=eps, x2_from=x2[0], x2_offset=x2[1], res_from=res[0], res_offset=res[1], res_ext=res_ext)


def _create(items, ops, dtype=F16, **opt):
    lib = load_lib()
    lib.sqllm_sequence_create_ops.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    arr = (SeqItem * len(items))(*items) if items else None
    oarr = (SeqOp * len(ops))(*ops) if ops is not None else None
    o = SeqOptions(lut_mode=opt.get("lut_mode", 0), world=opt.get("world", 1), rank=opt.get("rank", 0))
    h = ctypes.c_void_p()
    rc = lib.sqllm_sequence_create_ops(arr, oarr, len(items), ctypes.byref(o), dtype, ctypes.byref(h))
    msg = lib.sqllm_last_error().decode()
    if rc == 0:  # (a machine with a GPU gets this far with the made-up addresses; the sequence is never run)
        lib.sqllm_sequence_destroy.argtypes = [ctypes.c_void_p]
        lib.sqllm_sequence_destroy(h)
    return rc, msg


def _layer_items():
    """A decoder layer's shape: o = o_proj(x); gu = gate_up(o) [2 x 512]; d = down(gu[:512]) [256]; q = qkv(d)."""
    return [_item(K=256, N=256), _item(K=256, N=1024, x_from=0), _item(K=512, N=256, x_from=1), _item(K=256, N=768, x_from=2)]


BAD_OPS = [  # (item index, op, fragment of the message)
    (1, _op(x_op=3), "item 1: unknown x_op=3"),
    (1, _op(x_op=-1), "item 1: unknown x_op=-1"),
    (1, _op(RMSNORM, w=None), "item 1: norm_weight must be a 16-byte aligned"),
    (1, _op(RMSNORM, w=4096 + 8), "item 1: norm_weight must be a 16-byte aligned"),
    (1, _op(RMSNORM, w=4096, eps=-1e-6), "item 1: eps=-1e-06 must be finite and >= 0"),
    (1, _op(RMSNORM, w=4096, eps=math.inf), "item 1: eps=inf must be finite"),
    (1, _op(RMSNORM, w=4096, eps=math.nan), "item 1: eps=nan must be finite"),
    (2, _op(SILU, x2=(2, 512)), "item 2: x2_from=2 must name an earlier item"),
    (2, _op(SILU, x2=(-1, 0)), "item 2: x2_from=-1 must name an earlier item"),
    (2, _op(SILU, x2=(1, 768)), "item 2: x2 reads [768, 1280) of item 1's 1024 outputs"),
    (2, _op(SILU, x2=(1, 514)), "item 2: x2 reads [514, 1026)"),
    (2, _op(SILU, x2=(1, -4)), "item 2: x2 reads [-4,"),
    (2, _op(res=(2, 0)), "item 2: residual source res_from=2 must name an earlier item"),
    (2, _op(res=(3, 0)), "item 2: residual source res_from=3 must name an earlier item"),
    (2, _op(res=(-2, 0)), "item 2: residual source res_from=-2"),
    (3, _op(res=(0, 0)), "item 3: residual reads [0, 768) of item 0's 256 outputs"),      # a shorter source
    (2, _op(res=(1, 772)), "item 2: residual reads [772, 1028)"),
    (2, _op(res=(0, 2)), "item 2: residual reads [2, 258)"),
    (2, _op(res=(0, 0), res_ext=4096), "item 2: one residual source"),
    (2, _op(res_ext=4096 + 2), "item 2: res_ext must be a 16-byte aligned"),
]


@pytest.mark.parametrize("dtype,name", [(F16, "fp16"), (BF16, "bf16")])
@pytest.mark.parametrize("at,op,needle", BAD_OPS, ids=[f"{i}-{b[2].split(': ', 1)[1][:28]}" for i, b in enumerate(BAD_OPS)])
def test_create_ops_rejects_bad_ops(at, op, needle, dtype, name):
    ops = [_op() for _ in range(4)]
    ops[at] = op
    rc, msg = _create(_layer_items(), ops, dtype)
    assert rc == -1 and needle in msg, (rc, msg)
    if "aligned" in needle:
        assert f"aligned {name} vector" in msg, msg


def test_a_good_layer_passes_the_op_checks():
    """A whole decoder layer's ops are accepted by the checks: the call gets as far as the device (no GPU here: some later error, or
    success on a machine that has one), never to an op message."""
    ops = [_op(res_ext=4096), _op(RMSNORM, w=4096, eps=1e-5), _op(SILU, x2=(1, 512), res=(0, 0)), _op(RMSNORM, w=8192, eps=0.0)]
    rc, msg = _create(_layer_items(), ops)
    for frag in ("x_op", "norm_weight", "eps=", "x2", "residual", "res_ext"):
        assert rc == 0 or frag not in msg, msg


@pytest.mark.parametrize("items,kw,needle", [
    ([], {}, "null / empty"),
    ([_item(), _item(bits=3, x_from=0)], {}, "one sequence, one width"),
    ([_item(), _item(x_from=1)], {}, "must name an earlier item"),
    ([_item(N=256), _item(K=256, x_from=0, x_offset=2)], {}, "reads ["),
    ([_item(N=32)], {}, "out_features=32 <"),
    ([_item(N=256, members=3)], {}, "members of a multiple of 4"),
    ([_item()], {"world": 2, "rank": 0}, "peer-visible arena"),
    ([_item()], {"world": 2, "rank": 5}, "bad world / rank"),
])
@pytest.mark.parametrize("with_ops", [False, True])
def test_null_and_plain_ops_keep_the_sequence_checks(items, kw, needle, with_ops):
    ops = [_op() for _ in items] if with_ops else None
    rc, msg = _create(items, ops, **kw)
    assert rc == -1 and needle in msg, (rc, msg)
    # the item checks come before the op checks: the same message with a bad op on top
    if items and with_ops:
        rc2, msg2 = _create(items, [_op(x_op=7) for _ in items], **kw)
        assert rc2 == -1 and msg2 == msg


def test_dtype_is_checked_first():
    rc, msg = _create([_item()], [_op(x_op=9)], dtype=0)
    assert rc == -1 and "dtype=0" in msg, msg


def test_header_declares_and_library_exports_create_ops():
    syms = header_symbols()
    txt = open(HEADER).read()
    later = txt.split("#define SQLLM_ABI_VERSION")[1].split("*/")[0]
    assert "sqllm_sequence_create_ops" in syms and "sqllm_sequence_create_ops" in later
    lib = load_lib()
    assert hasattr(lib, "sqllm_sequence_create_ops") and lib.sqllm_abi_version() == 4
    for name, v in (("SQLLM_SEQ_X_PLAIN", 0), ("SQLLM_SEQ_X_RMSNORM", 1), ("SQLLM_SEQ_X_SILU_MUL", 2)):
        assert f"#define {name} {v}" in txt


# ---- the same through quant_cuda (the op checks that need no CUDA tensor run before the items' own) ----
def _qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def _py_items():
    import torch
    q = torch.zeros(256 // 32 * 4, 256, dtype=torch.int32)   # CPU tensors: the op checks reject before the items are looked at
    lut = torch.zeros(256, 16)
    it = (q, lut, 4, None, None, None, None, None, None, -1, 0, torch.zeros(256, dtype=torch.float16), 1, 256)
    it1 = (q, lut, 4, None, None, None, None, None, None, 0, 0, None, 1, 256)
    return [it, it1, it1]


PY_BAD = [
    (1, (3, None, 1e-6, -1, 0, -1, 0, None), "sequence item 1: unknown x_op=3"),
    (1, (1, None, 1e-6, -1, 0, -1, 0, None), "sequence item 1: RMSNorm needs norm_weight"),
    (1, (1, "cpu", 1e-6, -1, 0, -1, 0, None), "sequence item 1: norm_weight must be a contiguous fp16 CUDA tensor"),
    (1, (1, "cuda?", -1.0, -1, 0, -1, 0, None), "eps=-1 must be finite and >= 0"),
    (2, (2, None, 0.0, 2, 0, -1, 0, None), "sequence item 2: x2_from=2 must name an earlier item"),
    (2, (2, None, 0.0, -1, 0, -1, 0, None), "sequence item 2: x2_from=-1 must name an earlier item"),
    (1, (0, None, 0.0, -1, 0, 1, 0, None), "sequence item 1: residual source res_from=1 must name an earlier item"),
    (1, (0, None, 0.0, -1, 0, -1, 0, "cpu"), "sequence item 1: res_ext must be a contiguous fp16 CUDA tensor"),
    (1, (0, None, 0.0, -1, 0, -1, 0, "bf16"), "sequence item 1: res_ext must be a contiguous fp16 CUDA tensor"),
    (1, (0, None, 0.0, -1), "sequence op 1: expected None or an 8-tuple"),
]


@pytest.mark.parametrize("at,op,needle", PY_BAD, ids=[str(i) for i in range(len(PY_BAD))])
def test_quant_cuda_rejects_bad_ops(at, op, needle):
    import torch
    sub ={"cpu": torch.zeros(256, dtype=torch.float16), "bf16": torch.zeros(256, dtype=torch.bfloat16)}
    if op[1] == "cuda?":  # the eps check needs a weight that passes: on a machine without a GPU the weight check fires first
        if not torch.cuda.is_available():
            op = (1, sub["cpu"], op[2]) + op[3:]
            needle = "norm_weight must be a contiguous fp16 CUDA tensor"
        else:
            op = (1, torch.zeros(256, dtype=torch.float16, device="cuda")) + op[2:]
    op = tuple(sub.get(v, v) if isinstance(v, str) else v for v in op)
    ops = [None, None, None]
    ops[at] = op
    with pytest.raises(RuntimeError, match=re.escape(needle)):
        _qc().sequence_create(_py_items(), [], "exact", ops=ops)


def test_quant_cuda_ops_length_and_keyword():
    import torch
    with pytest.raises(RuntimeError, match="2 ops for 3 items"):
        _qc().sequence_create(_py_items(), [], "exact", ops=[None, None])
    with pytest.raises(TypeError):  # ops is keyword-only: the positional signature is the one it always was
        _qc().sequence_create(_py_items(), [], "exact", 1, 0, None, 0, torch.float16, [None] * 3)


@pytest.mark.parametrize("ops", [None, [None, None, None]])
def test_quant_cuda_none_ops_keep_the_item_checks(ops):
    """ops=None and all-None ops: the CPU qweight is rejected exactly as without the keyword."""
    with pytest.raises(RuntimeError) as e0:
        _qc().sequence_create(_py_items(), [], "exact")
    with pytest.raises(RuntimeError) as e1:
        _qc().sequence_create(_py_items(), [], "exact", ops=ops)
    assert str(e0.value).splitlines()[0] == str(e1.value).splitlines()[0]
    assert "qweight must be a packed CUDA matrix" in str(e1.value)
