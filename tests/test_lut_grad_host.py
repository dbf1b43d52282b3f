"""CPU tests of codebook training (QuantLinearLUT.train_codebook, sqllm_lut_grad): the fp64 gradient truth (tests/lut_grad_ref.py)
against torch's fp64 autograd through a dense restatement of W(LUT, vals, full_rows); sqllm_lut_grad's argument checks, answered
before anything touches a device; train_codebook's parameters, errors and checkpoint round trip; fuse_siblings leaving trained
groups unfused."""
import ctypes
import re

import numpy as np
import pytest
import torch

from lut_grad_ref import dense_w_torch, lut_grad_f64
from util import HEADER, Args, header_symbols, load_lib, orc, quant_layer

F32, F16, BF16 = 0, 1, 2


# ---- the fp64 truth ---------------------------------------------------------------------------------------------------------
def _layer(bits, K, N, seed):
    """Duplicate CSR entries, out-of-range CSR columns and dense-row channels, duplicate dense-row channels and one on channel 0."""
    L = orc.make_layer(bits, K, N, sparsity=0.05, topX=6, seed=seed, nonzero_full_rows=True)
    fri = L["full_row_indices"]
    fri[1] = fri[0]
    fri[2] = 0
    fri[3] = N + 2
    fri[4] = -1
    L["cols"] = L["cols"].copy()
    L["cols"][0] = K + 5
    L["cols"][-1] = -3
    rows = L["rows"]
    c = int(np.argmax(np.diff(rows)))
    assert rows[c + 1] - rows[c] >= 3
    L["cols"][rows[c] + 1] = L["cols"][rows[c]]
    return L


@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("bias", [False, True])
def test_truth_equals_fp64_autograd_of_the_dense_layer(bits, bias):
    K, N, M = 96, 40, 7
    L = _layer(bits, K, N, seed=bits + 3 * bias)
    rng = np.random.default_rng(5)
    x = rng.standard_normal((M, K))
    dy = rng.standard_normal((M, N))
    lut = torch.from_numpy(L["lookup_table"].astype(np.float64)).requires_grad_()
    vals = torch.from_numpy(L["vals"].astype(np.float64)).requires_grad_()
    fr = torch.from_numpy(L["full_rows"].astype(np.float64)).requires_grad_()
    b = torch.zeros(N, dtype=torch.float64, requires_grad=True)
    y = torch.from_numpy(x) @ dense_w_torch(L, lut, vals, fr)
    if bias:
        y = y + b
    y.backward(torch.from_numpy(dy))
    g, S = lut_grad_f64(L, x, dy)
    np.testing.assert_allclose(g["lookup_table"], lut.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(g["vals"], vals.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(g["full_rows"], fr.grad.numpy(), rtol=1e-12, atol=1e-12)
    if bias:
        np.testing.assert_allclose(b.grad.numpy(), dy.sum(0), rtol=1e-12)
    # the rules: out-of-range entries get 0, duplicates each get the full G
    assert g["vals"][0] == 0 and g["vals"][-1] == 0
    assert (g["full_rows"][:, 3] == 0).all() and (g["full_rows"][:, 4] == 0).all()
    np.testing.assert_array_equal(g["full_rows"][:, 1], g["full_rows"][:, 0])
    for k in g:
        assert (S[k] >= np.abs(g[k]) - 1e-12).all()


def test_truth_column_blocks():
    import lut_grad_ref
    L = _layer(4, 64, 300, seed=9)
    rng = np.random.default_rng(6)
    x, dy = rng.standard_normal((5, 64)), rng.standard_normal((5, 300))
    whole = lut_grad_f64(L, x, dy)
    old = lut_grad_ref.COL_BLOCK
    try:
        lut_grad_ref.COL_BLOCK = 64
        blocked = lut_grad_f64(L, x, dy)
    finally:
        lut_grad_ref.COL_BLOCK = old
    for part in (0, 1):
        for k in whole[part]:
            np.testing.assert_allclose(blocked[part][k], whole[part][k], rtol=1e-12, atol=1e-13)


# ---- sqllm_lut_grad's argument checks ---------------------------------------------------------------------------------------
def _call(a, x=16, x_dt=F16, dy=16, dy_dt=F16, dlut=16, dvals=0, dfull=0, path=0):
    lib = load_lib()
    lib.sqllm_lut_grad.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    rc = lib.sqllm_lut_grad(None if a is None else ctypes.byref(a), x, x_dt, dy, dy_dt, dlut or None, dvals or None, dfull or None,
                            path, None)
    return rc, lib.sqllm_last_error()


def _args(**kw):
    a = Args(bits=4, in_features=160, out_features=132, batch=7, qweight=16, lookup_table=16)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("change,frag", [
    (dict(bits=2), b"bits must be 3 or 4"), (dict(bits=5), b"bits must be 3 or 4"),
    (dict(in_features=100), b"in_features=100 must be a positive multiple of 32"),
    (dict(in_features=0), b"in_features=0 must be a positive multiple of 32"),
    (dict(out_features=0), b"out_features=0 must be positive"),
    (dict(out_features=65536 * 128), b"out_features=8388608 exceeds"),
    (dict(batch=0), b"batch (rows of x and dy) must be >= 1"), (dict(batch=-2), b"batch (rows of x and dy) must be >= 1"),
    (dict(qweight=0), b"qweight must not be null"), (dict(qweight=18), b"qweight must be 4-byte aligned"),
    (dict(topX=-1), b"topX < 0")])
def test_rejects_bad_descriptor(change, frag):
    rc, msg = _call(_args(**change))
    assert rc == -1 and frag in msg, msg


@pytest.mark.parametrize("kw,frag", [
    (dict(x=0), b"x / dy must not be null"), (dict(dy=0), b"x / dy must not be null"),
    (dict(x_dt=3), b"x_dtype=3 is not"), (dict(dy_dt=-1), b"dy_dtype=-1 is not"),
    (dict(path=3), b"path=3 must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)"), (dict(path=-1), b"path=-1 must be"),
    (dict(path=1, x_dt=F32, dy_dt=F32), b"path=1 (tensor cores) takes x and dy both fp16 or both bf16"),
    (dict(path=1, x_dt=F16, dy_dt=F32), b"path=1 (tensor cores) takes x and dy both fp16 or both bf16"),
    (dict(path=1, x_dt=F16, dy_dt=BF16), b"path=1 (tensor cores) takes x and dy both fp16 or both bf16"),
    (dict(dlut=0), b"no output requested"),
    (dict(dvals=16), b"dvals needs the CSR arrays (rows, cols)"),
    (dict(dfull=16), b"dfull_rows needs the dense rows (full_row_indices, topX >= 1)"),
    (dict(x=17), b"x and dy must be aligned to their element size"),
    (dict(dy=18, dy_dt=F32), b"x and dy must be aligned to their element size"),
    (dict(dlut=18), b"dlut, dvals and dfull_rows must be 4-byte aligned")])
def test_rejects_bad_pointers_dtypes_outputs_and_paths(kw, frag):
    rc, msg = _call(_args(), **kw)
    assert rc == -1 and frag in msg, msg


def test_rejects_outputs_without_their_inputs():
    rc, msg = _call(_args(rows=16), dvals=16)  # rows without cols
    assert rc == -1 and b"dvals needs the CSR arrays" in msg
    rc, msg = _call(_args(full_row_indices=16, topX=0), dfull=16)
    assert rc == -1 and b"dfull_rows needs the dense rows" in msg
    rc, msg = _call(_args(full_rows=16, topX=3), dfull=16)  # dense rows without their channel indices
    assert rc == -1 and b"dfull_rows needs the dense rows" in msg
    rc, msg = _call(_args(dlut=0, rows=16, cols=16, vals=16, full_rows=16, full_row_indices=16, topX=3, qweight=17), dvals=16, dfull=16)
    assert rc == -1 and b"qweight must be 4-byte aligned" in msg


def test_rejects_null_descriptor():
    rc, msg = _call(None)
    assert rc == -1 and b"null args" in msg


def test_declared_in_the_header_and_the_version_unchanged():
    assert "sqllm_lut_grad" in header_symbols()
    txt = open(HEADER).read()
    assert re.search(r"int sqllm_lut_grad\(const sqllm_lutgemv_args \*args, const void \*x, int x_dtype, const void \*dy, int dy_dtype, "
                     r"float \*dlut, float \*dvals,\s+float \*dfull_rows, int path, void \*stream\);", txt)
    assert re.search(r"#define SQLLM_LUT_GRAD_TC_MIN_ROWS \d+\b", txt)
    assert load_lib().sqllm_abi_version() == 4


# ---- the module: train_codebook ---------------------------------------------------------------------------------------------
def _module(L, bias=False):
    return quant_layer(L, bias=np.zeros(L["outfeatures"], dtype=np.float32) if bias else None)


def test_train_codebook_makes_parameters_on_the_same_storage():
    m = _module(orc.make_layer(4, 128, 64, sparsity=0.02, topX=3, seed=1, nonzero_full_rows=True), bias=True)
    keys = list(m.state_dict())
    ptrs = {n: getattr(m, n).data_ptr() for n in ("lookup_table", "vals", "full_rows", "bias")}
    assert list(m.parameters()) == []
    got = m.train_codebook()
    assert len(got) == 1 and got[0] is m.lookup_table and isinstance(m.lookup_table, torch.nn.Parameter)
    assert m.lookup_table.requires_grad and m.lookup_table.data_ptr() == ptrs["lookup_table"]
    got = m.train_codebook(lookup_table=False, vals=True, full_rows=True, bias=True)
    assert [p.data_ptr() for p in got] == [ptrs["vals"], ptrs["full_rows"], ptrs["bias"]]
    assert m._trained == ("lookup_table", "vals", "full_rows", "bias")
    assert sorted(m.state_dict()) == sorted(keys)
    assert {n for n, _ in m.named_parameters()} == {"lookup_table", "vals", "full_rows", "bias"}
    assert {n for n, _ in m.named_buffers()} == {"qweight", "rows", "cols", "full_row_indices"}


def test_train_codebook_rejects_missing_tensors_and_sibling_members():
    from squeezellm_b200.fusion import fuse_siblings
    plain = _module(orc.make_layer(3, 64, 32, seed=2))
    for kw, frag in ((dict(vals=True), "CSR outliers"), (dict(full_rows=True), "dense rows"), (dict(bias=True), "no bias")):
        with pytest.raises(ValueError, match=frag):
            plain.train_codebook(**kw)
    assert plain._trained == ()  # a rejected call changes nothing
    model = _Attn(train=None)
    assert len(fuse_siblings(model)) == 1
    with pytest.raises(RuntimeError, match="sibling group"):
        model.q_proj.train_codebook()


def test_train_codebook_checks_every_dtype_before_converting_any():
    m = _module(orc.make_layer(4, 128, 64, sparsity=0.02, seed=4))
    m.vals = m.vals.double()
    with pytest.raises(ValueError, match="`vals` must be fp32"):
        m.train_codebook(lookup_table=True, vals=True)
    assert m._trained == () and list(m.parameters()) == [] and "lookup_table" in dict(m.named_buffers())


def test_pack2_refuses_a_trained_layer():
    import types
    m = _module(orc.make_layer(4, 64, 32, seed=5))
    m.train_codebook()
    with pytest.raises(RuntimeError, match="pack2 fills the buffers of a layer before training"):
        m.pack2(types.SimpleNamespace(weight=torch.zeros(32, 64), bias=None), ([], None), False)


class _Attn(torch.nn.Module):
    def __init__(self, train):
        super().__init__()
        self.q_proj, self.k_proj, self.v_proj = (_module(orc.make_layer(4, 64, n, seed=n)) for n in (64, 32, 32))
        if train is not None:
            getattr(self, train).train_codebook()


@pytest.mark.parametrize("train", ["q_proj", "v_proj"])
def test_fuse_siblings_skips_trained_groups(train):
    from squeezellm_b200.fusion import fuse_siblings
    model = _Attn(train)
    assert fuse_siblings(model) == []
    assert all(getattr(model, n)._sibling_group is None for n in ("q_proj", "k_proj", "v_proj"))


def test_trained_layer_round_trips_through_the_checkpoint():
    from squeezellm_b200.checkpoint import load_quantized, quantized_state_dict

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.proj = torch.nn.Linear(128, 64, bias=True)

    L = orc.make_layer(4, 128, 64, sparsity=0.02, topX=2, seed=3, nonzero_full_rows=True, bias=True)
    src = Net()
    state = {f"proj.{k}": torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)}
    state["sparse_threshold.proj"] = len(L["vals"])
    load_quantized(src, state, wbits=4, include_sparse=True, topX=2)
    before = quantized_state_dict(src)
    params = src.proj.train_codebook(vals=True, full_rows=True, bias=True)
    after = quantized_state_dict(src)
    assert sorted(after) == sorted(before)  # same keys (parameters come first in state_dict order)
    with torch.no_grad():  # what an optimizer step does: in place
        for p in params:
            p.mul_(1.5).add_(0.25)
    saved = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in quantized_state_dict(src).items()}
    for fresh_trained in (False, True):
        dst = Net()
        missing, unexpected = load_quantized(dst, saved, wbits=4, include_sparse=True, topX=2)
        assert not missing and not unexpected
        if fresh_trained:  # loading into an already trained layer writes into its parameters
            dst.proj.train_codebook(vals=True, full_rows=True, bias=True)
            load_quantized(dst, saved, wbits=4, include_sparse=True, topX=2)
        for k, v in saved.items():
            if torch.is_tensor(v):
                assert torch.equal(dst.state_dict()[k], v), k
        assert torch.equal(dst.proj.lookup_table, src.proj.lookup_table.detach())
