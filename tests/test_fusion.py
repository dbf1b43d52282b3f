"""Sibling fusion (squeezellm_b200/fusion.py): stacked buffers are the members' buffers side by side, the one-result cache
hands every member its own slice, and - on the GPU - a stacked launch equals the members' own launches."""
import numpy as np
import pytest
import torch


from squeezellm_b200.quant import QuantLinearLUT
from squeezellm_b200 import fusion
from util import OUT_ROUNDING, abs_sum, bound_ratio, layer_as_read, make_activations, orc, quant_layer


def _layers(bits, K, widths, sparsity, topx, bias=False):
    return [orc.make_layer(bits, K, n, sparsity=sparsity if i != 1 else 0.0, topX=topx if i != 1 else 0, seed=31 + i,
                           nonzero_full_rows=True, bias=bias) for i, n in enumerate(widths)]


def _rowless_dense_member(bits, K, N, seed):
    """include_sparse and dense rows but no CSR arrays (make_quant_lut with numvals 0): its forward reads no outliers at all."""
    L = orc.make_layer(bits, K, N, topX=3, seed=seed, nonzero_full_rows=True, bias=True)
    m = QuantLinearLUT(bits, K, N, True, include_sparse=True, numvals=0, topX=3)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)})
    return m


STACK_CASES = [(3, "mixed"), (4, "mixed"), (3, "csr-next-to-rowless-dense"), (4, "csr-next-to-rowless-dense")]


@pytest.mark.parametrize("bits,group", STACK_CASES, ids=["3", "4", "3-csr-next-to-rowless-dense", "4-csr-next-to-rowless-dense"])
def test_stacked_buffers_equal_members_side_by_side(bits, group):
    """oracle(stacked layer) == concat(oracle(member_i as its own forward reads it)) exactly: same packed words, LUT rows, CSR
    entries, dense rows.  mixed: member 1 has no outliers at all (mixed groups must still stack).  csr-next-to-rowless-dense: a
    member with CSR and dense rows next to one whose dense rows its forward ignores (no CSR arrays)."""
    K = 256
    if group == "mixed":
        ms = [quant_layer(L) for L in _layers(bits, K, [64, 128, 192], 0.02, 3, bias=True)]
    else:
        ms = [quant_layer(orc.make_layer(bits, K, 64, sparsity=0.02, topX=3, seed=31, nonzero_full_rows=True, bias=True)),
              _rowless_dense_member(bits, K, 128, seed=32)]
    n = sum(m.outfeatures for m in ms)
    b = fusion.stack_buffers(ms)
    assert b["offsets"] == list(np.cumsum([0] + [m.outfeatures for m in ms])) and b["qweight"].shape == (K // 32 * bits, n)
    stacked = dict(bits=bits, infeatures=K, outfeatures=n, bias=None,
                   **{k: b[k].numpy() for k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices")})
    x = orc.make_vec(K, seed=3)
    got = orc.forward_f64(stacked, x)
    want = np.concatenate([orc.forward_f64(layer_as_read(m), x) for m in ms], axis=1)
    assert np.array_equal(got, want)
    assert torch.equal(b["bias"], torch.cat([m.bias for m in ms]))
    assert b["rows"][-1].item() == len(b["cols"]) == sum(len(m._sparse_args()[2]) for m in ms if m._sparse_args()[2] is not None)


def test_result_cache_protocol():
    """One stacked call per distinct input; each member consumes once; a new / modified x recomputes."""
    K = 64
    ms = [quant_layer(orc.make_layer(4, K, n, seed=n)) for n in (32, 64)]
    g = fusion.SiblingGroup(ms)
    # members expose their buffers as views of the stacked storage (state_dict keys unchanged)
    assert ms[1].qweight.data_ptr() == g.layer.qweight.data_ptr() + 32 * 4 and not ms[1].qweight.is_contiguous()
    assert ms[1].lookup_table.data_ptr() == g.layer.lookup_table.data_ptr() + 32 * 16 * 4
    assert set(ms[0].state_dict()) >= {"qweight", "lookup_table"}
    calls = []

    class Fake:
        def __call__(self, x):
            calls.append(x)
            return torch.arange(96, dtype=torch.float32).reshape(1, 96) + 1000 * len(calls)
    g.layer = Fake()
    x = torch.zeros(1, K)
    a, b = ms[0](x), ms[1](x)
    assert len(calls) == 1 and a.shape == (1, 32) and b.shape == (1, 64)
    assert a[0, 0].item() == 1000 and b[0, 0].item() == 1032
    assert g._x is None, "reference to x is dropped once every member has consumed"
    ms[0](x)
    ms[0](x)                      # same member twice: second call must not reuse a consumed result
    assert len(calls) == 3
    x2 = torch.zeros(1, K)
    ms[1](x2)                     # different tensor object
    assert len(calls) == 4
    ms[0](x2)
    assert len(calls) == 4        # sibling of the x2 result
    ms[0](x)
    x.add_(1.0)                   # in-place update bumps the version counter
    ms[1](x)
    assert len(calls) == 6


def test_fuse_siblings_walks_llama_like_modules():
    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
                setattr(self, n, quant_layer(orc.make_layer(4, 64, 64, seed=5)))

    class Mlp(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.gate_proj = quant_layer(orc.make_layer(4, 64, 128, seed=6))
            self.up_proj = quant_layer(orc.make_layer(4, 64, 128, seed=7))
            self.down_proj = quant_layer(orc.make_layer(4, 128, 64, seed=8))

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.self_attn, self.mlp = Attn(), Mlp()
    model = torch.nn.Sequential(Block(), Block())
    groups = fusion.fuse_siblings(model)
    assert len(groups) == 4 and sorted(len(g.members) for g in groups) == [2, 2, 3, 3]
    assert model[0].self_attn.o_proj._sibling_group is None and model[1].mlp.down_proj._sibling_group is None
    assert fusion.fuse_siblings(model) == [], "idempotent"


def _truth(L, x, bias_inside):
    """want, S and the rounded quantity of layer L on x [M, K] (numpy, the exact values the layer saw), with L's bias if it has one:
    inside the rounded sum for a one-row call, added after the rounding otherwise (tests/util.py, bound_ratio)."""
    b = L.get("bias")
    want, S = orc.forward_f64(L, x), abs_sum(L, x)
    if b is None:
        return want, S, want
    b = b.astype(np.float64)[None, :]
    return want + b, S + np.abs(b), (want + b if bias_inside else want)


def _bound(y, L, x, y_dtype):
    M = x.shape[0]
    want, S, rounded = _truth(L, x, bias_inside=M == 1)
    r, eta = OUT_ROUNDING[str(y_dtype).split(".")[1]]
    return bound_ratio(y.float().cpu().numpy().reshape(M, -1), want, S, rounded, r, eta=eta)


GPU_GROUPS = [(4, 4096, [4096, 4096, 4096], 0.0045, 10), (3, 4096, [11008, 11008], 0.0045, 10), (4, 512, [128, 256], 0.0, 0),
              # the middle member has no dense rows: 2 x topX stacked
              (4, 1024, [1024, 1024, 1024], 0.01, 16),   # 32: the topX <= 32 branch at its edge
              (3, 1024, [1024, 1024, 1024], 0.01, 17),   # 34: the general branch
              (4, 1024, [1024, 1024, 1024], 0.01, 70)]   # 140: more than the fused launch takes
GPU_IDS = ["w4-qkv", "w3-gateup", "w4-small-dense", "w4-qkv-t16", "w3-qkv-t17", "w4-qkv-t70"]


@pytest.mark.gpu
@pytest.mark.parametrize("bits,K,widths,sp,topx,bias", [g + (False,) for g in GPU_GROUPS] + [g + (True,) for g in GPU_GROUPS],
                         ids=GPU_IDS + [i + "-bias" for i in GPU_IDS])
def test_stacked_launch_matches_members(bits, K, widths, sp, topx, bias):
    """One row (the fused decode launch, bias inside the sum) and two rows (the multi-row launch, bias added after the rounding):
    every member's slice of the stacked launch against the fp64 oracle per element (bound_ratio), and next to its own launch."""
    Ls = _layers(bits, K, widths, sp, topx, bias=bias)
    ms = [quant_layer(L).cuda() for L in Ls]
    x = torch.from_numpy(orc.make_vec(K, seed=12)).cuda().half().reshape(1, 1, K)
    alone = [m(x) for m in ms]
    g = fusion.SiblingGroup(ms)
    together = [m(x) for m in ms]
    torch.cuda.synchronize()
    assert g.launches == 1
    for L, m, a, t in zip(Ls, ms, alone, together):
        assert t.shape == (1, 1, L["outfeatures"]) and t.dtype == torch.float16
        x_np = x.float().cpu().numpy().reshape(1, K)
        assert _bound(t, L, x_np, t.dtype) <= 1.0
        assert _bound(a, L, x_np, a.dtype) <= 1.0
        assert not m.qweight.is_contiguous() or len(widths) == 1  # a view of the stacked matrix, not a copy
    xb = torch.from_numpy(orc.make_vec(K, batch=2, seed=13)).cuda().half().reshape(1, 2, K)
    yb = [m(xb) for m in ms]
    assert g.launches == 2
    for L, y in zip(Ls, yb):
        assert y.shape == (1, 2, L["outfeatures"]) and y.dtype == (torch.float32 if bias else torch.float16)
        assert _bound(y, L, xb.float().cpu().numpy().reshape(2, K), torch.float16) <= 1.0


MIXED_BIAS_CASES = [(torch.float16, M) for M in (1, 5, 64)] + [(torch.bfloat16, M) for M in (1, 5, 80)] + \
                   [(torch.float32, M) for M in (1, 128)]


@pytest.fixture(scope="module")
def mixed_bias_layers():
    """q / k / v at GQA widths (1024 / 256 / 256 over 1024 inputs) with outliers and dense rows; q and v have a bias, k has none
    (Whisper's attention)."""
    return [orc.make_layer(4, 1024, n, sparsity=0.0045, topX=10, seed=71 + i, nonzero_full_rows=True, bias=i != 1)
            for i, n in enumerate((1024, 256, 256))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,M", MIXED_BIAS_CASES, ids=[f"{str(d).split('.')[1]}-M{m}" for d, m in MIXED_BIAS_CASES])
def test_member_without_bias_keeps_its_dtype_in_a_group_with_biases(mixed_bias_layers, dtype, M):
    """A batch through a stacked layer that has a bias comes back as out.to(dtype) + fp32 bias, i.e. fp32.  The member without a
    bias returns what it returns alone: x's dtype (HF's attention rejects q / k / v of mixed dtypes), the same shape, and values
    within the bound; on the launches whose bits do not depend on the call (the multi-row and the tensor-core LUT-GEMM) the same
    bits as alone."""
    Ls = mixed_bias_layers
    alone = [quant_layer(L).cuda() for L in Ls]
    ms = [quant_layer(L).cuda() for L in Ls]
    g = fusion.SiblingGroup(ms)
    x = torch.from_numpy(make_activations(1024, M, seed=M)).cuda().to(dtype).reshape(1, M, 1024)
    x_np = x.float().cpu().numpy().reshape(M, 1024)
    want_alone = [a(x) for a in alone]
    got = [m(x) for m in ms]
    torch.cuda.synchronize()
    assert g.launches == 1
    reproducible = M > 1 and (dtype != torch.float32 or M >= QuantLinearLUT.FP32_TC_MIN_ROWS)
    for L, a, y in zip(Ls, want_alone, got):
        assert y.dtype == a.dtype and y.shape == a.shape == (1, M, L["outfeatures"]), (y.dtype, a.dtype, y.shape)
        assert _bound(y, L, x_np, dtype) <= 1.0
        if reproducible:
            assert torch.equal(y, a)
    assert got[1].dtype == dtype
    assert got[0].dtype == (dtype if M == 1 else torch.float32)
