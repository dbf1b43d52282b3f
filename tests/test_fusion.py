"""Sibling fusion (squeezellm_b200/fusion.py): stacked buffers are the members' buffers side by side, the one-result cache
hands every member its own slice, and - on the GPU - a stacked launch equals the members' own launches."""
import numpy as np
import pytest
import torch


from squeezellm_b200.quant import QuantLinearLUT
from squeezellm_b200 import fusion
from util import orc, rel_err, REL_TOL


def _member(L, bias=False):
    sparse = L.get("rows") is not None
    topx = int(L["full_rows"].shape[1]) if L.get("full_rows") is not None else 0
    m = QuantLinearLUT(L["bits"], L["infeatures"], L["outfeatures"], bias, include_sparse=sparse,
                       numvals=len(L["vals"]) if sparse else 0, topX=topx)
    sd = {k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray) and k in m.state_dict()}
    m.load_state_dict(sd, strict=False)
    return m


def _layers(bits, K, widths, sparsity, topx, bias=False):
    return [orc.make_layer(bits, K, n, sparsity=sparsity if i != 1 else 0.0, topX=topx if i != 1 else 0, seed=31 + i,
                           nonzero_full_rows=True, bias=bias) for i, n in enumerate(widths)]


@pytest.mark.parametrize("bits", [3, 4])
def test_stacked_buffers_equal_members_side_by_side(bits):
    """oracle(stacked layer) == concat(oracle(member_i)) exactly: same packed words, LUT rows, CSR entries, dense rows.
    Member 1 has no outliers at all (mixed groups must still stack)."""
    K, widths = 256, [64, 128, 192]
    Ls = _layers(bits, K, widths, 0.02, 3, bias=True)
    ms = [_member(L, bias=True) for L in Ls]
    b = fusion.stack_buffers(ms)
    assert b["offsets"] == [0, 64, 192, 384] and b["qweight"].shape == (K // 32 * bits, 384)
    stacked = dict(bits=bits, infeatures=K, outfeatures=384, bias=None,
                   **{k: b[k].numpy() for k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices")})
    x = orc.make_vec(K, seed=3)
    got = orc.forward_f64(stacked, x)
    want = np.concatenate([orc.forward_f64(L, x) for L in Ls], axis=1)
    assert np.array_equal(got, want)
    assert torch.equal(b["bias"], torch.cat([torch.from_numpy(L["bias"]) for L in Ls]))
    assert b["rows"][-1].item() == len(b["cols"]) == sum(len(L["vals"]) for L in Ls if L.get("vals") is not None)


def test_result_cache_protocol():
    """One stacked call per distinct input; each member consumes once; a new / modified x recomputes."""
    K = 64
    ms = [_member(orc.make_layer(4, K, n, seed=n)) for n in (32, 64)]
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
                setattr(self, n, _member(orc.make_layer(4, 64, 64, seed=5)))

    class Mlp(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.gate_proj = _member(orc.make_layer(4, 64, 128, seed=6))
            self.up_proj = _member(orc.make_layer(4, 64, 128, seed=7))
            self.down_proj = _member(orc.make_layer(4, 128, 64, seed=8))

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.self_attn, self.mlp = Attn(), Mlp()
    model = torch.nn.Sequential(Block(), Block())
    groups = fusion.fuse_siblings(model)
    assert len(groups) == 4 and sorted(len(g.members) for g in groups) == [2, 2, 3, 3]
    assert model[0].self_attn.o_proj._sibling_group is None and model[1].mlp.down_proj._sibling_group is None
    assert fusion.fuse_siblings(model) == [], "idempotent"


@pytest.mark.gpu
@pytest.mark.parametrize("bits,K,widths,sp,topx", [(4, 4096, [4096, 4096, 4096], 0.0045, 10), (3, 4096, [11008, 11008], 0.0045, 10),
                                                   (4, 512, [128, 256], 0.0, 0),
                                                   # the middle member has no dense rows: 2 x topX stacked
                                                   (4, 1024, [1024, 1024, 1024], 0.01, 16),   # 32: the topX <= 32 branch at its edge
                                                   (3, 1024, [1024, 1024, 1024], 0.01, 17),   # 34: the general branch
                                                   (4, 1024, [1024, 1024, 1024], 0.01, 70)],  # 140: more than the fused launch takes
                         ids=["w4-qkv", "w3-gateup", "w4-small-dense", "w4-qkv-t16", "w3-qkv-t17", "w4-qkv-t70"])
def test_stacked_launch_matches_members(bits, K, widths, sp, topx):
    Ls = _layers(bits, K, widths, sp, topx)
    ms = [_member(L).cuda() for L in Ls]
    x = torch.from_numpy(orc.make_vec(K, seed=12)).cuda().half().reshape(1, 1, K)
    alone = [m(x) for m in ms]
    g = fusion.SiblingGroup(ms)
    together = [m(x) for m in ms]
    torch.cuda.synchronize()
    assert g.launches == 1
    for L, m, a, t in zip(Ls, ms, alone, together):
        assert t.shape == (1, 1, L["outfeatures"]) and t.dtype == torch.float16
        want = orc.forward_f64(L, x.float().cpu().numpy().reshape(1, K))
        assert rel_err(t.float().cpu().numpy(), want) < REL_TOL
        assert rel_err(t.float().cpu().numpy(), a.float().cpu().numpy()) < REL_TOL
        assert not m.qweight.is_contiguous() or len(widths) == 1  # a view of the stacked matrix, not a copy
    # prefill-shaped input goes through the stacked layer's batched symbols
    xb = torch.from_numpy(orc.make_vec(K, batch=2, seed=13)).cuda().half().reshape(1, 2, K)
    yb = [m(xb) for m in ms]
    for L, y in zip(Ls, yb):
        want = orc.forward_f64(L, xb.float().cpu().numpy().reshape(2, K))
        assert rel_err(y.float().cpu().numpy().reshape(2, -1), want) < REL_TOL
