"""bf16 sequences (runtime.DecodeSequence(dtype=torch.bfloat16), sqllm_sequence_create_dt): the chains of tests/test_sequence_gpu.py with
bf16 activations.  Every item is checked per element against the fp64 oracle applied to the bf16 vector it actually consumed, with the
condition-aware bound of tests/util.py (bound_ratio <= 1, bf16 output rounding); the whole chain in the max norm against the oracle chain
with bf16 hand-overs and against the same layers called one by one through QuantLinearLUT on one bf16 row."""
import numpy as np
import pytest
import torch

from test_sequence_gpu import CASES, IDS, _chain
from util import OUT_ROUNDING, REL_TOL, abs_sum, bound_ratio, orc, to_torch

pytestmark = pytest.mark.gpu

R_BF16, ETA_BF16 = OUT_ROUNDING["bfloat16"]
# Chain metric: outputs are bf16, so a hand-over or an output that the oracle rounds to the neighbouring bf16 value is one bf16 step
# apart (at most 2^-7 of the value); two such steps of the largest output.
CHAIN_TOL = 2 * 2.0 ** -7


def bf16_np(a):
    """numpy -> its bf16 rounding, as fp64 numpy."""
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).bfloat16().double().numpy()


def _seq(mods, dims, mode="exact", dtype=torch.bfloat16):
    from squeezellm_b200.runtime import DecodeSequence
    seq = DecodeSequence(dims[0][0], "cuda", lut_mode=mode, dtype=dtype)
    vecs, prev = [], seq.input
    for m, (K, N, off) in zip(mods, dims):
        prev = seq.matvec(m, prev[off:off + K])
        vecs.append(prev)
    seq.compile(outputs=vecs)
    return seq


def _bias(b, i):
    return None if b is None else b[i]


def oracle_chain_bf16(layers, dims, x, biases=None):
    """The fp64 oracle chain with bf16 hand-overs (each output rounded to bf16 once, the bias inside the sum)."""
    outs, prev = [], None
    for i, (L, (K, N, off)) in enumerate(zip(layers, dims)):
        xin = x if prev is None else prev[off:off + K]
        b = _bias(biases, i)
        y = orc.forward_f64(L, xin.astype(np.float32).reshape(1, K), mul_init=None if b is None else b[None, :]).reshape(N)
        prev = bf16_np(y)
        outs.append(prev)
    return outs


def check_items(got_all, layers, dims, x0, biases=None):
    """Per item, per element: the bound against the oracle on the bf16 vector the item consumed (x0, or its predecessor's output)."""
    worst = 0.0
    for i, (L, (K, N, off)) in enumerate(zip(layers, dims)):
        xin = (x0 if i == 0 else got_all[i - 1][off:off + K]).astype(np.float32).reshape(1, K)
        b = _bias(biases, i)
        want = orc.forward_f64(L, xin, mul_init=None if b is None else b[None, :]).reshape(N)
        S = abs_sum(L, xin, b).reshape(N)
        assert np.isfinite(got_all[i]).all(), f"item {i}: non-finite output"
        ratio = bound_ratio(got_all[i], want, S, want, R_BF16, eta=ETA_BF16)
        assert ratio <= 1.0, f"item {i}: bound ratio {ratio:.3f} against the oracle on the item's own input"
        worst = max(worst, ratio)
    return worst


def max_norm(got, want):
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _case_chain(case):
    bits, dims, sp, topX = case[:4]
    layers, mods = _chain(bits, dims, sp, topX, seed=bits * 100 + len(dims))
    rep_n = case[4] if len(case) > 4 else 1
    return bits, dims * rep_n, layers * rep_n, mods * rep_n


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_bf16_sequence_matches_oracle_and_layer_by_layer(case):
    bits, dims, layers, mods = _case_chain(case)
    x = bf16_np(orc.make_vec(dims[0][0], seed=5).reshape(-1))
    seq = _seq(mods, dims)
    assert seq.x.dtype == torch.bfloat16 and all(o.dtype == torch.bfloat16 for o in seq.outputs)
    seq.x.copy_(torch.from_numpy(x).cuda())
    # the same layers one by one through the module path (one bf16 row: the one-GEMV kernel, bias inside the sum)
    ys, cur = [], torch.from_numpy(x).cuda().bfloat16()
    for m, (K, N, off) in zip(mods, dims):
        cur = m(cur[off:off + K].clone() if ys else cur)
        assert cur.dtype == torch.bfloat16
        ys.append(cur.double().cpu().numpy())
    x_half = x * 0.5  # exact in bf16
    for rep in range(3):  # replays: the tags of the previous token must not be taken for this one's
        x0 = x if rep < 2 else x_half
        if rep == 2:
            seq.x.copy_(torch.from_numpy(x_half).cuda())
        outs = [o.clone() for o in seq.replay()]
        torch.cuda.synchronize()
        assert not seq.error(), "a bounded in-kernel wait of the sequence gave up"
        got_all = [o.double().cpu().numpy() for o in outs]
        check_items(got_all, layers, dims, x0)
        want = oracle_chain_bf16(layers, dims, x0)
        for i, (got, w) in enumerate(zip(got_all, want)):
            assert max_norm(got, w) < CHAIN_TOL, f"rep {rep} item {i}: max-norm error {max_norm(got, w):.3e} vs the oracle chain"
            if rep < 2:
                assert max_norm(got, ys[i]) < CHAIN_TOL, f"rep {rep} item {i}: {max_norm(got, ys[i]):.3e} vs the module path"


SMALL = CASES[1]  # w4, four items, CSR outliers and dense rows


def _with_bias(layers, mods, seed, scale=1.0):
    """Give every module an fp32 bias N(0, scale^2); returns the biases."""
    rng = np.random.default_rng(seed)
    biases = []
    for L, m in zip(layers, mods):
        b = (rng.standard_normal(L["outfeatures"]) * scale).astype(np.float32)
        m.bias = torch.from_numpy(b).cuda()
        biases.append(b)
    return biases


def test_bf16_activations_beyond_the_fp16_range():
    """|x| ~ 1e5 through the whole chain (the codebook keeps |y| ~ |x|): fp16 would give inf; bf16 stays finite and inside the bound,
    the bias inside the fp32 sum."""
    bits, dims, layers, mods = _case_chain(SMALL)
    biases = _with_bias(layers, mods, seed=3, scale=1e4)
    x = bf16_np(orc.make_vec(dims[0][0], seed=8).reshape(-1) * 1e5)
    assert np.abs(x).max() > 65504
    seq = _seq(mods, dims)
    seq.x.copy_(torch.from_numpy(x).cuda())
    got_all = [o.double().cpu().numpy() for o in seq.replay()]
    assert not seq.error()
    assert max(np.abs(g).max() for g in got_all) > 65504
    check_items(got_all, layers, dims, x, biases)
    for i, (got, w) in enumerate(zip(got_all, oracle_chain_bf16(layers, dims, x, biases))):
        assert max_norm(got, w) < CHAIN_TOL, i


def test_bf16_fp16_table_mode_keeps_the_exact_codebook():
    """lut_mode="fp16": a bf16 sequence still runs the exact fp32 codebook, so it meets the bound of the exact oracle."""
    bits, dims, layers, mods = _case_chain(SMALL)
    x = bf16_np(orc.make_vec(dims[0][0], seed=9).reshape(-1))
    for mode in ("fp16", "exact"):
        seq = _seq(mods, dims, mode=mode)
        seq.x.copy_(torch.from_numpy(x).cuda())
        got_all = [o.double().cpu().numpy() for o in seq.replay()]
        assert not seq.error()
        check_items(got_all, layers, dims, x)


def test_bf16_sequence_in_cuda_graph():
    from squeezellm_b200.runtime import GraphedDecodeStep
    bits, dims, layers, mods = _case_chain(SMALL)
    seq = _seq(mods, dims)
    runner = GraphedDecodeStep(lambda x: seq.replay()[-1], seq.x, warmup=2, static_input=True)
    for s in (1, 2, 3):
        x = bf16_np(orc.make_vec(dims[0][0], seed=s).reshape(-1))
        y = runner(torch.from_numpy(x).bfloat16()).clone().double().numpy()
        w = oracle_chain_bf16(layers, dims, x)[-1]
        assert max_norm(y, w) < CHAIN_TOL
    assert not seq.error()


def test_fp16_and_bf16_sequences_interleaved_on_one_stream():
    """Two sequences over the same layers, one fp16 and one bf16, replayed in turn: each keeps its own words, tags and results."""
    bits, dims, layers, mods = _case_chain(SMALL)
    biases = _with_bias(layers, mods, seed=4)
    s16, sbf = _seq(mods, dims, dtype=torch.float16), _seq(mods, dims)
    for s in (1, 2):
        x = bf16_np(orc.make_vec(dims[0][0], seed=20 + s).reshape(-1))
        x16 = x.astype(np.float16)
        s16.x.copy_(torch.from_numpy(x16).cuda())
        sbf.x.copy_(torch.from_numpy(x).cuda())
        o16 = [o.clone() for o in s16.replay()]
        obf = [o.clone() for o in sbf.replay()]
        o16b = [o.clone() for o in s16.replay()]
        torch.cuda.synchronize()
        assert not s16.error() and not sbf.error()
        assert all(o.dtype == torch.float16 for o in o16) and all(o.dtype == torch.bfloat16 for o in obf)
        got = [o.double().cpu().numpy() for o in obf]
        check_items(got, layers, dims, x, biases)
        for g, w in zip(got, oracle_chain_bf16(layers, dims, x, biases)):
            assert max_norm(g, w) < CHAIN_TOL
        # fp16 chain with fp16 hand-overs (test_sequence_gpu's oracle, bias added per item here)
        prev = None
        for i, (L, (K, N, off)) in enumerate(zip(layers, dims)):
            xin = x16.astype(np.float64) if prev is None else prev[off:off + K]
            prev = orc.forward_f64(L, xin.astype(np.float32).reshape(1, K), mul_init=biases[i][None, :]).reshape(N)
            prev = prev.astype(np.float16).astype(np.float64)
            for o in (o16, o16b):
                assert max_norm(o[i].double().cpu().numpy(), prev) < 2 * REL_TOL, (s, i)


def _item(T, x_ext, N, bits=4):
    return (T["qweight"], T["lookup_table"], bits, None, T.get("rows"), T.get("cols"), T.get("vals"), T.get("full_rows"),
            T.get("full_row_indices"), -1, 0, x_ext, 1, N)


def test_dtype_mismatches_are_rejected():
    from squeezellm_b200.quant import quant_cuda as qc
    from squeezellm_b200.runtime import DecodeSequence
    K, N = 512, 256
    T = to_torch(orc.make_layer(4, K, N, sparsity=0.01, topX=3, seed=3, nonzero_full_rows=True))
    xb = torch.zeros(K, device="cuda", dtype=torch.bfloat16)
    xh = torch.zeros(K, device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="x_ext must be fp16"):
        qc.sequence_create([_item(T, xb, N)], [], "exact", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="x_ext must be bf16"):
        qc.sequence_create([_item(T, xh, N)], [], "exact", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="destination must be a contiguous bf16"):
        qc.sequence_create([_item(T, xb, N)], [(0, torch.zeros(N, device="cuda", dtype=torch.float16))], "exact", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="destination must be a contiguous fp16"):
        qc.sequence_create([_item(T, xh, N)], [(0, torch.zeros(N, device="cuda", dtype=torch.bfloat16))], "exact")
    with pytest.raises(RuntimeError, match="dtype must be torch.float16 or torch.bfloat16"):
        qc.sequence_create([_item(T, xh, N)], [], "exact", dtype=torch.float32)
    with pytest.raises(ValueError, match="dtype must be"):
        DecodeSequence(K, "cuda", dtype=torch.float32)
    # the matching pairs are taken
    for x, dt in ((xb, torch.bfloat16), (xh, torch.float16)):
        h = qc.sequence_create([_item(T, x, N)], [(0, torch.zeros(N, device="cuda", dtype=dt))], "exact", dtype=dt)
        qc.sequence_destroy(h)
