"""GPU tests of the dequantize (quant_cuda.dequantize / sqllm_dequantize, QuantLinearLUT.dequantize / to_linear,
quantize.dequantize_model).  The truth is the oracle's codebook dequantize (oracle.dequant_f32, golden-pinned) with the CSR entries
added in storage order (np.add.at) and then the dense rows in ascending j, all in fp32, then one rounding: every comparison is bit
for bit."""
import numpy as np
import pytest
import torch

from test_gpu_parity import IDS, SHAPES
from util import abs_sum, bound_ratio, orc, quant_layer, to_torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.float16, torch.bfloat16]


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def truth(L):
    """fp32 [N, K]: codebook, + CSR entries in storage order, + dense rows in ascending j (out-of-range ones ignored)."""
    K, N = L["infeatures"], L["outfeatures"]
    W = np.ascontiguousarray(orc.dequant_f32(L["qweight"], L["lookup_table"], L["bits"]).T)
    if L.get("rows") is not None:
        rows, cols, vals = L["rows"].astype(np.int64), L["cols"], L["vals"]
        ch = np.repeat(np.arange(N), np.diff(rows))
        e = np.arange(rows[0], rows[N])
        keep = (cols[e] >= 0) & (cols[e] < K)
        np.add.at(W, (ch[keep], cols[e][keep]), vals[e][keep])
    if L.get("full_rows") is not None:
        for j, c in enumerate(L["full_row_indices"]):
            if 0 <= c < N:
                W[c] += L["full_rows"][:, j]
    return W


def deq(qc, T, dtype, col0=0, ncols=-1):
    return qc.dequantize(T["qweight"], T["lookup_table"], T["bits"], T.get("rows"), T.get("cols"), T.get("vals"), T.get("full_rows"),
                         T.get("full_row_indices"), dtype=dtype, col0=col0, ncols=ncols)


def bits_of(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def check_all_dtypes(qc, L, T=None):
    """Every output dtype bit-equal to the truth rounded once, and the 16-bit outputs bit-equal to rounding the fp32 output."""
    T = to_torch(L) if T is None else T
    want = torch.from_numpy(truth(L)).cuda()
    w32 = deq(qc, T, torch.float32)
    assert w32.shape == (L["outfeatures"], L["infeatures"])
    assert torch.equal(bits_of(w32), bits_of(want)), int((bits_of(w32) != bits_of(want)).sum())
    for dt in (torch.float16, torch.bfloat16):
        w = deq(qc, T, dt)
        assert w.dtype == dt and torch.equal(bits_of(w), bits_of(want.to(dt))), dt
        assert torch.equal(bits_of(w), bits_of(w32.to(dt))), dt
    return w32


def layer(bits, K, N, sparsity=0.0, topX=0, nz=True, skew=False, seed=0):
    L = orc.make_layer(bits, K, N, sparsity=sparsity, topX=topX, seed=seed, skew=skew, nonzero_full_rows=nz)
    if topX and sparsity == 0:
        L["full_rows"] = L["full_row_indices"] = None
    return L


# ---- shapes ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_parity_shapes_bit_exact(qc, shape, bits):
    _, K, N, sp, topx, nz, skew = shape
    check_all_dtypes(qc, layer(bits, K, N, sp, topx, nz, skew, seed=K + N + bits))


@pytest.mark.parametrize("bits,K,N", [(4, 256, 131072), (3, 64, 131072)])
def test_wide_and_large_layers(qc, bits, K, N):
    check_all_dtypes(qc, layer(bits, K, N, 0.0045, 10, seed=7))


@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("K", [32, 96, 160, 4128, 22016])
@pytest.mark.parametrize("N", [1, 60, 68, 132])
def test_ragged_shapes(qc, bits, K, N):
    check_all_dtypes(qc, layer(bits, K, N, 0.01, min(3, N), seed=K * 7 + N))


# ---- outliers ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [3, 4])
def test_empty_csr_and_no_sparse_buffers(qc, bits):
    L = layer(bits, 256, 132, seed=1)
    w_none = check_all_dtypes(qc, L)
    L["rows"] = np.zeros(133, dtype=np.int32)
    L["cols"] = np.zeros(0, dtype=np.int32)
    L["vals"] = np.zeros(0, dtype=np.float32)
    assert torch.equal(check_all_dtypes(qc, L), w_none)


@pytest.mark.parametrize("bits", [3, 4])
def test_a_3000_entry_row(qc, bits):
    rng = np.random.default_rng(5)
    K, N = 4128, 200
    L = layer(bits, K, N, seed=5)
    counts = rng.integers(0, 4, size=N)
    counts[77] = 3000
    rows = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    cols = np.concatenate([np.sort(rng.choice(K, size=n, replace=False)) for n in counts]).astype(np.int32)
    L.update(rows=rows, cols=cols, vals=rng.standard_normal(len(cols)).astype(np.float32))
    check_all_dtypes(qc, L)


def _dup_layer(bits, seed):
    """A layer whose CSR rows hold duplicate entries, out-of-range columns (negative and >= K) and entries of mixed magnitude
    (so that the order of the duplicates matters in fp32)."""
    rng = np.random.default_rng(seed)
    K, N = 160, 132
    L = layer(bits, K, N, seed=seed)
    counts = rng.integers(0, 12, size=N)
    rows = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    cols = rng.integers(-3, K + 3, size=int(rows[-1])).astype(np.int32)
    for c in range(N):  # sorted rows with many duplicates: columns from a small set
        seg = slice(rows[c], rows[c + 1])
        cols[seg] = np.sort(rng.choice(np.array([-2, 0, 5, 31, 32, 33, 100, K - 1, K, K + 7]), size=counts[c]))
    vals = (rng.standard_normal(len(cols)) * 10.0 ** rng.integers(-6, 2, size=len(cols))).astype(np.float32)
    L.update(rows=rows, cols=cols, vals=vals)
    return L


@pytest.mark.parametrize("bits", [3, 4])
def test_duplicates_out_of_range_and_shuffled_rows(qc, bits):
    L = _dup_layer(bits, seed=11 + bits)
    w_sorted = check_all_dtypes(qc, L)
    rng = np.random.default_rng(3)
    S = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    rows = L["rows"]
    for c in range(L["outfeatures"]):
        p = rows[c] + rng.permutation(rows[c + 1] - rows[c])
        S["cols"][rows[c]:rows[c + 1]] = L["cols"][p]
        S["vals"][rows[c]:rows[c + 1]] = L["vals"][p]
    w_shuf = check_all_dtypes(qc, S)
    # positions with at most one in-range entry do not depend on the order
    hits = np.zeros((L["outfeatures"], L["infeatures"]), dtype=np.int64)
    ch = np.repeat(np.arange(L["outfeatures"]), np.diff(rows))
    ok = (L["cols"] >= 0) & (L["cols"] < L["infeatures"])
    np.add.at(hits, (ch[ok], L["cols"][ok]), 1)
    single = torch.from_numpy(hits <= 1).cuda()
    assert torch.equal(w_shuf[single], w_sorted[single])
    assert (hits > 1).any()


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_csr_arrays_inside_a_larger_buffer(qc, offset):
    L = layer(4, 256, 132, 0.02, 4, seed=offset)
    T = to_torch(L)
    for k in ("cols", "vals"):
        buf = torch.zeros(T[k].numel() + 4, dtype=T[k].dtype, device="cuda")
        buf[offset:offset + T[k].numel()] = T[k]
        T[k] = buf[offset:offset + T[k].numel()]
        assert T[k].data_ptr() % 16 == 4 * offset
    check_all_dtypes(qc, L, T)


# ---- dense rows ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("topx", [1, 33, 128, 300])
@pytest.mark.parametrize("where", ["spread", "channel0", "one_tile", "out_of_range"])
def test_dense_rows(qc, bits, topx, where):
    rng = np.random.default_rng(topx)
    K, N = 160, 200
    L = layer(bits, K, N, 0.01, seed=topx)
    L["full_rows"] = (rng.standard_normal((K, topx)) * 10.0 ** rng.integers(-5, 1, size=(K, topx))).astype(np.float32)
    fri = {"spread": rng.integers(0, N, size=topx), "channel0": np.zeros(topx), "one_tile": rng.integers(64, 70, size=topx),
           "out_of_range": rng.choice(np.array([-5, -1, 0, 3, N - 1, N, N + 4, 2**31 - 1]), size=topx)}[where]
    L["full_row_indices"] = fri.astype(np.int32)
    check_all_dtypes(qc, L)


# ---- column ranges ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [3, 4])
def test_column_ranges_are_slices_of_the_whole(qc, bits):
    L = layer(bits, 416, 300, 0.02, 6, seed=bits)
    T = to_torch(L)
    for dt in DTYPES:
        whole = deq(qc, T, dt)
        for col0, ncols in ((0, 300), (0, 1), (299, 1), (1, 299), (3, 64), (37, 100), (64, 64), (100, 200), (63, 2), (130, -1)):
            part = deq(qc, T, dt, col0, ncols)
            n = 300 - col0 if ncols == -1 else ncols
            assert part.shape == (n, 416) and torch.equal(bits_of(part), bits_of(whole[col0:col0 + n])), (dt, col0, ncols)


# ---- repeatability, graphs, streams -----------------------------------------------------------------------------------------
def test_two_calls_bit_identical(qc):
    T = to_torch(layer(3, 4096, 4096, 0.0045, 10, skew=True, seed=2))
    for dt in DTYPES:
        assert torch.equal(bits_of(deq(qc, T, dt)), bits_of(deq(qc, T, dt)))


def test_cuda_graph_replay_with_new_buffers(qc):
    L = layer(4, 512, 264, 0.01, 5, seed=1)
    T = to_torch(L)
    deq(qc, T, torch.float16)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = deq(qc, T, torch.float16)
    for seed in (2, 3):
        rng = np.random.default_rng(seed)
        L2 = dict(L, qweight=rng.integers(-2**31, 2**31, size=L["qweight"].shape, dtype=np.int64).astype(np.int32),
                  lookup_table=rng.standard_normal(L["lookup_table"].shape).astype(np.float32),
                  vals=rng.standard_normal(L["vals"].shape).astype(np.float32),
                  full_rows=rng.standard_normal(L["full_rows"].shape).astype(np.float32))
        for k in ("qweight", "lookup_table", "vals", "full_rows"):
            T[k].copy_(torch.from_numpy(L2[k]))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits_of(out), bits_of(torch.from_numpy(truth(L2)).cuda().half()))


def test_three_streams_at_once(qc):
    Ts = [to_torch(layer(b, 4096, 4096, 0.0045, 10, seed=s)) for b, s in ((4, 1), (3, 2), (4, 3))]
    want = [deq(qc, T, torch.float16) for T in Ts]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in Ts]
    outs = []
    for T, s in zip(Ts, streams):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            outs.append([deq(qc, T, torch.float16) for _ in range(4)])
    torch.cuda.synchronize()
    for o, w in zip(outs, want):
        assert all(torch.equal(bits_of(x), bits_of(w)) for x in o)


@pytest.mark.parametrize("shape", [(4, 4096, 4096, 0.0045, 10), (3, 11008, 4096, 0.0045, 10), (3, 256, 192, 0.02, 4)])
def test_against_the_forward_oracle(qc, shape):
    """x . W^T in fp64 from the fp32 dequantized W agrees with the fp64 forward oracle within tests/util.py's bound: the matrix
    is the one every forward route multiplies by."""
    bits, K, N, sp, topx = shape
    L = layer(bits, K, N, sp, topx, seed=9)
    x = orc.make_vec(K, batch=4, seed=9)
    W = deq(qc, to_torch(L), torch.float32).cpu().numpy().astype(np.float64)
    got = x.astype(np.float64) @ W.T
    assert bound_ratio(got, orc.forward_f64(L, x), abs_sum(L, x)) <= 1.0


# ---- module ---------------------------------------------------------------------------------------------------------------------
def _module(kind, bits=4, K=256, N=192, seed=0):
    sp, topx = {"plain": (0.0, 0), "biased": (0.0, 0), "sparse": (0.02, 0), "hybrid": (0.02, 6)}[kind]
    L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=seed, nonzero_full_rows=True, bias=kind == "biased")
    return L, quant_layer(L).cuda()


@pytest.mark.parametrize("kind", ["plain", "biased", "sparse", "hybrid"])
def test_module_dequantize_and_to_linear(kind):
    L, m = _module(kind)
    want = torch.from_numpy(truth(L)).cuda()
    for dt in DTYPES:
        w = m.dequantize(dt)
        assert w.dtype == dt and not w.requires_grad and torch.equal(bits_of(w), bits_of(want.to(dt)))
        lin = m.to_linear(dt)
        assert isinstance(lin, torch.nn.Linear) and lin.weight.device == m.qweight.device
        assert torch.equal(lin.weight.data, w)
        if kind == "biased":
            assert lin.bias.dtype == dt and torch.equal(lin.bias.data, m.bias.to(dt))
        else:
            assert lin.bias is None
    assert set(m.to_linear().state_dict()) == ({"weight", "bias"} if kind == "biased" else {"weight"})


def test_module_sibling_members():
    from squeezellm_b200.fusion import fuse_siblings
    mods = torch.nn.Module()
    Ls = {}
    for i, (n, N) in enumerate((("q_proj", 192), ("k_proj", 68), ("v_proj", 132))):
        Ls[n], m = _module("hybrid", N=N, seed=i)
        setattr(mods, n, m)
    groups = fuse_siblings(mods)
    assert len(groups) == 1
    x = torch.from_numpy(orc.make_vec(256, batch=3, seed=1)).cuda()
    for n, L in Ls.items():
        m = getattr(mods, n)
        assert m._sibling_group is not None and not m.qweight.is_contiguous()
        for dt in DTYPES:
            assert torch.equal(bits_of(m.dequantize(dt)), bits_of(torch.from_numpy(truth(L)).cuda().to(dt))), (n, dt)
    y_fused = [getattr(mods, n)(x) for n in Ls]
    groups[0].dissolve()
    for (n, L), y in zip(Ls.items(), y_fused):
        m = getattr(mods, n)
        assert m._sibling_group is None and m.qweight.is_contiguous() and m.qweight._base is None and m.lookup_table._base is None
        assert torch.equal(m.dequantize(torch.float32), torch.from_numpy(truth(L)).cuda())
        assert torch.allclose(m(x), y, rtol=1e-5, atol=1e-6)


def test_module_train_codebook_uses_current_values():
    L, m = _module("hybrid", seed=4)
    params = m.train_codebook(lookup_table=True, vals=True, full_rows=True)
    opt = torch.optim.SGD(params, lr=0.5)
    x = torch.from_numpy(orc.make_vec(256, batch=16, seed=4)).cuda().half()
    before = m.dequantize(torch.float32)
    m(x).float().square().sum().backward()
    opt.step()
    after = m.dequantize(torch.float32)
    assert not after.requires_grad and not torch.equal(before, after)
    cur = dict(L, lookup_table=m.lookup_table.detach().cpu().numpy(), vals=m.vals.detach().cpu().numpy(),
               full_rows=m.full_rows.detach().cpu().numpy())
    assert torch.equal(after, torch.from_numpy(truth(cur)).cuda())
    assert torch.equal(m.to_linear(torch.float32).weight.data, after)


@pytest.mark.parametrize("rows", [1, 8, 2048])
def test_to_linear_forward_matches_the_module(rows):
    L, m = _module("hybrid", K=4096, N=512, seed=rows)
    L["bias"] = None
    x = orc.make_vec(4096, batch=rows, seed=rows)
    xt = torch.from_numpy(x).cuda()
    S, want = abs_sum(L, x), orc.forward_f64(L, x)
    with torch.no_grad():
        y_lin = m.to_linear(torch.float32)(xt).cpu().numpy()
        y_mod = m(xt if rows > 1 else xt.reshape(-1)).reshape(rows, -1).cpu().numpy()
    assert bound_ratio(y_lin, want, S) <= 1.0
    assert bound_ratio(y_mod, want, S) <= 1.0


@pytest.mark.parametrize("bits", [3, 4])
def test_quantize_round_trip(bits):
    from squeezellm_b200.quantize import kmeans_codebook, outlier_threshold, quantize_linear, split_outliers
    torch.manual_seed(bits)
    lin = torch.nn.Linear(512, 200).cuda()
    fisher = torch.rand_like(lin.weight) ** 4
    thr = outlier_threshold(lin.weight, 2.0)
    q = quantize_linear(lin, fisher, bits, threshold=thr, sensitivity=0.45)
    dense, outliers = split_outliers(lin.weight, fisher, thr, 0.45)
    lut, labels = kmeans_codebook(dense, fisher * (dense != 0), bits)
    assert torch.equal(lut, q.lookup_table)
    got = q.dequantize(torch.float32)
    w = lin.weight.detach().float()
    zero = lut.gather(1, lut.abs().argmin(dim=1, keepdim=True))
    at = outliers != 0
    assert int(at.sum()) > 0 and q.numvals == int(at.sum())
    want = torch.where(at, zero + (w - zero), lut.gather(1, labels.long()))
    assert torch.equal(bits_of(got), bits_of(want))


@pytest.mark.parametrize("fuse", [False, True])
def test_dequantize_model_tiny_llama(fuse):
    transformers = pytest.importorskip("transformers")
    from squeezellm_b200 import checkpoint as ck
    from squeezellm_b200.fusion import fuse_siblings
    from squeezellm_b200.quant import QuantLinearLUT
    from squeezellm_b200.quantize import dequantize_model, quantize_model
    cfg = transformers.LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=97, max_position_embeddings=32)
    torch.manual_seed(0)
    model = transformers.LlamaForCausalLM(cfg).eval().half().cuda()
    dense_keys = set(model.state_dict())
    fisher = {f"{n}.weight": torch.rand_like(m.weight, dtype=torch.float32) ** 4 for n, m in ck.find_linear_layers(model).items()}
    quantize_model(model, fisher, 4, outlier_range=3.0, sensitivity=0.45)
    if fuse:
        assert len(fuse_siblings(model)) == 4
    ids = torch.randint(0, 97, (2, 12), device="cuda")
    with torch.no_grad():
        logits_q = model(ids).logits.float()
    names = dequantize_model(model, torch.float16)
    assert len(names) == 14 and "lm_head" not in names
    assert set(model.state_dict()) == dense_keys
    assert not any(isinstance(m, QuantLinearLUT) or getattr(m, "_sibling_group", None) is not None for m in model.modules())
    ref = transformers.LlamaForCausalLM(cfg).eval().half().cuda()
    ref.load_state_dict(model.state_dict())
    with torch.no_grad():
        logits_d = model(ids).logits.float()
        logits_r = ref(ids).logits.float()
    assert torch.equal(logits_d, logits_r)
    assert float((logits_d - logits_q).abs().max()) <= 2e-2 * float(logits_q.abs().max())


# ---- argument checks of the binding ------------------------------------------------------------------------------------------
def test_binding_rejects_bad_arguments(qc):
    T = to_torch(layer(4, 256, 132, 0.02, 4, seed=0))
    with pytest.raises(RuntimeError, match="dtype must be torch.float32, torch.float16 or torch.bfloat16"):
        deq(qc, T, torch.int8)
    for col0, ncols in ((-1, 4), (0, 0), (0, 133), (130, 3), (0, -2), (132, -1)):
        with pytest.raises(RuntimeError, match=r"dequantize: columns \[col0="):
            deq(qc, T, torch.float16, col0, ncols)
    with pytest.raises(RuntimeError, match="bits must be 3 or 4"):
        deq(qc, dict(T, bits=5), torch.float16)
    with pytest.raises(RuntimeError, match="qweight must be a contiguous CUDA tensor"):
        deq(qc, dict(T, qweight=T["qweight"][:, ::2]), torch.float16)
    with pytest.raises(RuntimeError, match="lookup_table must be"):
        deq(qc, dict(T, lookup_table=T["lookup_table"][:-1]), torch.float16)
    with pytest.raises(RuntimeError, match="lookup_table must have dtype"):
        deq(qc, dict(T, lookup_table=T["lookup_table"].double()), torch.float16)
    with pytest.raises(RuntimeError, match="rows must have num_rows"):
        deq(qc, dict(T, rows=T["rows"][:-1]), torch.float16)
    with pytest.raises(RuntimeError, match="cols and vals differ"):
        deq(qc, dict(T, vals=T["vals"][:-1]), torch.float16)
    with pytest.raises(RuntimeError, match="rows given without cols / vals"):
        deq(qc, dict(T, cols=None), torch.float16)
    with pytest.raises(RuntimeError, match="full_rows must be"):
        deq(qc, dict(T, full_rows=T["full_rows"][:-32]), torch.float16)
    with pytest.raises(RuntimeError, match="full_rows given without full_row_indices"):
        deq(qc, dict(T, full_row_indices=None), torch.float16)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        deq(qc, dict(T, vals=T["vals"].cpu()), torch.float16)
