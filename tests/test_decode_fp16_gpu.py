"""fp16 decode per element against the fp64 oracle: one fp16 row through the one-GEMV kernel (lutgemv2_kernel in the default mode, the
multi-row kernel at one row in the deterministic one) with the exact table and the fp16 pair table, the sequence kernel
(lutgemv_seq_kernel) in both table modes, and the exchange entry point on one GPU.  The truth is the fp64 oracle with the bias inside the
sum, on the fp16 values the kernel consumed (a sequence item: its own input, the exported output of its predecessor) and, where the pair
table runs, on the codebook rounded to fp16 (round to nearest even).  The metric is the per-element bound of tests/util.py
(bound_ratio <= 1) with the fp16 output rounding; a non-finite output fails it.  Activations are make_activations rows: a 1e-3 row with
fp16 subnormals, a 1e2 row with massive channels, a one-entry row and an ordinary one.  Each test records its worst ratio."""
import numpy as np
import pytest
import torch

from test_decode_bf16_gpu import ONE_ROW_CASES, Mode, _cid, _edge_layer, _torch_layer, fused_dt, lib  # noqa: F401  (lib: fixture)
from test_sequence_bf16_gpu import _seq
from test_sequence_gpu import CASES, IDS, _chain
from test_zz_exchange_gpu import DATA, ERROR, EXCHANGE_IDS, EXCHANGE_LAYERS, FLAG, STATE, exchange_layer
from util import E_ACC, OUT_ROUNDING, abs_sum, bound_ratio, make_activations, orc, quant_layer

pytestmark = pytest.mark.gpu

R16, ETA16 = OUT_ROUNDING["float16"]
ROWS = [0, 1, 3, 5]          # make_activations: 1e-3 (fp16 subnormals), 1e2 (massive channels), one entry, ordinary


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


def fp16_table(L):
    """L with its codebook rounded to fp16 (round to nearest even): what the pair table multiplies."""
    return dict(L, lookup_table=L["lookup_table"].astype(np.float16).astype(np.float32))


def truth(L, x, bias):
    """(want, S) of the rows x [M, K]: the fp64 oracle with the bias inside the sum, and the condition of every output.  Every layer
    and row here keeps |want| below the largest fp16 (the 1e2 row with its massive channels included), so fp16 y is finite."""
    want = orc.forward_f64(L, x, mul_init=None if bias is None else bias[None, :])
    assert np.abs(want).max() < 65504.0
    return want, abs_sum(L, x, bias)


def check(got, want, S, y_dtype):
    """bound_ratio of got against (want, S) with y_dtype's output rounding; fails on a non-finite output or a ratio above 1."""
    got = got.double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, dtype=np.float64)
    got = got.reshape(want.shape)
    assert np.isfinite(got).all(), f"{np.count_nonzero(~np.isfinite(got))} non-finite outputs where the oracle is finite"
    r, eta = OUT_ROUNDING[y_dtype]
    ratio = bound_ratio(got, want, S, want, r, E_ACC, eta)
    assert ratio <= 1.0, f"bound ratio {ratio:.3f}"
    return ratio


# ---- one row ---------------------------------------------------------------------------------------------------------------------
_one = {}


def one_row_case(case):
    """The edge layer of `case`, its GPU tensors, the rows (fp32 numpy and fp16 on the GPU) and the truths per table."""
    if case not in _one:
        _one.clear()
        L, off = _edge_layer(case)
        x = make_activations(L["infeatures"], 6, seed=L["infeatures"] + L["bits"])[ROWS]
        _one[case] = dict(L=L, T=_torch_layer(L, off), x=x, xt=torch.from_numpy(x).cuda().half(), truth={})
    return _one[case]


def case_truth(c, pair):
    if pair not in c["truth"]:
        c["truth"][pair] = truth(fp16_table(c["L"]) if pair else c["L"], c["x"], c["L"]["bias"])
    return c["truth"][pair]


def run_rows(lib, c, y_dtype):
    return torch.stack([fused_dt(lib, c["L"], c["T"], c["xt"][i], y_dtype, bias=c["T"]["bias"]) for i in range(len(ROWS))])


@pytest.mark.parametrize("table", ["exact", "fp16"])
@pytest.mark.parametrize("case", ONE_ROW_CASES, ids=[_cid(c) for c in ONE_ROW_CASES])
def test_one_row_fp16_vs_oracle(lib, record, case, table):
    """fp32 and fp16 y in both summation modes.  The pair table (fp16 table mode) is the default mode's: the deterministic mode's
    multi-row kernel and layers narrower than one strip keep the exact codebook.  Deterministic fp16 y is bit-equal to the fp32 y
    rounded to nearest."""
    c = one_row_case(case)
    worst = 0.0
    lib.sqllm_set_lut_mode(int(table == "fp16"))
    try:
        for det in (0, 1):
            pair = table == "fp16" and det == 0 and c["L"]["outfeatures"] >= 64
            want, S = case_truth(c, pair)
            with Mode(lib, det):
                y32 = run_rows(lib, c, torch.float32)
                y16 = run_rows(lib, c, torch.float16)
            worst = max(worst, check(y32, want, S, "float32"), check(y16, want, S, "float16"))
            if det:
                assert y16.dtype == torch.float16 and torch.equal(y16, y32.half()), "fp16 y is not the fp32 y rounded to nearest"
    finally:
        lib.sqllm_set_lut_mode(0)
    record("worst_bound_ratio", worst)


def stress_codebook(kind, K=4096, N=1024, bits=4):
    """A layer whose codebook tests the pair table's fp16 rounding: "subnormal" puts half of every channel's centroids at ~1e-6 (fp16
    subnormals) next to ~1e-1; "halfway" puts every centroid exactly between two fp16 values, so ties-to-even decides each one."""
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=40 + len(kind), nonzero_full_rows=True, bias=True)
    rng = np.random.default_rng(41)
    lut = L["lookup_table"].astype(np.float64)
    if kind == "subnormal":
        lut[:, : lut.shape[1] // 2] = rng.standard_normal((N, lut.shape[1] // 2)) * 1e-6
        lut[:, lut.shape[1] // 2:] *= 5.0
        h = lut.astype(np.float32).astype(np.float16)
        assert (np.abs(h[:, : lut.shape[1] // 2]) < np.float16(2.0 ** -14)).all()
    else:
        h = lut.astype(np.float32).astype(np.float16)
        lut = (h.astype(np.float64) + np.nextafter(h, np.float16(np.inf)).astype(np.float64)) / 2
        assert np.array_equal(lut.astype(np.float32).astype(np.float64), lut)
        odd = (h.view(np.uint16) & 1).astype(bool)
        assert 0.3 < odd.mean() < 0.7  # ties that go up and ties that go down
    L["lookup_table"] = lut.astype(np.float32)
    return L


@pytest.mark.parametrize("kind", ["subnormal", "halfway"])
def test_pair_table_codebook_stress(lib, record, kind):
    L = stress_codebook(kind)
    x = make_activations(L["infeatures"], 6, seed=42)[ROWS]
    c = dict(L=L, T=_torch_layer(L, 0), x=x, xt=torch.from_numpy(x).cuda().half(), truth={})
    want, S = case_truth(c, True)
    lib.sqllm_set_lut_mode(1)
    try:
        worst = max(check(run_rows(lib, c, dt), want, S, name) for dt, name in ((torch.float32, "float32"), (torch.float16, "float16")))
    finally:
        lib.sqllm_set_lut_mode(0)
    record("worst_bound_ratio", worst)


def test_pair_table_through_quantlinearlut(record):
    """One fp16 row through QuantLinearLUT (quant_cuda.lutgemv_fused, the bias inside the sum) under set_lut_mode("fp16")."""
    from squeezellm_b200.quant import quant_cuda as qc
    L = orc.make_layer(4, 4096, 4096, sparsity=0.0045, topX=10, seed=43, nonzero_full_rows=True, bias=True)
    x = make_activations(4096, 6, seed=43)[ROWS]
    m = quant_layer(L).cuda()
    want, S = truth(fp16_table(L), x, L["bias"])
    qc.set_lut_mode("fp16")
    try:
        with torch.no_grad():
            y = torch.stack([m(torch.from_numpy(x[i]).cuda().half()) for i in range(len(ROWS))])
        torch.cuda.synchronize()
    finally:
        qc.set_lut_mode("exact")
    assert y.dtype == torch.float16 and not qc.workspace_error()
    record("worst_bound_ratio", check(y, want, S, "float16"))


# ---- the sequence kernel ----------------------------------------------------------------------------------------------------------
def check_items(got_all, layers, dims, x0, pair, biases=None):
    """Per item, per element: the bound against the oracle on the fp16 vector the item consumed (x0, or its predecessor's exported
    output), on the fp16-rounded codebook where the pair table runs."""
    worst = 0.0
    for i, (L, (K, N, off)) in enumerate(zip(layers, dims)):
        xin = (x0 if i == 0 else got_all[i - 1][off:off + K]).astype(np.float32).reshape(1, K)
        want, S = truth(fp16_table(L) if pair else L, xin, None if biases is None else biases[i])
        try:
            worst = max(worst, check(got_all[i], want, S, "float16"))
        except AssertionError as e:
            raise AssertionError(f"item {i}: {e}") from None
    return worst


def replay_rows(seq, layers, dims, mode, rows, biases=None):
    """x0 = each of `rows` (fp16-exact) in successive replays of seq; every item checked after each; returns the worst ratio."""
    worst = 0.0
    for j, x0 in enumerate(rows):
        seq.x.copy_(torch.from_numpy(x0).cuda().half())
        outs = [o.clone() for o in seq.replay()]
        torch.cuda.synchronize()
        assert not seq.error(), f"replay {j}: a bounded in-kernel wait of the sequence gave up"
        got_all = [o.double().cpu().numpy() for o in outs]
        try:
            worst = max(worst, check_items(got_all, layers, dims, x0, mode == "fp16", biases))
        except AssertionError as e:
            raise AssertionError(f"replay {j} ({mode} table): {e}") from None
    return worst


_chains = {}


def case_chain(case):
    """(dims, layers, modules) of a test_sequence_gpu case, as its test builds them (the same seeds)."""
    key = repr(case)
    if key not in _chains:
        _chains.clear()
        bits, dims, sp, topX = case[:4]
        layers, mods = _chain(bits, dims, sp, topX, seed=bits * 100 + len(dims))
        rep_n = case[4] if len(case) > 4 else 1
        _chains[key] = (dims * rep_n, layers * rep_n, mods * rep_n)
    return _chains[key]


def chain_rows(K, seed):
    return make_activations(K, 6, seed=seed)[[0, 1, 5]]


@pytest.mark.parametrize("mode", ["exact", "fp16"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_sequence_items_fp16_vs_oracle(record, case, mode):
    """Every chain of tests/test_sequence_gpu.py with x0 = the 1e-3, the 1e2 and an ordinary row in successive replays."""
    dims, layers, mods = case_chain(case)
    seq = _seq(mods, dims, mode=mode, dtype=torch.float16)
    record("worst_bound_ratio", replay_rows(seq, layers, dims, mode, chain_rows(dims[0][0], seed=len(dims))))


def _shim(L, T):
    """A QuantLinearLUT over L's GPU tensors T whose _sparse_args gives T's outliers as they are (offset views, dense rows without
    CSR, none at all), as test_sequence_gpu's DenseRowsOnly does."""
    from squeezellm_b200.quant import QuantLinearLUT

    class Shim(QuantLinearLUT):
        def _sparse_args(self):
            return T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"]

    return Shim.from_buffers(L["bits"], {k: T[k] for k in ("qweight", "lookup_table", "bias")})


EDGE_ITEMS = [c for c in ONE_ROW_CASES if not (c[0] == "shape" and c[2] < 64)]  # a sequence item has at least one strip


@pytest.mark.parametrize("mode", ["exact", "fp16"])
@pytest.mark.parametrize("case", EDGE_ITEMS, ids=[_cid(c) for c in EDGE_ITEMS])
def test_sequence_edge_layer_then_a_slice(record, case, mode):
    """Item 0: an outlier edge layer of the one-row tests (fed through a shim: offset CSR views, empty CSR, no sparse buffers, a
    3000-entry row, topX 1 to 128 on channel 0); item 1 reads the last up-to-256 outputs of item 0 (the ragged last strip)."""
    c = one_row_case(case)
    L0, T0 = c["L"], c["T"]
    N0 = L0["outfeatures"]
    K1 = min(256, N0 // 64 * 64)
    off = (N0 - K1) // 4 * 4
    L1 = orc.make_layer(L0["bits"], K1, 192, sparsity=0.02, topX=3, seed=N0, nonzero_full_rows=True, bias=True)
    T1 = _torch_layer(L1, 0)
    layers, dims = [L0, L1], [(L0["infeatures"], N0, 0), (K1, 192, off)]
    seq = _seq([_shim(L0, T0), _shim(L1, T1)], dims, mode=mode, dtype=torch.float16)
    record("worst_bound_ratio", replay_rows(seq, layers, dims, mode, c["x"], biases=[L0["bias"], L1["bias"]]))


def test_sequence_wide_item_with_csr_outliers(record):
    """A 131072-column item with 0.45 % CSR outliers (about 1000 CSR rows per CTA) and 128 dense rows in late-owned strips, then an item
    that reads its last 4096 outputs, in both table modes."""
    dims = [(128, 131072, 0), (4096, 768, 126976), (768, 256, 0)]
    layers, mods = _chain(4, dims, 0.0045, 128, seed=131)
    assert len(layers[0]["vals"]) > 0.004 * 128 * 131072
    worst = 0.0
    for mode in ("exact", "fp16"):
        seq = _seq(mods, dims, mode=mode, dtype=torch.float16)
        worst = max(worst, replay_rows(seq, layers, dims, mode, chain_rows(128, seed=131)))
    record("worst_bound_ratio", worst)


def test_sequence_fp16_biases(record):
    """CASES[1] with biases that are fp16 values from fp16 subnormals to 1e3 (the module holds them in fp32, the kernel's bias type),
    in both table modes; an fp16 bias tensor itself is refused."""
    dims, layers, mods = case_chain(CASES[1])
    rng = np.random.default_rng(7)
    biases = []
    for L, m in zip(layers, mods):
        b = rng.standard_normal(L["outfeatures"]) * 10.0 ** rng.uniform(-7, 3, size=L["outfeatures"])
        b = b.astype(np.float16).astype(np.float32)
        assert (np.abs(b[b != 0]) < 2.0 ** -14).any()
        m.bias = torch.from_numpy(b).cuda()
        biases.append(b)
    worst = 0.0
    try:
        for mode in ("exact", "fp16"):
            seq = _seq(mods, dims, mode=mode, dtype=torch.float16)
            worst = max(worst, replay_rows(seq, layers, dims, mode, chain_rows(dims[0][0], seed=8), biases))
        mods[0].bias = mods[0].bias.half()
        with pytest.raises(RuntimeError, match="bias must have dtype Float"):
            _seq(mods, dims, dtype=torch.float16)
    finally:
        for m in mods:
            m.bias = None
    record("worst_bound_ratio", worst)


# ---- the exchange entry point on one GPU --------------------------------------------------------------------------------------------
EXCHANGE_EDGES = [c for c in ONE_ROW_CASES if c[0] in ("topx", "offset")]


def exchange_case(p):
    """(L, T, x rows) of an exchange layer (test_zz_exchange_gpu) or an edge layer of the one-row tests."""
    if p[0] in ("topx", "offset"):
        c = one_row_case(p)
        return c["L"], c["T"], c["x"]
    L = exchange_layer(*p)
    x = make_activations(L["infeatures"], 6, seed=L["infeatures"])[ROWS]
    return L, _torch_layer(L, 0), x


@pytest.mark.parametrize("p", EXCHANGE_LAYERS + EXCHANGE_EDGES, ids=EXCHANGE_IDS + [_cid(c) for c in EXCHANGE_EDGES])
def test_exchange_world1_fp16_vs_oracle(record, p):
    """The arena values (fp16) of world = 1, members = 1 (or the stacked width of the exchange layers) in both table modes."""
    from squeezellm_b200.quant import quant_cuda as qc
    L, T, x = exchange_case(p)
    N = L["outfeatures"]
    members = p[3] if p[0] not in ("topx", "offset") else 1
    w = N // members
    arena = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    base = torch.tensor([arena.data_ptr()], dtype=torch.int64, device="cuda")
    worst = 0.0
    for mode in ("exact", "fp16"):
        pair = mode == "fp16" and N >= 64
        want, S = truth(fp16_table(L) if pair else L, x, L["bias"])
        got = []
        qc.set_lut_mode(mode)
        try:
            for i in range(len(ROWS)):
                arena[DATA:DATA + 2 * N].zero_()
                qc.lutgemv_fused_exchange(torch.from_numpy(x[i]).cuda().half(), T["qweight"], T["lookup_table"], L["bits"], T["bias"],
                                          T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"], base.data_ptr(),
                                          DATA, FLAG, STATE, ERROR, 1, 0, members, w)
                torch.cuda.synchronize()
                got.append(arena[DATA:DATA + 2 * N].view(torch.float16).float().cpu().numpy())
                assert int(arena[ERROR:ERROR + 4].view(torch.int32).item()) == 0
        finally:
            qc.set_lut_mode("exact")
        try:
            worst = max(worst, check(np.stack(got), want, S, "float16"))
        except AssertionError as e:
            raise AssertionError(f"{mode} table: {e}") from None
    record("worst_bound_ratio", worst)
