"""The tensor-core LUT-GEMM for fp32 x (`sqllm_lutgemm_fused_f32`, `quant_cuda.lutgemm_fused_f32`, csrc/lutgemm_tc.cuh with x and the
weights each split into three bf16 parts) that runs fp32 inputs of QuantLinearLUT.FP32_TC_MIN_ROWS or more rows.  The truth is the
fp64 oracle on the fp32 activations themselves, which here carry full 24-bit mantissas (so the third part of x is in play); the
metric is the per-element bound of tests/util.py (bound_ratio <= 1, E_ACC) beside rel_err < TIGHT_TOL, on the fp32 output.
Covered: every parity shape at both bit widths and the row counts at the tile edges, 2048- and 2049-row prefills, numerics stress
(1e-30 to 1e30 rows, x whose parts are bf16 subnormals, tiny next to large centroids, CSR and dense-row edge cases, ragged K and N),
reproducibility, streams and graphs, the module routing and training, the batched route's second pass over a 2049-row batch, and an
fp32 Llama model as the reference's loader builds it."""
import ctypes

import numpy as np
import pytest
import torch

from test_backward_gpu import _module
from test_error_bound_host import SHAPES as BOUND_SHAPES
from util import (E_ACC, TIGHT_TOL, Args, abs_layer, abs_sum, bound_ratio, load_lib, make_activations, orc, rel_err,
                  to_torch)

pytestmark = pytest.mark.gpu


def full_mantissa(x, seed=0):
    """fp32 activations with all 24 bits in use: x (e.g. make_activations' fp16-exact rows) times 1 + N(0, 1e-3), zeros kept."""
    rng = np.random.default_rng(seed + 777)
    return (x.astype(np.float64) * (1.0 + 1e-3 * rng.standard_normal(x.shape))).astype(np.float32)


def make_x(K, M, seed=0):
    return full_mantissa(make_activations(K, M, seed=seed), seed)


def parts(x):
    """The three bf16 parts of fp32 x (numpy), as the kernel splits it."""
    t = torch.from_numpy(np.ascontiguousarray(x))
    h = t.bfloat16().float()
    m = (t - h).bfloat16().float()
    lo = (t - h - m).bfloat16().float()
    return h.numpy(), m.numpy(), lo.numpy()


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemm_fused_f32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def f32_call(lib, L, x, bias=None, T=None, stream=None):
    """sqllm_lutgemm_fused_f32 on the layer dict L (numpy; T: its torch tensors) and x [M, K] (numpy or torch cuda fp32) -> y [M, N]
    (torch, fp32)."""
    T = to_torch(L) if T is None else T
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    M, N = x.shape[0], L["outfeatures"]
    y = torch.empty((M, N), device="cuda", dtype=torch.float32)
    a = Args(bits=L["bits"], in_features=L["infeatures"], out_features=N, batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    b = None if bias is None else torch.from_numpy(bias).cuda()
    s = torch.cuda.current_stream() if stream is None else stream
    rc = lib.sqllm_lutgemm_fused_f32(ctypes.byref(a), x.data_ptr(), y.data_ptr(), None if b is None else b.data_ptr(), s.cuda_stream)
    assert rc == 0, lib.sqllm_last_error()
    if stream is None:
        torch.cuda.synchronize()
    return y


def check(got, L, x, bias=None, want=None, S=None, old=True, eta=0.0):
    """bound_ratio <= 1 (E_ACC, fp32 output) and rel_err < TIGHT_TOL of got [M, N] against the oracle on the fp32 rows x."""
    got = got.float().cpu().numpy() if isinstance(got, torch.Tensor) else got
    mul = None if bias is None else bias[None, :]
    want = orc.forward_f64(L, x, mul_init=mul) if want is None else want
    S = abs_sum(L, x, bias) if S is None else S
    ratio = bound_ratio(got, want, S, eta=eta)
    assert ratio <= 1.0, ratio
    if old:
        e = rel_err(got, want)
        assert e < TIGHT_TOL, e
    return ratio


def test_activations_use_the_third_part():
    """make_activations' values are fp16-exact (x_l = 0); these are not: x_l is non-zero for nearly every non-zero entry."""
    x = make_x(4096, 64, seed=1)
    h, m, lo = parts(x)
    assert np.array_equal(h.astype(np.float64) + m + lo, x.astype(np.float64))  # the split is exact
    nz = x != 0
    assert (lo[nz] != 0).mean() > 0.9
    assert (parts(make_activations(4096, 64, seed=1))[2] == 0).all()


# ---- every parity shape, both bit widths, the row counts at the tile edges --------------------------------------------------------
M_LIST = [1, 2, 63, 64, 65, 127, 128, 129]
PAIRS = sorted({(K, N) for K, N, _ in BOUND_SHAPES})
CASES = [((K, N, bits), M) for K, N in PAIRS for bits in (3, 4) for M in M_LIST]
_cache = {}


def parity_case(shape):
    if shape not in _cache:
        _cache.clear()
        K, N, bits = shape
        L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True)
        x = make_x(K, M_LIST[-1], seed=K + bits)
        _cache[shape] = (L, to_torch(L), x, torch.from_numpy(x).cuda(), orc.forward_f64(L, x), abs_sum(L, x))
    return _cache[shape]


@pytest.mark.parametrize("shape,M", CASES, ids=[f"w{s[2]}_{s[0]}x{s[1]}-M{m}" for s, m in CASES])
def test_c_abi_vs_oracle(lib, shape, M):
    L, T, x, xt, want, S = parity_case(shape)
    got = f32_call(lib, L, xt[:M].contiguous(), T=T)
    check(got, L, x[:M], want=want[:M], S=S[:M])


LARGE = [(4, 4096, 12288), (4, 4096, 4096), (4, 4096, 22016), (4, 11008, 4096)]


@pytest.mark.parametrize("M", [2048, 2049])
@pytest.mark.parametrize("shape", LARGE, ids=["qkv", "o", "gate_up", "down"])
def test_c_abi_vs_oracle_prefill_rows(lib, shape, M):
    """An fp32 prefill on the 7B shapes, with a bias: both edges of the first and last M-tiles and a fixed spread of rows."""
    bits, K, N = shape
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=7, skew=(N == 12288), nonzero_full_rows=True)
    x = make_x(K, M, seed=11)
    bias = np.random.default_rng(3).standard_normal(N).astype(np.float32)
    got = f32_call(lib, L, x, bias=bias).cpu().numpy()
    rows = sorted(set([0, 1, 2, 3, 63, 64, 127, 128, 1023, 1919, 1920, 2046, 2047, M - 1] + list(range(5, M, 397))))
    check(got[rows], L, x[rows], bias=bias)


# ---- numerics stress --------------------------------------------------------------------------------------------------------------
def _stress(lib, L, M=70, seed=0):
    x = full_mantissa(orc.make_vec(L["infeatures"], batch=M, seed=seed), seed)
    got = f32_call(lib, L, x).cpu().numpy()
    check(got, L, x)
    return got, x


def test_rows_from_1e_minus_30_to_1e30(lib):
    K, N, M = 4096, 1024, 130
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=51, nonzero_full_rows=True)
    x = make_x(K, M, seed=51)
    scale = 10.0 ** np.linspace(-30.0, 30.0, M)
    x = (x.astype(np.float64) * scale[:, None] / np.maximum(np.abs(x).max(axis=1, keepdims=True), 1e-30)).astype(np.float32)
    got = f32_call(lib, L, x).cpu().numpy()
    assert np.isfinite(got).all()
    # rel_err's floor is 1 % of the largest output of the whole array: the bound judges each element, rel_err each row
    check(got, L, x, old=False)
    for r in (0, 1, 64, 128, 129):
        assert np.abs(got[r]).max() > 0
        check(got[r:r + 1], L, x[r:r + 1])


def test_x_whose_parts_are_bf16_subnormals(lib):
    """Rows at |x| ~ 1e-33 ... 1e-37: x_m and x_l (or x_m alone) fall below 2^-126, where bf16 keeps fewer bits.  The split then
    holds x to within 2^-134 absolute (half bf16's smallest subnormal), so each output is within E_ACC S + 2^-133 sum_k |w_kc|."""
    K, N, M = 4096, 512, 8
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=52, nonzero_full_rows=True)
    x = make_x(K, M, seed=52)
    scale = np.array([1e-33, 1e-34, 1e-35, 1e-35, 1e-36, 1e-36, 1e-37, 1e-37])
    x = (x.astype(np.float64) * scale[:, None] / np.maximum(np.abs(x).max(axis=1, keepdims=True), 1e-30)).astype(np.float32)
    _, _, lo = parts(x)
    nz = x[2:] != 0
    assert (np.abs(lo[2:][nz]) < 2.0 ** -126).mean() > 0.9  # the lowest part is subnormal (or rounds to zero) in these rows
    got = f32_call(lib, L, x).cpu().numpy()
    want = orc.forward_f64(L, x)
    S = abs_sum(L, x)
    W1 = orc.forward_f64(abs_layer(L), np.ones((1, K), dtype=np.float32))  # sum_k |w_kc|
    ratio = bound_ratio(got, want, S, eta=0.0 + 2.0 ** -133 * W1)
    assert ratio <= 1.0, ratio
    assert rel_err(got[:2], want[:2]) < TIGHT_TOL  # 1e-33 / 1e-34: the parts are still normal or nearly so


def test_tiny_and_large_centroids_side_by_side(lib):
    """Channels with centroids around 1e-6 next to channels around 1e-1: each group within the bound of its own magnitude."""
    L = orc.make_layer(4, 512, 256, sparsity=0.01, topX=4, seed=1, nonzero_full_rows=True)
    L["lookup_table"][0::2] *= 5e-5
    L["lookup_table"][1::2] *= 5.0
    tiny = np.arange(0, 256, 2)
    tiny = tiny[~np.isin(tiny, L["full_row_indices"])]
    hit = np.repeat(np.arange(256), np.diff(L["rows"]))
    L["vals"][np.isin(hit, tiny)] *= 5e-5
    got, x = _stress(lib, L)
    assert rel_err(got[:, tiny], orc.forward_f64(L, x)[:, tiny]) < TIGHT_TOL


def test_shuffled_duplicate_and_out_of_range_csr_entries(lib):
    """Shuffled columns within each CSR row, duplicate columns (they add up) and columns outside [0, K) (ignored)."""
    K, N = 2048, 320
    L = orc.make_layer(4, K, N, sparsity=0.02, seed=5, skew=True)
    rng = np.random.default_rng(5)
    U = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    for c in range(N):
        e0, e1 = L["rows"][c], L["rows"][c + 1]
        perm = rng.permutation(e1 - e0) + e0
        U["cols"][e0:e1], U["vals"][e0:e1] = L["cols"][perm], L["vals"][perm]
    assert not np.array_equal(U["cols"], L["cols"])
    got_u, x = _stress(lib, U)
    got_s = f32_call(lib, L, x).cpu().numpy()
    assert bound_ratio(got_u, got_s, abs_sum(L, x), e=2 * E_ACC) <= 1.0  # both within the bound of the same truth
    # duplicates and out-of-range columns: the oracle sees the duplicates and a zero in place of each ignored entry
    D = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    busy = [c for c in range(N) if L["rows"][c + 1] - L["rows"][c] >= 3][:40]
    for i, c in enumerate(busy):
        e0 = L["rows"][c]
        D["cols"][e0 + 1] = D["cols"][e0]  # a duplicate of the entry before it
        D["cols"][e0 + 2] = (-1, K, K + 1000)[i % 3]
    got = f32_call(lib, D, x).cpu().numpy()
    O = dict(D, cols=np.where((D["cols"] >= 0) & (D["cols"] < K), D["cols"], 0).astype(np.int32),
             vals=np.where((D["cols"] >= 0) & (D["cols"] < K), D["vals"], 0.0).astype(np.float32))
    check(got, O, x)


def test_all_128_dense_rows_on_channel_0(lib):
    L = orc.make_layer(4, 1024, 256, sparsity=0.005, topX=128, seed=3, nonzero_full_rows=True)
    L["full_row_indices"][:] = 0
    L["full_rows"] /= 128.0
    got, x = _stress(lib, L)
    assert rel_err(got[:, 0], orc.forward_f64(L, x)[:, 0]) < TIGHT_TOL


def test_topx_300_with_duplicates_and_ignored_indices(lib):
    K, N = 512, 384
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=300, seed=4, nonzero_full_rows=True)
    rng = np.random.default_rng(4)
    fri = rng.integers(0, N, size=300).astype(np.int32)
    fri[:20] = 5
    L["full_rows"][:, :20] /= 20.0
    fri[290], fri[291], fri[292] = -1, N, N + 1000
    L["full_row_indices"] = fri
    x = make_x(K, 70, seed=0)
    got = f32_call(lib, L, x).cpu().numpy()
    keep = (fri >= 0) & (fri < N)
    L2 = dict(L, full_rows=np.ascontiguousarray(L["full_rows"][:, keep]), full_row_indices=np.ascontiguousarray(fri[keep]))
    check(got, L2, x)


@pytest.mark.parametrize("bits,K,N", [(4, 160, 200), (3, 96, 60), (4, 4128, 136), (3, 4128, 4100)])
def test_partial_last_k_chunk_ragged_n_and_empty_csr(lib, bits, K, N):
    """K a multiple of 32 but not of 64 (the second half of the last chunk is zero-filled), N not a multiple of 128."""
    L = orc.make_layer(bits, K, N, sparsity=0.0, topX=3, seed=K, nonzero_full_rows=True)
    L["rows"] = np.zeros(N + 1, dtype=np.int32)
    L["cols"] = np.zeros(0, dtype=np.int32)
    L["vals"] = np.zeros(0, dtype=np.float32)
    _stress(lib, L, M=131)


# ---- reproducibility ------------------------------------------------------------------------------------------------------------
def test_two_calls_are_bit_identical(lib):
    L = orc.make_layer(3, 4096, 4096, sparsity=0.0045, topX=10, seed=61, nonzero_full_rows=True)
    T = to_torch(L)
    xt = torch.from_numpy(make_x(4096, 300, seed=61)).cuda()
    assert torch.equal(f32_call(lib, L, xt, T=T), f32_call(lib, L, xt, T=T))


def test_row_is_independent_of_other_rows_and_of_M(lib):
    """A row's result is bit-identical whatever M is and whatever the other rows hold."""
    K, N = 4096, 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=31, nonzero_full_rows=True)
    T = to_torch(L)
    x = make_x(K, 200, seed=31)
    other = make_x(K, 200, seed=32)
    keep = np.array([0, 1, 2, 3, 37, 63, 128])
    run = lambda xx: f32_call(lib, L, np.ascontiguousarray(xx), T=T).cpu().numpy()
    base = run(x)
    variants = {f"M={M}": run(x[:M]) for M in (1, 64, 65, 128, 129)}
    perm = np.random.default_rng(31).permutation(200)
    perm = perm[~np.isin(perm, keep)]
    xp = x.copy()
    xp[np.setdiff1d(np.arange(200), keep)] = x[perm]
    variants["permuted others"] = run(xp)
    for M in (65, 200):
        xn = other[:M].copy()
        rows = keep[keep < M]
        xn[rows] = x[rows]
        variants[f"new others M={M}"] = run(xn)
    for name, y in variants.items():
        rows = keep[keep < y.shape[0]]
        assert np.array_equal(y[rows].view(np.uint32), base[rows].view(np.uint32)), name
    check(base, L, x)


def _args(T, bits, bias=None):
    return (T["qweight"], T["lookup_table"], bits, bias, T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])


def test_graph_capture_and_replay_with_new_inputs(qc):
    K, N, M = 4096, 4096, 256
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=9, nonzero_full_rows=True)
    T = to_torch(L)
    x = torch.from_numpy(make_x(K, M, seed=1)).cuda()
    x2 = make_x(K, M, seed=2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        qc.lutgemm_fused_f32(x, *_args(T, 3))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = qc.lutgemm_fused_f32(x, *_args(T, 3))
    x.copy_(torch.from_numpy(x2))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, qc.lutgemm_fused_f32(torch.from_numpy(x2).cuda(), *_args(T, 3)))
    check(out, L, x2)


def test_three_streams_at_once(qc):
    """Three fp32 tensor-core calls on three streams with no synchronisation between them: the bits of the calls run alone."""
    Ls = [orc.make_layer(4, 4096, 4096, sparsity=0.0045, topX=10, seed=81, nonzero_full_rows=True, bias=True),
          orc.make_layer(3, 4096, 12288, sparsity=0.0045, topX=10, seed=82, nonzero_full_rows=True),
          orc.make_layer(4, 11008, 4096, sparsity=0.0045, topX=10, seed=83, nonzero_full_rows=True)]
    Ts = [to_torch(L) for L in Ls]
    xs = [make_x(4096, 300, seed=81), make_x(4096, 128, seed=82), make_x(11008, 200, seed=83)]
    xg = [torch.from_numpy(x).cuda() for x in xs]
    bias = [Ts[0]["bias"], None, None]
    alone = [qc.lutgemm_fused_f32(xg[i], *_args(Ts[i], Ls[i]["bits"], bias[i])) for i in range(3)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    out = []
    for i, s in enumerate(streams):
        with torch.cuda.stream(s):
            out.append(qc.lutgemm_fused_f32(xg[i], *_args(Ts[i], Ls[i]["bits"], bias[i])))
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(out[i], alone[i]), i
    check(out[0], Ls[0], xs[0], bias=Ls[0]["bias"])
    check(out[1], Ls[1], xs[1])
    check(out[2], Ls[2], xs[2])


# ---- quant_cuda.lutgemm_fused_f32 -------------------------------------------------------------------------------------------------
def test_pybind_fp32_in_fp32_out_and_other_dtypes_raise(qc):
    K, N, M = 4096, 4096, 100
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=8, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = make_x(K, M, seed=8)
    xt = torch.from_numpy(x).cuda()
    y = qc.lutgemm_fused_f32(xt, *_args(T, 4, T["bias"]))
    torch.cuda.synchronize()
    assert y.dtype == torch.float32 and y.shape == (M, N)
    check(y, L, x, bias=L["bias"])
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        with pytest.raises(RuntimeError, match="lutgemm_fused_f32: x must be fp32"):
            qc.lutgemm_fused_f32(xt.to(dt), *_args(T, 4, T["bias"]))
    with pytest.raises(RuntimeError, match="fp16 or bf16"):
        qc.lutgemm_fused(xt, *_args(T, 4, T["bias"]))


# ---- QuantLinearLUT ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def spy(qc, monkeypatch):
    calls = []
    real = qc.lutgemm_fused_f32

    def wrapped(*a, **kw):
        calls.append((tuple(a[0].shape), a[0].dtype))
        return real(*a, **kw)
    monkeypatch.setattr(qc, "lutgemm_fused_f32", wrapped)
    return calls


def _run(m, x, fused=True):
    from squeezellm_b200.quant import QuantLinearLUT
    QuantLinearLUT.use_fused = fused
    try:
        y = m(x)
    finally:
        QuantLinearLUT.use_fused = True
    torch.cuda.synchronize()
    return y


def test_module_routing_dtype_shape_and_bias(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    T = QuantLinearLUT.FP32_TC_MIN_ROWS
    K = N = 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=12, nonzero_full_rows=True)
    x = make_x(K, 2048, seed=12)
    xt = torch.from_numpy(x).cuda()
    for bias_on in (False, True):
        m = _module(L, bias=bias_on)
        bias = m.bias.cpu().numpy() if bias_on else None
        for M in (T, 2048):
            del spy[:]
            xx = xt[:M].reshape(1, M, K)
            y = _run(m, xx)
            assert spy == [((M, K), torch.float32)]
            y_b = _run(m, xx, fused=False)  # the batched branch
            assert spy == [((M, K), torch.float32)]
            assert y.dtype == y_b.dtype == torch.float32 and y.shape == y_b.shape == (1, M, N)
            rows = [0, 1, 2, 3, T - 1, M - 1] + ([127, 128, 1000] if M > 128 else [])
            want = orc.forward_f64(L, x[rows])  # the bias is added to the fp32 sum afterwards
            S = abs_sum(L, x[rows], bias)
            b = 0.0 if bias is None else bias.astype(np.float64)[None, :]
            assert bound_ratio(y[0][rows].cpu().numpy(), want + b, S) <= 1.0
            assert bound_ratio(y_b[0][rows].cpu().numpy(), want + b, S) <= 1.0
            assert rel_err(y[0][rows].cpu().numpy(), y_b[0][rows].cpu().numpy()) < TIGHT_TOL
    del spy[:]
    m = _module(L)
    _run(m, xt[:T - 1].reshape(1, T - 1, K))
    _run(m, xt[:T].reshape(1, T, K), fused=False)
    _run(m, xt[:2048], fused=False)
    assert spy == []


def test_misaligned_fp32_view_through_the_module_is_bit_identical(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 4096, 1024, QuantLinearLUT.FP32_TC_MIN_ROWS
    m = _module(orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=13, nonzero_full_rows=True), bias=True)
    xa = torch.from_numpy(make_x(K, M, seed=13)).cuda()
    want = _run(m, xa)
    for off in (1, 2, 3):
        buf = torch.zeros(M * K + 4, device="cuda", dtype=torch.float32)
        xv = buf[off:off + M * K].view(M, K)
        xv.copy_(xa)
        assert xv.is_contiguous() and xv.data_ptr() % 16
        assert torch.equal(_run(m, xv), want), off
        assert torch.equal(xv, xa)
    assert len(spy) == 4


def test_stacked_qkv_group_in_one_launch(spy):
    from squeezellm_b200.fusion import fuse_siblings
    from squeezellm_b200.quant import QuantLinearLUT
    K, M = 512, QuantLinearLUT.FP32_TC_MIN_ROWS
    Ls = [orc.make_layer(4, K, n, sparsity=0.01, topX=3, seed=20 + n, nonzero_full_rows=True) for n in (256, 128, 192)]
    block = torch.nn.Module()
    for name, L in zip(("q_proj", "k_proj", "v_proj"), Ls):
        setattr(block, name, _module(L))
    assert len(fuse_siblings(block)) == 1
    x = make_x(K, M, seed=21)
    xt = torch.from_numpy(x).cuda().reshape(1, M, K)
    outs = [block.q_proj(xt), block.k_proj(xt), block.v_proj(xt)]
    torch.cuda.synchronize()
    assert spy == [((M, K), torch.float32)]
    for y, L in zip(outs, Ls):
        assert y.dtype == torch.float32
        check(y[0], L, x)


def test_grad_forward_is_bit_identical_and_dx_stays_on_the_cuda_cores(spy, monkeypatch):
    from squeezellm_b200 import quant
    QuantLinearLUT = quant.QuantLinearLUT
    K, N = 4096, 2048
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=90, nonzero_full_rows=True)
    m = _module(L, bias=True)
    paths = []
    real_t = quant.quant_cuda.lutgemm_t

    def wrapped_t(*a, **kw):
        paths.append(kw.get("path"))
        return real_t(*a, **kw)
    monkeypatch.setattr(quant.quant_cuda, "lutgemm_t", wrapped_t)
    rows = QuantLinearLUT.FP32_TC_MIN_ROWS
    xt = torch.from_numpy(make_x(K, rows, seed=90)).cuda()
    with torch.no_grad():
        y0 = m(xt.reshape(1, rows, K))
    x = xt.reshape(1, rows, K).clone().requires_grad_(True)
    y = m(x)
    assert y.grad_fn is not None
    assert torch.equal(y.detach(), y0)
    y.sum().backward()
    assert x.grad is not None and x.grad.dtype == torch.float32 and x.grad.shape == x.shape
    assert paths == ["cuda"]
    assert spy == [((rows, K), torch.float32)] * 2  # with and without grad


def test_train_codebook_forward_is_the_plain_forward(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 1024, 512, QuantLinearLUT.FP32_TC_MIN_ROWS
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=4, seed=91, nonzero_full_rows=True)
    plain, trained = _module(L, bias=True), _module(L, bias=True)
    trained.train_codebook(lookup_table=True, vals=True, full_rows=True, bias=True)
    xt = torch.from_numpy(make_x(K, M, seed=91)).cuda()
    with torch.no_grad():
        y0 = plain(xt)
    y1 = trained(xt)
    assert y1.grad_fn is not None
    assert torch.equal(y1.detach(), y0)
    y1.sum().backward()
    assert trained.lookup_table.grad is not None
    assert spy == [((M, K), torch.float32)] * 2


# ---- the batched route's second pass over the batch (use_fused = False), which the fused route now skips at these sizes -----------
@pytest.mark.parametrize("bias_on", [True, False])
def test_unfused_2049_rows_on_a_7b_shape(bias_on):
    """fp32 x of 2049 rows through use_fused = False on the 7B q/k/v shape: csr_batched_kernel's second pass over the batch."""
    K, N, bits = 4096, 12288, 4
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True)
    m = _module(L, bias=bias_on)
    x = make_activations(K, 2049, seed=K + bits)
    y = _run(m, torch.from_numpy(x).cuda(), fused=False).cpu().numpy()
    rows = [0, 1, 2, 3, 127, 128, 1919, 1920, 2015, 2016, 2017, 2047, 2048]
    bias = m.bias.cpu().numpy().astype(np.float64) if bias_on else None
    want = orc.forward_f64(L, x[rows])
    S = abs_sum(L, x[rows], bias)
    b = 0.0 if bias is None else bias[None, :]
    assert bound_ratio(y[rows], want + b, S) <= 1.0
    assert rel_err(y[rows], want + b) < TIGHT_TOL


# ---- an fp32 Llama model as the reference's loader builds it -----------------------------------------------------------------------
def test_fp32_llama_prefill_matches_the_batched_route(spy):
    """A tiny LlamaForCausalLM built in fp32 (AutoModelForCausalLM.from_config, as llama.py does), its Linears replaced from a
    reference-format sparse checkpoint by checkpoint.load_quantized: a prefill of FP32_TC_MIN_ROWS tokens gives the logits of the
    use_fused = False route (the _batched symbols) within rel_err 1e-4.  Both are fp32 sums of the same products in different
    orders, a few u apart per layer output; the tolerance leaves room for their growth through two blocks and the softmaxes."""
    transformers = pytest.importorskip("transformers")
    from squeezellm_b200 import checkpoint as ck
    from squeezellm_b200.quant import QuantLinearLUT
    T = QuantLinearLUT.FP32_TC_MIN_ROWS
    cfg = transformers.LlamaConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=97, max_position_embeddings=max(T, 64))
    torch.manual_seed(0)
    model = transformers.AutoModelForCausalLM.from_config(cfg).eval()
    assert next(model.parameters()).dtype == torch.float32
    state = {k: v.clone() for k, v in model.state_dict().items()}
    n = 0
    for name, lin in ck.find_linear_layers(model).items():
        if name == "lm_head":
            continue
        L = orc.make_layer(4, lin.in_features, lin.out_features, sparsity=0.01, topX=0, seed=100 + n)
        n += 1
        del state[name + ".weight"]
        state[name + ".qweight"] = torch.from_numpy(L["qweight"])
        state[name + ".lookup_table"] = torch.from_numpy(L["lookup_table"] * 5.0)  # keep activations O(1) through the blocks
        for k in ("rows", "cols", "vals"):
            state[name + "." + k] = torch.from_numpy(L[k])
        state["sparse_threshold." + name] = len(L["vals"])
    res = ck.load_quantized(model, state, 4, include_sparse=True)
    assert not res.missing_keys and not res.unexpected_keys and n == 14
    model = model.cuda()
    ids = torch.randint(0, 97, (1, T), generator=torch.Generator().manual_seed(1)).cuda()
    with torch.no_grad():
        del spy[:]
        fused = model(ids).logits
        assert len(spy) == 14 and all(shape[0] == T and dt == torch.float32 for shape, dt in spy)
        del spy[:]
        QuantLinearLUT.use_fused = False
        try:
            unfused = model(ids).logits
        finally:
            QuantLinearLUT.use_fused = True
        assert spy == []
    assert fused.dtype == torch.float32 and torch.isfinite(fused).all() and fused.abs().max() > 0
    assert rel_err(fused.cpu().numpy(), unfused.cpu().numpy()) < 1e-4
