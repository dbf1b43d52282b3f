"""The tensor-core LUT-GEMM for bf16 x (`sqllm_lutgemm_fused_dt`, `quant_cuda.lutgemm_fused`, csrc/lutgemm_tc.cuh with three bf16
weight parts) that runs bf16 inputs of QuantLinearLUT.BF16_TC_MIN_ROWS or more rows.  The truth is the fp64 oracle on the
bf16-rounded activations; the metric is the per-element bound of tests/util.py (bound_ratio <= 1) beside the old rel_err < TIGHT_TOL,
both on fp32 output.  Covered: every parity shape at both bit widths and a range of row counts, 2048-row prefills, numerics stress,
activations fp16 cannot hold, bf16 output, reproducibility and row independence, fp16 x through the new entry point, graphs and
streams, the pybind adapter, the module routing and training."""
import ctypes

import numpy as np
import pytest
import torch

from test_backward_gpu import _module
from test_error_bound_host import SHAPES as BOUND_SHAPES
from test_prefill_tc_gpu import abi_call
from util import OUT_ROUNDING, TIGHT_TOL, Args, abs_sum, bound_ratio, load_lib, make_activations, orc, rel_err, to_torch

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 0, 1, 2
DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemm_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p]
    lib.sqllm_lutgemm_fused.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def dt_call(lib, L, x, y_dtype=torch.float32, bias=None, T=None):
    """sqllm_lutgemm_fused_dt on the layer dict L (numpy; T: its torch tensors) and x [M, K] (torch, cuda, fp16 / bf16) -> y [M, N]
    (torch, y_dtype)."""
    T = to_torch(L) if T is None else T
    M, N = x.shape[0], L["outfeatures"]
    y = torch.empty((M, N), device="cuda", dtype=y_dtype)
    a = Args(bits=L["bits"], in_features=L["infeatures"], out_features=N, batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    b = None if bias is None else torch.from_numpy(bias).cuda()
    rc = lib.sqllm_lutgemm_fused_dt(ctypes.byref(a), x.data_ptr(), DT[x.dtype], y.data_ptr(), DT[y_dtype],
                                    None if b is None else b.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    return y


def bf16(x):
    """numpy fp32 -> its bf16 rounding (fp32 numpy) and the bf16 tensor on the GPU."""
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda().bfloat16()
    return t.float().cpu().numpy(), t


def check(got, L, xb, bias=None, y_dtype="float32", want=None, S=None, old=True):
    """bound_ratio <= 1 (and rel_err < TIGHT_TOL on fp32 output) of got [M, N] against the oracle on the bf16-exact rows xb."""
    got = got.float().cpu().numpy() if isinstance(got, torch.Tensor) else got
    mul = None if bias is None else bias[None, :]
    want = orc.forward_f64(L, xb, mul_init=mul) if want is None else want
    S = abs_sum(L, xb, bias) if S is None else S
    r, eta = OUT_ROUNDING[y_dtype]
    ratio = bound_ratio(got, want, S, want, r, eta=eta)
    assert ratio <= 1.0, ratio
    if old and y_dtype == "float32":
        e = rel_err(got, want)
        assert e < TIGHT_TOL, e
    return ratio


# ---- every parity shape, both bit widths, a range of row counts -------------------------------------------------------------------
M_LIST = [1, 17, 64, 129, 200]
PAIRS = sorted({(K, N) for K, N, _ in BOUND_SHAPES})
CASES = [((K, N, bits), M) for K, N in PAIRS for bits in (3, 4) for M in M_LIST]
_cache = {}


def parity_case(shape):
    """Layer, M_LIST[-1] bf16-exact activation rows and the oracle and S on all of them, shared by the row counts of one shape
    (a row's result does not depend on the other rows)."""
    if shape not in _cache:
        _cache.clear()
        K, N, bits = shape
        L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True)
        xb, xt = bf16(make_activations(K, M_LIST[-1], seed=K + bits))
        _cache[shape] = (L, to_torch(L), xb, xt, orc.forward_f64(L, xb), abs_sum(L, xb))
    return _cache[shape]


@pytest.mark.parametrize("shape,M", CASES, ids=[f"w{s[2]}_{s[0]}x{s[1]}-M{m}" for s, m in CASES])
def test_c_abi_vs_oracle(lib, shape, M):
    L, T, xb, xt, want, S = parity_case(shape)
    got = dt_call(lib, L, xt[:M].contiguous(), T=T)
    check(got, L, xb[:M], want=want[:M], S=S[:M])


@pytest.mark.parametrize("shape", [(4, 4096, 12288), (4, 4096, 22016), (4, 11008, 4096)], ids=["qkv", "gate_up", "down"])
def test_c_abi_vs_oracle_2048_rows(lib, shape):
    """A 2048-token bf16 prefill on the 7B shapes, with a bias: both edges of the first and last M-tile and a fixed spread of rows."""
    bits, K, N = shape
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=7, skew=(N == 12288), nonzero_full_rows=True)
    M = 2048
    xb, xt = bf16(make_activations(K, M, seed=11))
    bias = np.random.default_rng(3).standard_normal(N).astype(np.float32)
    got = dt_call(lib, L, xt, bias=bias).cpu().numpy()
    rows = sorted(set([0, 1, 2, 3, 63, 64, 127, 128, 1023, 1919, 1920, 2046, 2047] + list(range(5, M, 397))))
    check(got[rows], L, xb[rows], bias=bias)


# ---- numerics stress (the cases of the fp16 kernel's tests) ------------------------------------------------------------------------
def _stress(lib, L, M=70, seed=0):
    xb, xt = bf16(orc.make_vec(L["infeatures"], batch=M, seed=seed))
    got = dt_call(lib, L, xt).cpu().numpy()
    check(got, L, xb)
    return got, xb, xt


def test_tiny_and_large_centroids_side_by_side(lib):
    """Channels with centroids around 1e-6 next to channels around 1e-1: each group within the bound of its own magnitude."""
    L = orc.make_layer(4, 512, 256, sparsity=0.01, topX=4, seed=1, nonzero_full_rows=True)
    L["lookup_table"][0::2] *= 5e-5
    L["lookup_table"][1::2] *= 5.0
    tiny = np.arange(0, 256, 2)
    tiny = tiny[~np.isin(tiny, L["full_row_indices"])]
    hit = np.repeat(np.arange(256), np.diff(L["rows"]))
    L["vals"][np.isin(hit, tiny)] *= 5e-5
    got, xb, _ = _stress(lib, L)
    want = orc.forward_f64(L, xb)
    assert rel_err(got[:, tiny], want[:, tiny]) < TIGHT_TOL


def test_outlier_a_million_times_the_codebook(lib):
    L = orc.make_layer(3, 1024, 192, sparsity=0.005, seed=2)
    c = 37
    e = L["rows"][c]
    assert L["rows"][c + 1] > e
    L["vals"][e] = 1e6 * np.abs(L["lookup_table"][c]).max()
    got, xb, _ = _stress(lib, L)
    want = orc.forward_f64(L, xb)
    others = np.arange(192) != c
    assert rel_err(got[:, others], want[:, others]) < TIGHT_TOL
    assert rel_err(got[:, c], want[:, c]) < TIGHT_TOL


def test_all_128_dense_rows_on_channel_0(lib):
    L = orc.make_layer(4, 1024, 256, sparsity=0.005, topX=128, seed=3, nonzero_full_rows=True)
    L["full_row_indices"][:] = 0
    L["full_rows"] /= 128.0
    got, xb, _ = _stress(lib, L)
    assert rel_err(got[:, 0], orc.forward_f64(L, xb)[:, 0]) < TIGHT_TOL


def test_topx_300_with_duplicates_and_ignored_indices(lib):
    K, N = 512, 384
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=300, seed=4, nonzero_full_rows=True)
    rng = np.random.default_rng(4)
    fri = rng.integers(0, N, size=300).astype(np.int32)
    fri[:20] = 5
    L["full_rows"][:, :20] /= 20.0
    fri[290], fri[291], fri[292] = -1, N, N + 1000
    L["full_row_indices"] = fri
    xb, xt = bf16(orc.make_vec(K, batch=70, seed=0))
    got = dt_call(lib, L, xt).cpu().numpy()
    keep = (fri >= 0) & (fri < N)
    L2 = dict(L, full_rows=np.ascontiguousarray(L["full_rows"][:, keep]), full_row_indices=np.ascontiguousarray(fri[keep]))
    check(got, L2, xb)


def test_unsorted_csr_rows(lib):
    """Shuffled column indices within each CSR row: within the bound of the oracle, and of the sorted rows' result."""
    L = orc.make_layer(4, 2048, 320, sparsity=0.02, seed=5, skew=True)
    rng = np.random.default_rng(5)
    U = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    for c in range(320):
        e0, e1 = L["rows"][c], L["rows"][c + 1]
        perm = rng.permutation(e1 - e0) + e0
        U["cols"][e0:e1], U["vals"][e0:e1] = L["cols"][perm], L["vals"][perm]
    assert not np.array_equal(U["cols"], L["cols"])
    got_u, xb, xt = _stress(lib, U)
    got_s = dt_call(lib, L, xt).cpu().numpy()
    assert rel_err(got_u, got_s) < TIGHT_TOL
    assert bound_ratio(got_u, got_s, abs_sum(L, xb), r=0.0, e=2 * 2.0 ** -20) <= 1.0  # both within the bound of the same truth


@pytest.mark.parametrize("bits,K,N", [(4, 160, 200), (3, 96, 60), (4, 4128, 136)])
def test_partial_last_k_chunk_and_empty_csr(lib, bits, K, N):
    L = orc.make_layer(bits, K, N, sparsity=0.0, topX=3, seed=K, nonzero_full_rows=True)
    L["rows"] = np.zeros(N + 1, dtype=np.int32)
    L["cols"] = np.zeros(0, dtype=np.int32)
    L["vals"] = np.zeros(0, dtype=np.float32)
    _stress(lib, L, M=131)


# ---- bf16-only ground: activations fp16 cannot hold -------------------------------------------------------------------------------
def test_activations_at_1e20_and_1e_minus_30(lib):
    K, N, M = 4096, 1024, 130
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=51, nonzero_full_rows=True)
    x = make_activations(K, M, seed=51)
    x[0] *= 1e20 / np.abs(x[0]).max()
    x[1] *= 1e-30 / np.abs(x[1]).max()
    x[129] = np.random.default_rng(51).standard_normal(K) * 1e20
    xb, xt = bf16(x)
    assert np.abs(xb[0]).max() > 65504 and np.abs(xb[1]).max() < 2.0 ** -25  # outside fp16: overflow, and zero
    got = dt_call(lib, L, xt).cpu().numpy()
    assert np.isfinite(got).all()
    # rel_err's floor is 1 % of the largest output of the whole array (1e20 rows next to 1e-30 rows): the bound judges each element
    check(got, L, xb, old=False)
    for r in (0, 1, 129):
        assert np.abs(got[r]).max() > 0
        check(got[r:r + 1], L, xb[r:r + 1])


# ---- bf16 output ----------------------------------------------------------------------------------------------------------------
def test_bf16_output(lib):
    K, N, M = 4096, 4096 + 64 + 2, 150  # a ragged last N-tile with an even N; see below for an odd one
    for n, bias_on in ((N, True), (N + 1, False)):
        L = orc.make_layer(4, K, n, sparsity=0.0045, topX=10, seed=n, nonzero_full_rows=True)
        bias = np.random.default_rng(n).standard_normal(n).astype(np.float32) if bias_on else None
        xb, xt = bf16(make_activations(K, M, seed=n))
        y16 = dt_call(lib, L, xt, y_dtype=torch.bfloat16, bias=bias)
        y32 = dt_call(lib, L, xt, bias=bias)
        assert y16.dtype == torch.bfloat16
        assert torch.equal(y16, y32.bfloat16())  # the same fp32 value, rounded once
        check(y16, L, xb, bias=bias, y_dtype="bfloat16")


# ---- reproducibility ------------------------------------------------------------------------------------------------------------
def test_two_calls_are_bit_identical(lib):
    L = orc.make_layer(3, 4096, 4096, sparsity=0.0045, topX=10, seed=61, nonzero_full_rows=True)
    T = to_torch(L)
    _, xt = bf16(make_activations(4096, 300, seed=61))
    assert torch.equal(dt_call(lib, L, xt, T=T), dt_call(lib, L, xt, T=T))
    assert torch.equal(dt_call(lib, L, xt, torch.bfloat16, T=T), dt_call(lib, L, xt, torch.bfloat16, T=T))


def test_row_is_independent_of_other_rows_and_of_M(lib):
    """A row's fp32 result is bit-identical whatever M (>= 64) is and whatever the other rows hold."""
    K, N = 4096, 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=31, nonzero_full_rows=True)
    T = to_torch(L)
    xb, _ = bf16(make_activations(K, 200, seed=31))
    other, _ = bf16(make_activations(K, 200, seed=32))
    fixed = [0, 1, 2, 3, 37, 63]
    keep = np.array(fixed + [128])
    run = lambda xx: dt_call(lib, L, torch.from_numpy(np.ascontiguousarray(xx)).cuda().bfloat16(), T=T).cpu().numpy()
    base = run(xb)
    variants = {f"M={M}": run(xb[:M]) for M in (64, 65, 128, 129)}
    perm = np.random.default_rng(31).permutation(200)
    perm = perm[~np.isin(perm, keep)]
    xp = xb.copy()
    xp[np.setdiff1d(np.arange(200), keep)] = xb[perm]
    variants["permuted others"] = run(xp)
    for M in (65, 200):
        xn = other[:M].copy()
        rows = keep[keep < M]
        xn[rows] = xb[rows]
        variants[f"new others M={M}"] = run(xn)
    for name, y in variants.items():
        rows = keep[keep < y.shape[0]]
        assert np.array_equal(y[rows].view(np.uint32), base[rows].view(np.uint32)), name
    check(base, L, xb)


@pytest.mark.parametrize("bits", [3, 4])
def test_fp16_x_through_the_dtype_entry_is_the_fp16_entry(lib, bits):
    """sqllm_lutgemm_fused is sqllm_lutgemm_fused_dt with SQLLM_DT_F16: the same bits, fp32 and fp16 output, with a bias."""
    K, N, M = 4096, 4096 + 40, 140
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=70 + bits, nonzero_full_rows=True)
    bias = np.random.default_rng(70).standard_normal(N).astype(np.float32)
    x16 = torch.from_numpy(make_activations(K, M, seed=70)).cuda().half()
    for y_dtype in (torch.float32, torch.float16):
        old = abi_call(lib, L, x16, y_half=y_dtype == torch.float16, bias=bias)
        new = dt_call(lib, L, x16, y_dtype=y_dtype, bias=bias).float().cpu().numpy()
        assert np.array_equal(old.view(np.uint32), new.view(np.uint32)), y_dtype


# ---- graphs and streams -----------------------------------------------------------------------------------------------------------
def _args(T, bits, bias=None):
    return (T["qweight"], T["lookup_table"], bits, bias, T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])


def test_graph_capture_and_replay_with_new_inputs(qc):
    K, N, M = 4096, 4096, 256
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=9, nonzero_full_rows=True)
    T = to_torch(L)
    x = torch.from_numpy(make_activations(K, M, seed=1)).cuda().bfloat16()
    x2b, x2 = bf16(make_activations(K, M, seed=2))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        qc.lutgemm_fused(x, *_args(T, 3))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = qc.lutgemm_fused(x, *_args(T, 3))
    x.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, qc.lutgemm_fused(x2, *_args(T, 3)))
    check(out, L, x2b, y_dtype="bfloat16")


def test_three_streams_at_once(qc):
    """bf16 tensor-core, fp16 tensor-core and batched calls on three streams with no synchronisation between them."""
    Ls = [orc.make_layer(4, 4096, 4096, sparsity=0.0045, topX=10, seed=81, nonzero_full_rows=True, bias=True),
          orc.make_layer(3, 4096, 12288, sparsity=0.0045, topX=10, seed=82, nonzero_full_rows=True),
          orc.make_layer(4, 11008, 4096, sparsity=0.0045, topX=10, seed=83, nonzero_full_rows=True)]
    Ts = [to_torch(L) for L in Ls]
    xs = [make_activations(4096, 300, seed=81), make_activations(4096, 128, seed=82), make_activations(11008, 9, seed=83)]
    xb0, xg0 = bf16(xs[0])
    xg1 = torch.from_numpy(xs[1]).cuda().half()
    xg2 = torch.from_numpy(xs[2]).cuda()
    streams = [torch.cuda.Stream() for _ in range(3)]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    out = {}
    with torch.cuda.stream(streams[0]):
        out["bf16 tc"] = qc.lutgemm_fused(xg0, *_args(Ts[0], 4, Ts[0]["bias"]))
    with torch.cuda.stream(streams[1]):
        out["fp16 tc"] = qc.lutgemm_fused(xg1, *_args(Ts[1], 3))
    with torch.cuda.stream(streams[2]):
        y = torch.zeros((9, 4096), device="cuda")
        qc.vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(Ts[2]["rows"], Ts[2]["cols"], Ts[2]["vals"], xg2, Ts[2]["full_rows"],
                                                              Ts[2]["full_row_indices"], y, 4096, Ts[2]["qweight"], Ts[2]["lookup_table"])
        out["batched"] = y
    torch.cuda.synchronize()
    check(out["bf16 tc"], Ls[0], xb0, bias=Ls[0]["bias"], y_dtype="bfloat16")
    check(out["fp16 tc"], Ls[1], xs[1], y_dtype="float16")
    check(out["batched"], Ls[2], xs[2])


# ---- quant_cuda.lutgemm_fused -------------------------------------------------------------------------------------------------------
def test_pybind_bf16_in_bf16_out_and_fp32_raises(qc):
    K, N, M = 4096, 4096, 100
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=8, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    xb, xt = bf16(make_activations(K, M, seed=8))
    y = qc.lutgemm_fused(xt, *_args(T, 4, T["bias"]))
    torch.cuda.synchronize()
    assert y.dtype == torch.bfloat16 and y.shape == (M, N)
    check(y, L, xb, bias=L["bias"], y_dtype="bfloat16")
    with pytest.raises(RuntimeError, match="fp16 or bf16"):
        qc.lutgemm_fused(xt.float(), *_args(T, 4, T["bias"]))


# ---- QuantLinearLUT ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def spy(qc, monkeypatch):
    calls = []
    real = qc.lutgemm_fused

    def wrapped(*a, **kw):
        calls.append((tuple(a[0].shape), a[0].dtype))
        return real(*a, **kw)
    monkeypatch.setattr(qc, "lutgemm_fused", wrapped)
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


def test_module_routing(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    T = QuantLinearLUT.BF16_TC_MIN_ROWS
    assert T > QuantLinearLUT.TC_MIN_ROWS
    K = N = 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=12, nonzero_full_rows=True)
    xb, xt = bf16(make_activations(K, 2048, seed=12))
    for bias_on in (False, True):
        m = _module(L, bias=bias_on)
        bias = m.bias.cpu().numpy() if bias_on else None
        for M in (T, 2048):
            del spy[:]
            x = xt[:M].reshape(1, M, K)
            y = _run(m, x)
            assert spy == [((M, K), torch.bfloat16)]
            y_b = _run(m, x, fused=False)  # the batched branch
            assert y.dtype == y_b.dtype == (torch.float32 if bias_on else torch.bfloat16) and y.shape == y_b.shape == (1, M, N)
            rows = [0, 1, 2, 3, 63, 64, M - 1] + ([127, 128, 1000] if M > 128 else [])
            want = orc.forward_f64(L, xb[rows])  # the module rounds to bf16 first and adds the bias afterwards
            S = abs_sum(L, xb[rows], bias)
            r, eta = OUT_ROUNDING["bfloat16"]
            b = 0.0 if bias is None else bias.astype(np.float64)[None, :]
            assert bound_ratio(y[0][rows].float().cpu().numpy(), want + b, S, want, r, eta=eta) <= 1.0
    del spy[:]
    m = _module(L)
    _run(m, xt[:T - 1].reshape(1, T - 1, K))
    _run(m, xt[:T].reshape(1, T, K), fused=False)
    _run(m, xt[:T].float().reshape(1, T, K))
    assert spy == []


def test_misaligned_bf16_view_through_the_module_is_bit_identical(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 4096, 1024, QuantLinearLUT.BF16_TC_MIN_ROWS
    m = _module(orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=13, nonzero_full_rows=True), bias=True)
    _, xa = bf16(make_activations(K, M, seed=13))
    want = _run(m, xa)
    for off in (1, 3, 7):
        buf = torch.zeros(M * K + 8, device="cuda", dtype=torch.bfloat16)
        xv = buf[off:off + M * K].view(M, K)
        xv.copy_(xa)
        assert xv.is_contiguous() and xv.data_ptr() % 16
        assert torch.equal(_run(m, xv), want), off
        assert torch.equal(xv, xa)
    assert len(spy) == 4


def test_stacked_qkv_group_in_bf16(spy):
    from squeezellm_b200.fusion import fuse_siblings
    from squeezellm_b200.quant import QuantLinearLUT
    K, M = 512, QuantLinearLUT.BF16_TC_MIN_ROWS
    Ls = [orc.make_layer(4, K, n, sparsity=0.01, topX=3, seed=20 + n, nonzero_full_rows=True) for n in (256, 128, 192)]
    block = torch.nn.Module()
    for name, L in zip(("q_proj", "k_proj", "v_proj"), Ls):
        setattr(block, name, _module(L))
    assert len(fuse_siblings(block)) == 1
    xb, xt = bf16(make_activations(K, M, seed=21))
    x = xt.reshape(1, M, K)
    outs = [block.q_proj(x), block.k_proj(x), block.v_proj(x)]
    torch.cuda.synchronize()
    assert spy == [((M, K), torch.bfloat16)]
    for y, L in zip(outs, Ls):
        assert y.dtype == torch.bfloat16
        check(y[0], L, xb, y_dtype="bfloat16")


# ---- training ----------------------------------------------------------------------------------------------------------------------
def test_grad_forward_is_bit_identical_and_dx_takes_the_tensor_cores(qc, spy, monkeypatch):
    from squeezellm_b200 import quant
    QuantLinearLUT = quant.QuantLinearLUT
    K, N = 4096, 2048
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=90, nonzero_full_rows=True)
    m = _module(L)  # no bias: y and so dy stay bf16
    paths = []
    real_t = quant.quant_cuda.lutgemm_t

    def wrapped_t(*a, **kw):
        paths.append(kw.get("path"))
        return real_t(*a, **kw)
    monkeypatch.setattr(quant.quant_cuda, "lutgemm_t", wrapped_t)
    row_counts = sorted({QuantLinearLUT.BF16_TC_MIN_ROWS, max(QuantLinearLUT.BF16_TC_MIN_ROWS, QuantLinearLUT.BWD_TC_MIN_ROWS)})
    for rows in row_counts:
        _, xt = bf16(make_activations(K, rows, seed=90))
        with torch.no_grad():
            y0 = m(xt.reshape(1, rows, K))
        x = xt.reshape(1, rows, K).clone().requires_grad_(True)
        y = m(x)
        assert y.grad_fn is not None
        assert torch.equal(y.detach(), y0)
        y.float().sum().backward()
        assert x.grad is not None and x.grad.dtype == torch.bfloat16 and x.grad.shape == x.shape
        assert paths[-1] == ("tc" if rows >= QuantLinearLUT.BWD_TC_MIN_ROWS else "cuda")
    assert paths[-1] == "tc"
    assert spy == [((r, K), torch.bfloat16) for r in row_counts for _ in range(2)]  # with and without grad


def test_train_codebook_forward_is_the_plain_forward(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 1024, 512, QuantLinearLUT.BF16_TC_MIN_ROWS
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=4, seed=91, nonzero_full_rows=True)
    plain, trained = _module(L, bias=True), _module(L, bias=True)
    trained.train_codebook(lookup_table=True, vals=True, full_rows=True, bias=True)
    _, xt = bf16(make_activations(K, M, seed=91))
    with torch.no_grad():
        y0 = plain(xt)
    y1 = trained(xt)
    assert y1.grad_fn is not None
    assert torch.equal(y1.detach(), y0)
    y1.float().sum().backward()
    assert trained.lookup_table.grad is not None
    assert spy == [((M, K), torch.bfloat16)] * 2
