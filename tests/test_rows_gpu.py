"""The multi-row LUT-GEMV (`sqllm_lutgemv_rows`, `quant_cuda.lutgemv_rows`, csrc/lutgemv_rows.cuh) that runs fp16 inputs of 2 to
QuantLinearLUT.ROWS_MAX rows: every route-test shape at row counts on both sides of every row-group boundary against the fp64
oracle (fp32 y: the accumulation error alone), outlier and dense-row patterns, in_features and out_features at the edges of the
slab and strip tiling, bitwise reproducibility and row independence, the reference kernels' stored outputs, CUDA-graph replay,
several streams at once and the module routing."""
import ctypes
import os

import numpy as np
import pytest
import torch

from test_error_bound_host import SHAPES
from test_gpu_parity import BATCHED_SHAPES, batched_id, batched_inputs, ref_comparable
from util import (GOLDEN, OUT_ROUNDING, REL_TOL, TIGHT_TOL, Args, abs_sum, bound_ratio, load_lib, make_activations, orc, quant_layer,
                  rel_err, sample_idx, to_torch)

pytestmark = pytest.mark.gpu

M_ALL = [2, 8, 9, 63]
M_DENSE = [1, 2, 3, 7, 8, 9, 16, 17, 31, 32, 33, 63]  # both sides of the 2 / 4 / 8-row groups and of 16, 32, 48 rows
DENSE_SHAPES = [(4096, 12288, 4), (512, 132, 3), (512, 132, 4)]


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemv_rows.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


def rows_call(lib, L, x16, y_half=False, bias=None, T=None):
    """sqllm_lutgemv_rows on the layer dict L (numpy; T: its torch tensors, if the caller placed them) and fp16 x [M, K] (torch,
    cuda) -> y [M, N] as fp32 numpy (y is fp32 unless y_half)."""
    T = to_torch(L) if T is None else T
    M, N = x16.shape[0], L["outfeatures"]
    y = torch.empty((M, N), device="cuda", dtype=torch.float16 if y_half else torch.float32)
    a = Args(bits=L["bits"], in_features=L["infeatures"], out_features=N, batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    b = None if bias is None else torch.from_numpy(bias).cuda()
    rc = lib.sqllm_lutgemv_rows(ctypes.byref(a), x16.data_ptr(), y.data_ptr(), int(y_half), None if b is None else b.data_ptr(),
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    return y.float().cpu().numpy()


def check_f32(got, L, x, bias=None, record=None):
    """fp32 y against the oracle: rel_err within TIGHT_TOL and the condition-aware bound (bias inside the sum)."""
    want = orc.forward_f64(L, x, mul_init=None if bias is None else bias[None, :])
    ratio = bound_ratio(got, want, abs_sum(L, x, bias))
    if record is not None:
        record("bound_ratio", ratio)
    assert ratio <= 1.0, ratio
    assert rel_err(got, want) < TIGHT_TOL, rel_err(got, want)
    return want


# ---- accuracy through the C ABI, fp32 y ---------------------------------------------------------------------------------------------
_cache = {}


def layer_case(shape):
    """Layer (0.45 % CSR outliers, 10 dense rows, bias), 63 rows of prefill-like activations and the oracle on all of them."""
    if shape not in _cache:
        _cache.clear()
        K, N, bits = shape
        L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True, bias=True)
        x = make_activations(K, 63, seed=K + bits)
        _cache[shape] = (L, x, orc.forward_f64(L, x, mul_init=L["bias"][None, :]), abs_sum(L, x, L["bias"]))
    return _cache[shape]


def _accuracy_cases():
    out = []
    for K, N, bits in SHAPES:
        for M in sorted(set(M_ALL + (M_DENSE if (K, N, bits) in DENSE_SHAPES else []))):
            out.append(pytest.param((K, N, bits), M, id=f"w{bits}_{K}x{N}-M{M}"))
    return out


@pytest.mark.parametrize("shape,M", _accuracy_cases())
def test_c_abi_fp32_vs_oracle(lib, record, shape, M):
    L, x, want, S = layer_case(shape)
    got = rows_call(lib, L, torch.from_numpy(x[:M]).cuda().half(), bias=L["bias"])
    ratio = bound_ratio(got, want[:M], S[:M])
    record("bound_ratio", ratio)
    assert ratio <= 1.0, ratio
    assert rel_err(got, want[:M]) < TIGHT_TOL
    if M > 2:  # the all-zero row of make_activations: exactly the bias
        assert np.array_equal(got[2], L["bias"])


# ---- outliers ----------------------------------------------------------------------------------------------------------------------
def _dense_rows(L, topx, pattern, seed):
    """topX dense rows on a layer: 'channel0' puts every one on channel 0; 'mixed' has duplicates inside one strip, indices outside
    [0, N), and channel 0 and the last channel of the (ragged) last strip.  Returns the layer and its oracle twin (ignored
    indices dropped)."""
    K, N = L["infeatures"], L["outfeatures"]
    rng = np.random.default_rng(seed)
    fr = (rng.standard_normal((K, topx)) * 0.05 / max(1, topx) ** 0.5).astype(np.float32)
    if pattern == "channel0":
        fri = np.zeros(topx, dtype=np.int32)
    else:
        fri = rng.integers(0, N, size=topx).astype(np.int32)
        special = [0, N - 1, 70, 70, 71, -1, N, N + 1000, 65, 127]
        fri[:min(topx, len(special))] = special[:topx]
    L = dict(L, full_rows=fr, full_row_indices=fri)
    keep = (fri >= 0) & (fri < N)
    W = dict(L, full_rows=np.ascontiguousarray(fr[:, keep]), full_row_indices=np.ascontiguousarray(fri[keep]))
    if not keep.any():
        W["full_rows"] = W["full_row_indices"] = None
    return L, W


@pytest.mark.parametrize("topx,pattern", [(0, "none"), (1, "channel0"), (1, "mixed"), (33, "channel0"), (33, "mixed"),
                                          (128, "channel0"), (128, "mixed"), (300, "channel0"), (300, "mixed")])
def test_dense_row_patterns(lib, record, topx, pattern):
    K, N = 512, 132
    L = orc.make_layer(4, K, N, sparsity=0.01, seed=topx, bias=True)
    W = L
    if topx:
        L, W = _dense_rows(L, topx, pattern, seed=topx)
    x = make_activations(K, 9, seed=topx)
    got = rows_call(lib, L, torch.from_numpy(x).cuda().half(), bias=L["bias"])
    check_f32(got, W, x, L["bias"], record)


@pytest.mark.parametrize("case", ["empty_csr", "no_sparse_buffers"])
def test_empty_csr_and_no_sparse_buffers(lib, record, case):
    K, N = 1024, 132
    L = orc.make_layer(3, K, N, sparsity=0.0, topX=3, seed=2, nonzero_full_rows=True)
    if case == "empty_csr":
        L["rows"] = np.zeros(N + 1, dtype=np.int32)
        L["cols"] = np.zeros(0, dtype=np.int32)
        L["vals"] = np.zeros(0, dtype=np.float32)
    else:
        L["full_rows"] = L["full_row_indices"] = None
    x = make_activations(K, 8, seed=2)
    check_f32(rows_call(lib, L, torch.from_numpy(x).cuda().half()), L, x, record=record)


def _with_csr_row(L, c, cols, vals):
    """L with channel c's CSR row replaced by (cols, vals)."""
    rows, oc, ov = L["rows"], L["cols"], L["vals"]
    e0, e1 = rows[c], rows[c + 1]
    new_rows = rows.copy()
    new_rows[c + 1:] += len(cols) - (e1 - e0)
    return dict(L, rows=new_rows, cols=np.concatenate([oc[:e0], cols, oc[e1:]]).astype(np.int32),
                vals=np.concatenate([ov[:e0], vals, ov[e1:]]).astype(np.float32))


def test_one_row_with_3000_nonzeros(lib, record):
    K, N = 4096, 128
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=4, seed=6, nonzero_full_rows=True)
    rng = np.random.default_rng(6)
    L = _with_csr_row(L, 37, np.sort(rng.permutation(K)[:3000]), (rng.standard_normal(3000) * 0.01).astype(np.float32))
    x = make_activations(K, 9, seed=6)
    check_f32(rows_call(lib, L, torch.from_numpy(x).cuda().half()), L, x, record=record)


def test_shuffled_csr_rows(lib, record):
    """Shuffled column indices within each CSR row: within the bound of the oracle, and of the sorted rows."""
    L = orc.make_layer(4, 2048, 320, sparsity=0.02, seed=5, skew=True)
    rng = np.random.default_rng(5)
    U = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    for c in range(320):
        e0, e1 = L["rows"][c], L["rows"][c + 1]
        perm = rng.permutation(e1 - e0) + e0
        U["cols"][e0:e1], U["vals"][e0:e1] = L["cols"][perm], L["vals"][perm]
    assert not np.array_equal(U["cols"], L["cols"])
    x = make_activations(2048, 17, seed=5)
    xt = torch.from_numpy(x).cuda().half()
    got_u, got_s = rows_call(lib, U, xt), rows_call(lib, L, xt)
    check_f32(got_u, L, x, record=record)
    assert bound_ratio(got_u, got_s, abs_sum(L, x)) <= 1.0


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_csr_arrays_inside_a_buffer(lib, record, offset):
    """cols / vals (and rows) that start `offset` elements into a larger buffer: only 4-byte aligned."""
    K, N = 1024, 196
    L = orc.make_layer(3, K, N, sparsity=0.01, topX=5, seed=offset, nonzero_full_rows=True)
    T = to_torch(L)
    for k in ("rows", "cols", "vals"):
        buf = torch.zeros(T[k].numel() + 4, dtype=T[k].dtype, device="cuda")
        buf[offset:offset + T[k].numel()] = T[k]
        T[k] = buf[offset:offset + T[k].numel()]
        assert T[k].data_ptr() % 16
    x = make_activations(K, 5, seed=offset)
    check_f32(rows_call(lib, L, torch.from_numpy(x).cuda().half(), T=T), L, x, record=record)


# ---- edges of the tiling -----------------------------------------------------------------------------------------------------------
_EDGES = [(b, K, 132) for K in (32, 96, 160, 4128, 22016) for b in (3, 4)] + [(4, 256, N) for N in (4, 60, 64, 68, 132)] + [(4, 64, 131072)]


@pytest.mark.parametrize("bits,K,N", _EDGES, ids=[f"w{b}-{k}x{n}" for b, k, n in _EDGES])
def test_in_and_out_features_edges(lib, record, bits, K, N):
    """K from one unit to 22016 (odd unit counts, slabs that are not a multiple of S units), N from 4 to wider than
    SQLLM_FUSED_MAX_OUT / 2 (this route has no width limit)."""
    L = orc.make_layer(bits, K, N, sparsity=0.01, topX=3, seed=K + N, nonzero_full_rows=N >= 3, bias=True)
    x = make_activations(K, 9, seed=K)
    check_f32(rows_call(lib, L, torch.from_numpy(x).cuda().half(), bias=L["bias"]), L, x, L["bias"], record)


# ---- reproducibility -----------------------------------------------------------------------------------------------------------------
def test_bitwise_reproducible_and_rows_independent(lib):
    """Two calls give the same bits; a row's fp32 result is bit-identical whatever the other rows hold, at whatever position it
    sits and whatever M (and with it the rows per CTA: 2, 4 or 8) is."""
    K, N = 4096, 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=31, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = make_activations(K, 63, seed=31)
    other = make_activations(K, 63, seed=32)
    run = lambda xx: rows_call(lib, L, torch.from_numpy(np.ascontiguousarray(xx)).cuda().half(), bias=L["bias"], T=T)
    base = run(x)
    assert np.array_equal(base.view(np.uint32), run(x).view(np.uint32))
    probe = [0, 1, 3, 37]
    for M in (2, 3, 5, 8, 9, 17, 63):
        rows = [r for r in probe if r < M]
        assert np.array_equal(run(x[:M])[rows].view(np.uint32), base[rows].view(np.uint32)), f"M={M}"
        xn = other[:M].copy()
        xn[rows] = x[rows]
        assert np.array_equal(run(xn)[rows].view(np.uint32), base[rows].view(np.uint32)), f"new others M={M}"
    for M, pos in ((2, 1), (4, 3), (9, 8), (40, 22)):  # row 37 at another position
        xp = other[:M].copy()
        xp[pos] = x[37]
        assert np.array_equal(run(xp)[pos].view(np.uint32), base[37].view(np.uint32)), f"M={M} pos={pos}"
    # the all-zero row: exactly the bias, and exactly zero without one
    assert np.array_equal(base[2], L["bias"])
    y0 = rows_call(lib, L, torch.from_numpy(x[:5]).cuda().half(), T=T)
    assert np.array_equal(y0[2], np.zeros(N, np.float32))


# ---- through quant_cuda -----------------------------------------------------------------------------------------------------------
def _args(T, bits, bias=True):
    return (T["qweight"], T["lookup_table"], bits, T.get("bias") if bias else None, T["rows"], T["cols"], T["vals"], T["full_rows"],
            T["full_row_indices"])


def test_quant_cuda_fp16_output_vs_oracle_bound(qc, record):
    K, N, M = 4096, 11008, 7
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=8, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = make_activations(K, M, seed=8)
    y = qc.lutgemv_rows(torch.from_numpy(x).cuda().half(), *_args(T, 4))
    torch.cuda.synchronize()
    assert y.dtype == torch.float16 and y.shape == (M, N)
    want = orc.forward_f64(L, x, mul_init=L["bias"][None, :])
    r, eta = OUT_ROUNDING["float16"]
    ratio = bound_ratio(y.float().cpu().numpy(), want, abs_sum(L, x, L["bias"]), want, r, eta=eta)
    record("bound_ratio", ratio)
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("batch", [2, 5, 16])
@pytest.mark.parametrize("shape", [s for s in BATCHED_SHAPES if ref_comparable(s)], ids=batched_id)
def test_quant_cuda_vs_reference_kernels(qc, shape, batch):
    """The reference's own batched kernels on the same inputs (golden outputs); x is fp16-exact there."""
    g = np.load(os.path.join(GOLDEN, "reference_outputs.npz"))
    key = f"b{batch}__{batched_id(shape)}"
    L, x = batched_inputs(shape, batch)
    T = to_torch(L)
    y = qc.lutgemv_rows(torch.from_numpy(x).cuda().half(), *_args(T, shape[0], bias=False))
    got = y.float().cpu().numpy().reshape(-1)
    assert rel_err(got[sample_idx(got.size)], g[key], b_absmax=float(g[key + "__absmax"])) < REL_TOL


def test_graph_capture_and_replay_with_new_inputs(qc):
    K, N, M = 4096, 4096, 12
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=9, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = torch.from_numpy(make_activations(K, M, seed=1)).cuda().half()
    x2 = torch.from_numpy(make_activations(K, M, seed=2)).cuda().half()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        qc.lutgemv_rows(x, *_args(T, 3))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = qc.lutgemv_rows(x, *_args(T, 3))
    x.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, qc.lutgemv_rows(x2, *_args(T, 3)))


def test_three_streams_at_once(qc, record):
    """Three layers on three streams with no synchronisation between them: each matches its own call on one stream, bit for bit."""
    shapes = [(4, 4096, 12288, 8), (3, 11008, 4096, 5), (4, 4096, 22016, 33)]
    Ls = [orc.make_layer(b, K, N, sparsity=0.0045, topX=10, seed=50 + i, nonzero_full_rows=True, bias=True)
          for i, (b, K, N, _) in enumerate(shapes)]
    Ts = [to_torch(L) for L in Ls]
    xs = [torch.from_numpy(make_activations(K, M, seed=50 + i)).cuda().half() for i, (_, K, _, M) in enumerate(shapes)]
    alone = [qc.lutgemv_rows(xs[i], *_args(Ts[i], shapes[i][0])) for i in range(3)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [None] * 3
    for rep in range(3):
        for i, s in enumerate(streams):
            with torch.cuda.stream(s):
                outs[i] = qc.lutgemv_rows(xs[i], *_args(Ts[i], shapes[i][0]))
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(outs[i], alone[i]), i


# ---- QuantLinearLUT routing ---------------------------------------------------------------------------------------------------------
def _module(L, bias=False):
    return quant_layer(L, bias=L["bias"] if bias else None).cuda()


@pytest.fixture
def spy(qc, monkeypatch):
    calls = []
    real = qc.lutgemv_rows

    def wrapped(*a, **kw):
        calls.append(tuple(a[0].shape))
        return real(*a, **kw)
    monkeypatch.setattr(qc, "lutgemv_rows", wrapped)
    return calls


def test_module_routing(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K = N = 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=12, nonzero_full_rows=True)
    m = _module(L)
    x = make_activations(K, QuantLinearLUT.TC_MIN_ROWS, seed=12)
    top = min(QuantLinearLUT.ROWS_MAX, QuantLinearLUT.TC_MIN_ROWS - 1)
    for M in (2, top):
        y = m(torch.from_numpy(x[:M]).cuda().half().reshape(1, M, K))
        assert y.shape == (1, M, N) and y.dtype == torch.float16
        want = orc.forward_f64(L, x[:M])
        r, eta = OUT_ROUNDING["float16"]
        assert bound_ratio(y[0].float().cpu().numpy(), want, abs_sum(L, x[:M]), want, r, eta=eta) <= 1.0
    assert spy == [(2, K), (top, K)]
    m(torch.from_numpy(x[:1]).cuda().half().reshape(1, 1, K))
    m(torch.from_numpy(x).cuda().half())
    for xin in (torch.from_numpy(x[:8]).cuda(), torch.from_numpy(x[:8]).cuda().bfloat16()):
        m(xin)
    QuantLinearLUT.use_fused = False
    try:
        m(torch.from_numpy(x[:8]).cuda().half())
    finally:
        QuantLinearLUT.use_fused = True
    torch.cuda.synchronize()
    assert spy == [(2, K), (top, K)]


@pytest.mark.parametrize("bias", [False, True])
def test_module_output_dtype_and_shape_match_the_batched_branch(bias):
    """fp16 rows through the new route and through the batched symbols: same dtype (fp32 with a bias: out.to(fp16) + bias), shape
    and, within fp16 rounding, values."""
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 1024, 260, 6
    L = orc.make_layer(3, K, N, sparsity=0.01, topX=4, seed=13, nonzero_full_rows=True, bias=True)
    m = _module(L, bias=bias)
    if bias:
        m.bias = torch.from_numpy(L["bias"]).cuda()
    x = torch.from_numpy(make_activations(K, M, seed=13)).cuda().half().reshape(2, 3, K)
    y = m(x)
    QuantLinearLUT.use_fused = False
    try:
        yb = m(x)
    finally:
        QuantLinearLUT.use_fused = True
    assert y.shape == yb.shape == (2, 3, N) and y.dtype == yb.dtype == (torch.float32 if bias else torch.float16)
    assert rel_err(y.float().cpu().numpy(), yb.float().cpu().numpy()) < REL_TOL


def test_sibling_group_members_get_their_slices(spy):
    from squeezellm_b200.fusion import fuse_siblings
    K, M = 512, 9
    Ls = [orc.make_layer(4, K, n, sparsity=0.01, topX=3, seed=20 + n, nonzero_full_rows=True) for n in (256, 128, 192)]
    block = torch.nn.Module()
    for name, L, n in zip(("q_proj", "k_proj", "v_proj"), Ls, (256, 128, 192)):
        setattr(block, name, _module(L))
    assert len(fuse_siblings(block)) == 1
    x = make_activations(K, M, seed=21)
    xt = torch.from_numpy(x).cuda().half().reshape(1, M, K)
    outs = [block.q_proj(xt), block.k_proj(xt), block.v_proj(xt)]
    assert spy == [(M, K)]
    r, eta = OUT_ROUNDING["float16"]
    for y, L in zip(outs, Ls):
        want = orc.forward_f64(L, x)
        assert bound_ratio(y[0].float().cpu().numpy(), want, abs_sum(L, x), want, r, eta=eta) <= 1.0


@pytest.mark.parametrize("offset", [1, 3, 7])
def test_module_misaligned_x(spy, offset):
    """A contiguous fp16 view that starts `offset` elements into its storage gives the aligned input's result, bit for bit."""
    K, N, M = 4096, 4096, 5
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=14, nonzero_full_rows=True)
    m = _module(L)
    xa = torch.from_numpy(make_activations(K, M, seed=14)).cuda().half()
    buf = torch.zeros(M * K + 8, device="cuda", dtype=torch.float16)
    xv = buf[offset:offset + M * K].view(1, M, K)
    xv.copy_(xa.reshape(1, M, K))
    assert xv.is_contiguous() and xv.data_ptr() % 16
    y = m(xv)
    assert torch.equal(xv, xa.reshape(1, M, K))
    assert torch.equal(y, m(xa.reshape(1, M, K)))
    assert spy == [(M, K), (M, K)]
