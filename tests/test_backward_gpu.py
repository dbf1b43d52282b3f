"""The input gradient of QuantLinearLUT (`sqllm_lutgemm_t`, `quant_cuda.lutgemm_t`, csrc/lutgemm_t.cuh, and the autograd path of
QuantLinearLUT.forward): every route-test shape at row counts on both sides of every row-group boundary against the fp64 truth
(tests/backward_ref.py) per element, through the C ABI with fp32 dx; outlier and dense-row patterns; in_features and out_features
at the edges of the slab and strip tiling; bitwise reproducibility and row independence; CUDA-graph replay; several streams at
once; and the module level: autograd.grad, LoRA adapters over quantized layers, sibling groups, and the unchanged no-grad path.

The bound is that of the forward kernels (tests/util.py, bound_ratio): |got - want| <= r |want| + eta + (1 + r) e S with
S = sum_c |dy| |w| and e = 2^-20; r, eta the rounding of dx to its dtype (0 for fp32 dx)."""
import ctypes

import numpy as np
import pytest
import torch

from backward_ref import backward_and_abs_sum, backward_f64
from test_error_bound_host import SHAPES
from util import OUT_ROUNDING, Args, bound_ratio, load_lib, make_activations, orc, quant_layer, to_torch

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 0, 1, 2
DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
M_ALL = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129]
SEVEN_B = {(4096, 12288, 4), (4096, 4096, 3), (4096, 22016, 4), (11008, 4096, 3)}


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemm_t.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_void_p]
    return lib


def t_call(lib, L, dy, path=2, T=None, dx_dtype=torch.float32, stream=None, sync=True):
    """sqllm_lutgemm_t on the layer dict L (numpy; T: its torch tensors) and dy [M, N] (torch, cuda) -> dx [M, K] (torch)."""
    T = to_torch(L) if T is None else T
    M, K = dy.shape[0], L["infeatures"]
    dx = torch.empty((M, K), device="cuda", dtype=dx_dtype)
    a = Args(bits=L["bits"], in_features=K, out_features=L["outfeatures"], batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = lib.sqllm_lutgemm_t(ctypes.byref(a), dy.data_ptr(), DT[dy.dtype], dx.data_ptr(), DT[dx_dtype], path, st)
    assert rc == 0, lib.sqllm_last_error()
    if sync:
        torch.cuda.synchronize()
    return dx


def check(got, L, dy_exact, r=0.0, eta=0.0, want_S=None):
    """got (torch) against the fp64 truth for dy_exact (numpy: the values the kernel saw) within the bound."""
    want, S = backward_and_abs_sum(L, dy_exact) if want_S is None else want_S
    ratio = bound_ratio(got.double().cpu().numpy(), want, S, r=r, eta=eta)
    assert ratio <= 1.0, ratio
    return ratio


def _layer(K, N, bits, seed, topX=10, sparsity=0.0045):
    return orc.make_layer(bits, K, N, sparsity=sparsity, topX=topX, seed=seed, nonzero_full_rows=topX > 0)


def _dy(N, M, dtype, seed):
    """make_activations-style gradient rows (1e-3 .. 1e2, row 2 all zero) in dtype, and the exact values as fp64 numpy."""
    if N < 16:  # too narrow for make_activations' fixed channels: N(0, 1) rows scaled by 1e-3 .. 1e2
        g = np.random.default_rng(seed).standard_normal((M, N)) * (10.0 ** np.linspace(-3, 2, M))[:, None]
        d = torch.from_numpy(g.astype(np.float32)).cuda().to(dtype)
        return d, d.double().cpu().numpy()
    d = torch.from_numpy(make_activations(N, M, seed=seed)).cuda().to(dtype)
    return d, d.double().cpu().numpy()


def paths(dtype):
    """The kernels that take dy of this dtype: tensor cores (1) for fp16 / bf16, CUDA cores (2) for all."""
    return (1, 2) if dtype != torch.float32 else (2,)


# every (K, N) of the route tests at both bit widths
KN = sorted({(k, n) for k, n, _ in SHAPES})
ALL_SHAPES = [(k, n, b) for k, n in KN for b in (3, 4)]


# ---- every route-test shape, every row count, every dy dtype, both kernels, through the C ABI with fp32 dx ------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
@pytest.mark.parametrize("K,N,bits", ALL_SHAPES, ids=[f"w{b}_{k}x{n}" for k, n, b in ALL_SHAPES])
def test_per_element_all_rows(lib, K, N, bits, dtype):
    L = _layer(K, N, bits, seed=K + N + bits)
    T = to_torch(L)
    Mmax = 2048 if (K, N) in {(k, n) for k, n, _ in SEVEN_B} else max(M_ALL)
    dy, dy_np = _dy(N, Mmax, dtype, seed=N)
    # truth for the first 129 rows and, at 2048 rows, every 16th row beyond (a row's result does not depend on M)
    keep = np.unique(np.concatenate([np.arange(max(M_ALL)), np.arange(max(M_ALL), Mmax, 16)]))
    want, S = backward_and_abs_sum(L, dy_np[keep])
    for M in M_ALL + ([2048] if Mmax == 2048 else []):
        got = {}
        for path in paths(dtype):
            got[path] = t_call(lib, L, dy[:M].contiguous(), path=path, T=T)
            dx = got[path].double().cpu().numpy()
            k = keep[keep < M]
            ratio = bound_ratio(dx[k], want[:len(k)], S[:len(k)])
            assert ratio <= 1.0, (M, path, ratio)
            if M > 2:
                assert (dx[2] == 0).all()  # the all-zero row
        auto = 1 if dtype != torch.float32 and M >= 96 else 2  # SQLLM_BWD_TC_MIN_ROWS
        assert torch.equal(t_call(lib, L, dy[:M].contiguous(), path=0, T=T), got[auto])


# ---- outliers and dense rows --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("topX", [1, 33, 128, 300])
@pytest.mark.parametrize("bits", [3, 4])
def test_dense_rows(lib, bits, topX):
    K, N = 1024, 640
    L = _layer(K, N, bits, seed=topX + bits, topX=topX, sparsity=0.01)
    fri = np.random.default_rng(topX).integers(0, N, size=topX).astype(np.int32)
    if topX >= 33:
        fri[:5] = fri[0]          # duplicates in one 64-column strip: they add up
        fri[5] = 0                # column 0
        fri[6] = N - 1            # the last column
        fri[7] = N + 3            # out of range: ignored
        fri[8] = -2
    L["full_row_indices"] = fri
    for M in (1, 9, 65):
        for dtype in (torch.float32, torch.float16, torch.bfloat16):
            dy, dy_np = _dy(N, M, dtype, seed=M)
            for path in paths(dtype):
                check(t_call(lib, L, dy, path=path), L, dy_np)


def test_all_dense_rows_on_channel_0(lib):
    K, N = 512, 132
    L = _layer(K, N, 4, seed=3, topX=40)
    L["full_row_indices"] = np.zeros(40, dtype=np.int32)
    dy, dy_np = _dy(N, 9, torch.float16, seed=4)
    for path in (1, 2):
        check(t_call(lib, L, dy, path=path), L, dy_np)


@pytest.mark.parametrize("path", [1, 2])
def test_csr_edges(lib, path):
    """Empty CSR, no sparse buffers, one 3000-entry CSR row, duplicate and out-of-range CSR columns, shuffled rows (against the
    truth and the sorted copy), CSR arrays 1-3 elements into a buffer."""
    K, N, bits = 4096, 132, 4
    dy, dy_np = _dy(N, 17, torch.float16 if path == 1 else torch.float32, seed=5)
    base = _layer(K, N, bits, seed=6, topX=0, sparsity=0.01)
    empty = dict(base, rows=np.zeros(N + 1, dtype=np.int32), cols=np.zeros(0, dtype=np.int32), vals=np.zeros(0, dtype=np.float32))
    check(t_call(lib, empty, dy, path=path), empty, dy_np)
    none = dict(base, rows=None, cols=None, vals=None)
    check(t_call(lib, none, dy, path=path), none, dy_np)
    # one 3000-entry row on channel 70, plus a duplicated and two out-of-range columns
    rng = np.random.default_rng(7)
    counts = np.diff(base["rows"])
    counts[70] = 3000
    rows = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    cols = np.concatenate([np.sort(rng.permutation(K)[:c]) for c in counts]).astype(np.int32)
    vals = (rng.standard_normal(len(cols)) * 0.1).astype(np.float32)
    cols[rows[70] + 1] = cols[rows[70]]
    cols[rows[3]] = K + 1
    cols[rows[4]] = -1
    big = dict(base, rows=rows, cols=cols, vals=vals)
    sorted_dx = t_call(lib, big, dy, path=path)
    want_S = backward_and_abs_sum(big, dy_np)
    check(sorted_dx, big, dy_np, want_S=want_S)
    shuf, svals = cols.copy(), vals.copy()
    for c in range(N):
        seg = slice(rows[c], rows[c + 1])
        perm = rng.permutation(rows[c + 1] - rows[c])
        shuf[seg] = cols[seg][perm]
        svals[seg] = vals[seg][perm]
    shuffled = dict(big, cols=shuf, vals=svals)
    shuf_dx = t_call(lib, shuffled, dy, path=path)
    check(shuf_dx, shuffled, dy_np, want_S=want_S)
    assert bound_ratio(shuf_dx.double().cpu().numpy(), sorted_dx.double().cpu().numpy(), want_S[1]) <= 1.0
    # CSR arrays starting 1-3 elements into a buffer
    for off in (1, 2, 3):
        T = to_torch(big)
        for k in ("rows", "cols", "vals"):
            buf = torch.zeros(T[k].numel() + off, dtype=T[k].dtype, device="cuda")
            buf[off:] = T[k]
            T[k] = buf[off:]
        check(t_call(lib, big, dy, T=T, path=path), big, dy_np, want_S=want_S)


@pytest.mark.parametrize("K", [32, 96, 160, 4128])
@pytest.mark.parametrize("N", [1, 4, 60, 64, 66, 68, 132])
@pytest.mark.parametrize("bits", [3, 4])
def test_tiling_edges(lib, bits, K, N):
    L = _layer(K, N, bits, seed=K * 7 + N, topX=min(3, N), sparsity=0.02)
    for M in (1, 5, 9, 130):
        for dtype in (torch.float16, torch.bfloat16, torch.float32):
            dy, dy_np = _dy(N, M, dtype, seed=M + N)
            want_S = backward_and_abs_sum(L, dy_np)
            for path in paths(dtype):
                check(t_call(lib, L, dy, path=path), L, dy_np, want_S=want_S)


def tc_limit(L, dy):
    """The tensor-core kernel's documented absolute term: each weight is kept to 2^-39 of the largest |w| of its 64-column chunk
    (the lo part's fp16 subnormal step), so dx[m][k] may be off by up to 2^-39 sum_chunks max|w| sum_(c in chunk) |dy[m][c]|.
    The chunk's largest weight is taken over all of K (the kernel's is over one 128-input tile): an upper bound.  [M, 1]."""
    from backward_ref import dense_w_f64
    W = np.abs(dense_w_f64(L))
    ady = np.abs(np.asarray(dy, dtype=np.float64))
    eta = np.zeros((ady.shape[0], 1))
    for c0 in range(0, W.shape[1], 64):
        eta[:, 0] += W[:, c0:c0 + 64].max() * ady[:, c0:c0 + 64].sum(axis=1)
    return 2.0 ** -39 * eta


@pytest.mark.parametrize("path", [1, 2])
def test_tiny_next_to_large_centroids_and_huge_outlier(lib, path):
    """Centroids of 1e-6 next to 1e-1 in one 64-column chunk (the tiny group against its own magnitude), and a CSR outlier 1e6 x its
    channel's largest centroid (against the whole chunk: on the tensor cores a weight more than about 2^20 below the largest
    weight of its chunk is kept to about 2^-40 of that weight, include/sqllm_b200.h)."""
    K, N, bits = 1024, 128, 4
    L = _layer(K, N, bits, seed=9, topX=0, sparsity=0.005)
    lut = L["lookup_table"].copy()
    lut[:32] *= 1e-6 / 0.02
    lut[32:64] *= 1e-1 / 0.02
    L["lookup_table"] = lut
    dt = torch.float16 if path == 1 else torch.float32
    dy, dy_np = _dy(N, 9, dt, seed=10)
    check(t_call(lib, L, dy, path=path), L, dy_np)
    small = dy.clone()
    small[:, 32:] = 0  # only the tiny group: its own magnitude, plus (tensor cores) the documented absolute term
    assert small[:, :32].abs().max() > 0
    small_np = small.double().cpu().numpy()
    want, S = backward_and_abs_sum(L, small_np)
    ratio = bound_ratio(t_call(lib, L, small, path=path).double().cpu().numpy(), want, S,
                        eta=tc_limit(L, small_np) if path == 1 else 0.0)
    assert ratio <= 1.0, ratio
    c = 40
    e = L["rows"][c]
    assert L["rows"][c + 1] > e
    L["vals"] = L["vals"].copy()
    L["vals"][e] = 1e6 * np.abs(lut[c]).max()
    want, S = backward_and_abs_sum(L, dy_np)  # tensor cores: the outlier sets its chunk's scale, the absolute term grows with it
    ratio = bound_ratio(t_call(lib, L, dy, path=path).double().cpu().numpy(), want, S, eta=tc_limit(L, dy_np) if path == 1 else 0.0)
    assert ratio <= 1.0, ratio
    if path == 2:  # exact fp32 codebook: the tiny group keeps its own accuracy next to the outlier too
        check(t_call(lib, L, small, path=path), L, small.double().cpu().numpy())


# ---- reproducibility, row independence, graphs, streams -----------------------------------------------------------------
def test_bitwise_reproducible_and_row_independent(lib):
    K, N, bits = 4096, 4096, 3
    L = _layer(K, N, bits, seed=11)
    T = to_torch(L)
    dy, _ = _dy(N, 77, torch.float16, seed=12)
    a = t_call(lib, L, dy, T=T)
    b = t_call(lib, L, dy, T=T)
    assert torch.equal(a, b)
    for M in (1, 2, 3, 5, 9, 64):
        for start in (0, 13):
            part = t_call(lib, L, dy[start:start + M].contiguous(), T=T)
            assert torch.equal(part, a[start:start + M]), (M, start)
    other = dy.clone()
    other[1:] = other[1:].flip(0)  # row 0 kept, every other row changed
    assert torch.equal(t_call(lib, L, other, T=T)[0], a[0])
    for dt in (torch.float16, torch.bfloat16):  # the tensor-core kernel: two calls, same bits
        d, _ = _dy(N, 200, dt, seed=17)
        assert torch.equal(t_call(lib, L, d, T=T, path=1), t_call(lib, L, d, T=T, path=1))


@pytest.mark.parametrize("path", [1, 2])
def test_cuda_graph_replay(lib, path):
    K, N, bits = 4096, 4096, 4
    L = _layer(K, N, bits, seed=13)
    T = to_torch(L)
    M = 24 if path == 2 else 200
    dy, _ = _dy(N, M, torch.bfloat16, seed=14)
    static = dy.clone()
    dx = torch.empty((M, K), device="cuda")
    t_call(lib, L, static, T=T, path=path)  # warm-up (sets the kernel's shared-memory limit outside the capture)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = t_call(lib, L, static, T=T, stream=s, sync=False, path=path)
    for seed in (15, 16):
        new, new_np = _dy(N, M, torch.bfloat16, seed=seed)
        static.copy_(new)
        g.replay()
        torch.cuda.synchronize()
        dx.copy_(out)
        assert torch.equal(dx, t_call(lib, L, new, T=T, path=path))
        check(dx, L, new_np)


def test_three_streams_at_once(lib):
    K, N = 4096, 4096
    layers = [_layer(K, N, b, seed=20 + i) for i, b in enumerate((4, 3, 4))]
    Ts = [to_torch(L) for L in layers]
    dys = [_dy(N, m, dt, seed=30 + m)[0] for m, dt in ((5, torch.float16), (40, torch.float32), (130, torch.bfloat16))]
    alone = [t_call(lib, L, d, T=T, path=0) for L, d, T in zip(layers, dys, Ts)]  # 130 bf16 rows: tensor cores
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = []
    torch.cuda.synchronize()
    for L, d, T, s in zip(layers, dys, Ts, streams):
        with torch.cuda.stream(s):
            outs.append(t_call(lib, L, d, T=T, stream=s, sync=False, path=0))
    torch.cuda.synchronize()
    for o, a in zip(outs, alone):
        assert torch.equal(o, a)


# ---- module level -------------------------------------------------------------------------------------------------------
def _module(L, bias=False):
    K, N = L["infeatures"], L["outfeatures"]
    return quant_layer(L, bias=np.random.default_rng(K).standard_normal(N).astype(np.float32) if bias else None).cuda()


@pytest.fixture
def deterministic():
    """The one-GEMV kernel's default mode adds its partial sums in arrival order (last bits vary from run to run): comparisons of
    two forwards for bit equality run in the deterministic mode."""
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.set_deterministic(True)
    yield
    quant_cuda.set_deterministic(False)


@pytest.fixture
def fused_mode(deterministic):
    from squeezellm_b200.quant import QuantLinearLUT
    old = QuantLinearLUT.use_fused
    yield QuantLinearLUT
    QuantLinearLUT.use_fused = old


@pytest.mark.parametrize("use_fused", [True, False])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["f16", "bf16", "f32"])
def test_autograd_grad_matches_truth(fused_mode, dtype, bias, use_fused):
    fused_mode.use_fused = use_fused
    K, N = 4096, 1024
    L = _layer(K, N, 4, seed=40)
    m = _module(L, bias)
    for shape in ((1, 1, K), (1, 5, K), (2, 40, K), (96, K)):  # decode, few rows, 3-D prefill, tensor-core rows
        x = torch.from_numpy(make_activations(K, int(np.prod(shape[:-1])), seed=41)).cuda().to(dtype).reshape(shape).requires_grad_()
        y = m(x)
        g = torch.randn(y.shape, device="cuda", dtype=torch.float32).to(y.dtype)
        (dx,) = torch.autograd.grad(y, x, g)
        assert dx.dtype == x.dtype and dx.shape == x.shape
        r, eta = OUT_ROUNDING[str(dtype).split(".")[1]]
        check(dx.reshape(-1, K), L, g.double().cpu().numpy().reshape(-1, N), r=r, eta=eta)
        with torch.no_grad():
            assert_same_forward(y, m(x), reproducible_route(x, use_fused))


def reproducible_route(x, use_fused=True):
    """Routes whose forward gives the same bits on every call: the fused decode kernel (deterministic mode), the rows kernel and
    the tensor-core kernel - fused, and one row or fp16 x.  The reference's 12 symbols and the _batched symbols add with atomics in
    arrival order."""
    return use_fused and (x.shape[-1] == x.numel() or x.dtype == torch.float16)


def assert_same_forward(y_grad, y0, exact):
    """The grad path's forward takes the route the plain forward takes: the same bits on a reproducible route, else the same
    values up to the order of the atomic additions."""
    assert y_grad.dtype == y0.dtype and y_grad.shape == y0.shape
    if exact:
        assert torch.equal(y_grad.detach(), y0)
    else:
        r = OUT_ROUNDING[str(y0.dtype).split(".")[1]][0]  # one rounding of the output apart
        torch.testing.assert_close(y_grad.detach().float(), y0.float(), rtol=2 * r + 1e-5, atol=1e-5 * y0.float().abs().max().item())


def test_lora_adapters_over_quantized_layers():
    """h = base(x) + B(A(x)) twice; adapter gradients against an fp64 dense re-implementation."""
    torch.manual_seed(0)
    K, H, r = 1024, 512, 8
    L1, L2 = _layer(K, H, 4, seed=50), _layer(H, K, 3, seed=51)
    q1, q2 = _module(L1), _module(L2)
    A1, B1 = (torch.randn(K, r, device="cuda") * 0.05).requires_grad_(), (torch.randn(r, H, device="cuda") * 0.05).requires_grad_()
    A2, B2 = (torch.randn(H, r, device="cuda") * 0.05).requires_grad_(), (torch.randn(r, K, device="cuda") * 0.05).requires_grad_()
    x = torch.randn(6, K, device="cuda")
    h = q1(x) + (x @ A1) @ B1
    h = torch.tanh(h)
    out = q2(h) + (h @ A2) @ B2
    loss = (out ** 2).sum()
    grads = torch.autograd.grad(loss, [A1, B1, A2, B2])
    W1 = torch.from_numpy(backward_ref_dense(L1)).cuda()
    W2 = torch.from_numpy(backward_ref_dense(L2)).cuda()
    P = [p.detach().double().requires_grad_() for p in (A1, B1, A2, B2)]
    xd = x.double()
    hd = torch.tanh(xd @ W1 + (xd @ P[0]) @ P[1])
    od = hd @ W2 + (hd @ P[2]) @ P[3]
    want = torch.autograd.grad((od ** 2).sum(), P)
    for g, w in zip(grads, want):
        err = (g.double() - w).abs().max().item() / w.abs().max().item()
        assert err < 1e-4, err


def backward_ref_dense(L):
    from backward_ref import dense_w_f64
    return dense_w_f64(L)


def test_sibling_group_matches_members():
    from squeezellm_b200.fusion import fuse_siblings
    K = 1024
    Ls = [_layer(K, n, 4, seed=60 + i) for i, n in enumerate((1024, 256, 256))]

    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj, self.v_proj = (_module(L) for L in Ls)

    x0 = torch.from_numpy(make_activations(K, 70, seed=61)).cuda().half().reshape(2, 35, K)
    gs = [torch.randn(2, 35, L["outfeatures"], device="cuda").half() for L in Ls]
    want = []
    plain = Attn()
    for name in ("q_proj", "k_proj", "v_proj"):
        x = x0.clone().requires_grad_()
        (dx,) = torch.autograd.grad(getattr(plain, name)(x), x, gs[("q_proj", "k_proj", "v_proj").index(name)])
        want.append(dx.float())
    fused = Attn()
    assert len(fuse_siblings(fused)) == 1
    x = x0.clone().requires_grad_()
    ys = [fused.q_proj(x), fused.k_proj(x), fused.v_proj(x)]
    (dx,) = torch.autograd.grad(ys, x, gs)
    ref = sum(want)
    S = sum(w.abs() for w in want)
    assert (dx.float() - ref).abs().le(2.0 ** -10 * S + 2.0 ** -10 * ref.abs() + 1e-6).all()


def test_no_grad_calls_and_bits_unchanged(monkeypatch, deterministic):
    """With requires_grad=False or under no_grad, the forward calls exactly the extension functions it calls without this
    feature; the outputs are bit-identical with and without grad enabled, and the grad path calls the same functions."""
    from squeezellm_b200 import quant
    K, N = 4096, 1024
    L = _layer(K, N, 4, seed=70)
    m = _module(L, bias=True)
    names = [n for n in dir(quant.quant_cuda) if n.startswith(("lutge", "vecquant"))]
    calls = []
    for n in names:
        real = getattr(quant.quant_cuda, n)
        monkeypatch.setattr(quant.quant_cuda, n, (lambda real, n: lambda *a, **kw: (calls.append(n), real(*a, **kw))[1])(real, n))
    for shape, dtype in (((1, 1, K), torch.float16), ((1, 1, K), torch.float32), ((8, K), torch.float16), ((8, K), torch.bfloat16),
                         ((128, K), torch.float16), ((128, K), torch.float32)):
        x = torch.from_numpy(make_activations(K, int(np.prod(shape[:-1])), seed=71)).cuda().to(dtype).reshape(shape)
        calls.clear()
        y0 = m(x)
        plain = list(calls)
        assert y0.grad_fn is None and "lutgemm_t" not in plain
        calls.clear()
        with torch.no_grad():
            y1 = m(x.clone().requires_grad_())
        assert calls == plain and y1.grad_fn is None
        calls.clear()
        xg = x.clone().requires_grad_()
        y2 = m(xg)
        assert calls == plain and y2.grad_fn is not None
        assert_same_forward(y1, y0, reproducible_route(x))
        assert_same_forward(y2, y0, reproducible_route(x))
        calls.clear()
        y2.sum().backward()
        assert calls == ["lutgemm_t"]
        assert xg.grad.dtype == x.dtype and xg.grad.shape == x.shape


def test_module_backward_routing(monkeypatch):
    """fp16 / bf16 gradients of at least BWD_TC_MIN_ROWS rows take the tensor cores, all others the CUDA cores."""
    from squeezellm_b200 import quant
    QuantLinearLUT = quant.QuantLinearLUT
    K, N = 1024, 512
    m = _module(_layer(K, N, 4, seed=80))
    seen = []
    real = quant.quant_cuda.lutgemm_t
    monkeypatch.setattr(quant.quant_cuda, "lutgemm_t", lambda *a, **kw: (seen.append((a[0].shape[0], a[0].dtype, kw["path"])),
                                                                        real(*a, **kw))[1])
    T = QuantLinearLUT.BWD_TC_MIN_ROWS
    for rows, dtype in ((T - 1, torch.float16), (T, torch.float16), (T, torch.bfloat16), (T, torch.float32), (1, torch.bfloat16)):
        x = torch.randn(rows, K, device="cuda", dtype=dtype, requires_grad=True)
        m(x).sum().backward()
        want = "tc" if dtype != torch.float32 and rows >= T else "cuda"
        assert seen[-1] == (rows, dtype, want), seen[-1]


def test_modified_buffers_between_forward_and_backward_raise():
    K, N = 1024, 512
    m = _module(_layer(K, N, 4, seed=81))
    x = torch.randn(8, K, device="cuda", dtype=torch.float16, requires_grad=True)
    y = m(x)
    m.lookup_table.mul_(2.0)  # e.g. a weight reload in place
    with pytest.raises(RuntimeError, match="modified or replaced"):
        y.sum().backward()
