"""bf16 decode on the fused kernels: one bf16 row through the one-GEMV kernels (`sqllm_lutgemv_fused_dt`, `quant_cuda.lutgemv_fused`;
lutgemv2_kernel in the default mode, the multi-row kernel at one row in the deterministic one) and 2 to QuantLinearLUT.BF16_ROWS_MAX bf16 rows
through the multi-row GEMV (`sqllm_lutgemv_rows_dt`, `quant_cuda.lutgemv_rows_bf16`).  The truth is the fp64 oracle on the
bf16-rounded activations; the metric is the per-element bound of tests/util.py (bound_ratio <= 1) beside rel_err < TIGHT_TOL, both
with fp32 output.  Covered: the parity shapes at both bit widths, narrow and wide layers, dense-row and CSR edge cases in both
summation modes, activations fp16 cannot hold, bf16 output, fp16 / fp32 x through the new entry points, the fp16 table mode,
reproducibility and row independence, graphs and streams, the module routing, training and the paths that stay fp16 / fp32."""
import ctypes

import numpy as np
import pytest
import torch

from test_backward_gpu import _module
from test_error_bound_host import SHAPES
from util import OUT_ROUNDING, TIGHT_TOL, Args, abs_sum, bound_ratio, load_lib, make_activations, orc, rel_err, to_torch

pytestmark = pytest.mark.gpu

F32, F16, BF16 = 0, 1, 2
DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemv_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.sqllm_lutgemv_fused.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.sqllm_lutgemv_rows_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_void_p]
    lib.sqllm_lutgemv_rows.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    lib.sqllm_workspace_error.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    yield lib
    lib.sqllm_set_deterministic(0)
    lib.sqllm_set_lut_mode(0)


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def _args(T, L, M):
    a = Args(bits=L["bits"], in_features=L["infeatures"], out_features=L["outfeatures"], batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    return a


def fused_dt(lib, L, T, x, y_dtype=torch.float32, bias=None, old=False):
    """One row x [K] (torch, cuda, fp32 / fp16 / bf16) through sqllm_lutgemv_fused_dt (old: sqllm_lutgemv_fused) -> y [N] (torch)."""
    a = _args(T, L, 1)
    nbytes = lib.sqllm_workspace_bytes(L["bits"], L["infeatures"], L["outfeatures"], a.topX)
    assert nbytes > 0
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    y = torch.empty(L["outfeatures"], dtype=y_dtype, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    b = None if bias is None else bias.data_ptr()
    if old:
        rc = lib.sqllm_lutgemv_fused(ctypes.byref(a), x.data_ptr(), int(x.dtype == torch.float16), y.data_ptr(),
                                     int(y_dtype == torch.float16), b, ws.data_ptr(), nbytes, st)
    else:
        rc = lib.sqllm_lutgemv_fused_dt(ctypes.byref(a), x.data_ptr(), DT[x.dtype], y.data_ptr(), DT[y_dtype], b, ws.data_ptr(), nbytes, st)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    assert lib.sqllm_workspace_error(ws.data_ptr(), st) == 0
    return y


def rows_dt(lib, L, T, x, y_dtype=torch.float32, bias=None, old=False):
    """x [M, K] (torch, cuda, fp16 / bf16) through sqllm_lutgemv_rows_dt (old: sqllm_lutgemv_rows) -> y [M, N] (torch)."""
    a = _args(T, L, x.shape[0])
    y = torch.empty((x.shape[0], L["outfeatures"]), dtype=y_dtype, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    b = None if bias is None else bias.data_ptr()
    if old:
        rc = lib.sqllm_lutgemv_rows(ctypes.byref(a), x.data_ptr(), y.data_ptr(), int(y_dtype == torch.float16), b, st)
    else:
        rc = lib.sqllm_lutgemv_rows_dt(ctypes.byref(a), x.data_ptr(), DT[x.dtype], y.data_ptr(), DT[y_dtype], b, st)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    return y


def bf16(x):
    """numpy fp32 -> its bf16 rounding (fp32 numpy) and the bf16 tensor on the GPU."""
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda().bfloat16()
    return t.float().cpu().numpy(), t


def check(got, L, xb, bias=None, y_dtype="float32", old=True):
    """bound_ratio <= 1 (and rel_err < TIGHT_TOL on fp32 output) of got [M, N] against the oracle on the bf16-exact rows xb [M, K],
    the bias inside the sum."""
    got = got.float().cpu().numpy() if isinstance(got, torch.Tensor) else got
    got = got.reshape(xb.shape[0], -1)
    want = orc.forward_f64(L, xb, mul_init=None if bias is None else bias[None, :])
    r, eta = OUT_ROUNDING[y_dtype]
    ratio = bound_ratio(got, want, abs_sum(L, xb, bias), want, r, eta=eta)
    assert ratio <= 1.0, ratio
    if old and y_dtype == "float32":
        e = rel_err(got, want)
        assert e < TIGHT_TOL, e
    return ratio


class Mode:
    """The summation mode (sqllm_set_deterministic) for the duration of a block, set through the C ABI and through quant_cuda."""

    def __init__(self, lib, det):
        from squeezellm_b200.quant import quant_cuda
        self.lib, self.qc, self.det = lib, quant_cuda, det

    def __enter__(self):
        self.lib.sqllm_set_deterministic(int(self.det))
        self.qc.set_deterministic(bool(self.det))

    def __exit__(self, *exc):
        self.lib.sqllm_set_deterministic(0)
        self.qc.set_deterministic(False)


# ---- layers: the parity shapes and the outlier edge cases ------------------------------------------------------------------------
def _edge_layer(case):
    """Layers whose outliers sit at the edges of both kernels' work split: topX on channel 0, duplicates inside one strip, channel 0
    and the last column of a ragged strip; an empty CSR, no sparse buffers, one 3000-entry CSR row, CSR arrays that start 1 to 3
    elements into a buffer."""
    kind, *p = case
    if kind == "shape":
        K, N, bits = p
        return orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True, bias=True), 0
    if kind == "topx":
        topx, pattern = p
        K, N = 1024, 1000
        rng = np.random.default_rng(topx)
        L = orc.make_layer(4, K, N, sparsity=0.01, topX=min(topx, N), seed=topx, nonzero_full_rows=True, bias=True)
        if pattern == "chan0":
            fri = np.zeros(topx, dtype=np.int32)
        else:  # duplicates inside the strip [512, 576), channel 0, the last column of the ragged last strip, the rest spread
            fri = rng.integers(0, N, size=topx).astype(np.int32)
            fri[0::4] = 512 + rng.integers(0, 64, size=len(fri[0::4]))
            fri[1::4] = 0
            fri[2::4] = N - 1
        L["full_row_indices"] = fri
        m = np.bincount(fri, minlength=N)[fri]  # rows on one channel scaled by 1/m: the channel's sum keeps one row's size
        L["full_rows"] = (L["full_rows"] / m[None, :]).astype(np.float32)
        return L, 0
    K, N = 2048, 1000
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=4, seed=7, nonzero_full_rows=True, bias=True)
    if kind == "empty_csr":
        L["rows"], L["cols"], L["vals"] = np.zeros(N + 1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32)
    elif kind == "no_sparse":
        for k in ("rows", "cols", "vals", "full_rows", "full_row_indices"):
            L[k] = None
    elif kind == "long_row":  # 3000 entries in one row, next to rows of 0 to 8
        K = 4096
        L = orc.make_layer(4, K, N, topX=4, seed=8, nonzero_full_rows=True, bias=True)
        rng = np.random.default_rng(3)
        counts = rng.integers(0, 9, size=N)
        counts[N // 3] = 3000
        L["rows"] = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        L["cols"] = np.concatenate([np.sort(rng.choice(K, size=c, replace=c > K)) for c in counts]).astype(np.int32)
        L["vals"] = (rng.standard_normal(len(L["cols"])) * 0.01).astype(np.float32)
    else:
        assert kind == "offset"
        return L, p[0]
    return L, 0


def _torch_layer(L, off):
    """L's tensors on the GPU; off > 0: rows / cols / vals start off, off + 1, off + 2 elements into larger buffers."""
    T = to_torch({k: v for k, v in L.items() if v is not None})
    for k in ("rows", "cols", "vals", "full_rows", "full_row_indices"):
        T.setdefault(k, None)
    if off:
        for i, k in enumerate(("rows", "cols", "vals")):
            o = (off + i - 1) % 3 + 1
            buf = torch.zeros(T[k].numel() + o + 4, dtype=T[k].dtype, device="cuda")
            buf[o:o + T[k].numel()].copy_(T[k])
            T[k] = buf[o:o + T[k].numel()]
            assert T[k].data_ptr() % 16
    return T


PAIRS = sorted({(K, N) for K, N, _ in SHAPES})
ONE_ROW_CASES = ([("shape", K, N, bits) for K, N in PAIRS for bits in (3, 4)] + [("shape", 512, 60, 4), ("shape", 128, 131072, 4)]
                 + [("topx", t, p) for t in (1, 33, 128) for p in ("chan0", "mixed")]
                 + [("empty_csr",), ("no_sparse",), ("long_row",), ("offset", 1), ("offset", 2), ("offset", 3)])


def _cid(c):
    return "-".join(str(v) for v in c)


_one_cache = {}


def one_row_case(case):
    if case not in _one_cache:
        _one_cache.clear()
        L, off = _edge_layer(case)
        T = _torch_layer(L, off)
        x = make_activations(L["infeatures"], 6, seed=L["infeatures"] + L["bits"])
        _one_cache[case] = (L, T, x[[0, 1, 3, 5]])  # 1e-3, 1e2, a one-entry row and an ordinary one
    return _one_cache[case]


# ---- one row, C ABI -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", [0, 1], ids=["fast", "deterministic"])
@pytest.mark.parametrize("case", ONE_ROW_CASES, ids=[_cid(c) for c in ONE_ROW_CASES])
def test_one_row_c_abi_vs_oracle(lib, case, det):
    L, T, x = one_row_case(case)
    xb, xt = bf16(x)
    bias = T.get("bias")
    with Mode(lib, det):
        got = torch.stack([fused_dt(lib, L, T, xt[i], bias=bias) for i in range(xt.shape[0])])
    check(got, L, xb, bias=L["bias"])


@pytest.mark.parametrize("det", [0, 1], ids=["fast", "deterministic"])
def test_one_row_activations_at_1e20_and_1e_minus_30(lib, det):
    K, N = 4096, 1024
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=51, nonzero_full_rows=True)
    T = to_torch(L)
    x = make_activations(K, 6, seed=51)[[4, 5, 4]]
    x[0] *= 1e20 / np.abs(x[0]).max()
    x[1] *= 1e-30 / np.abs(x[1]).max()
    x[2] = np.random.default_rng(51).standard_normal(K) * 1e20
    xb, xt = bf16(x)
    assert np.abs(xb[0]).max() > 65504 and np.abs(xb[1]).max() < 2.0 ** -25  # outside fp16: overflow, and zero
    with Mode(lib, det):
        for i in range(3):
            got = fused_dt(lib, L, T, xt[i]).cpu().numpy()
            assert np.isfinite(got).all() and np.abs(got).max() > 0
            check(got, L, xb[i:i + 1])


def test_one_row_bf16_output_is_the_rounded_fp32_output(lib):
    """Deterministic mode: y in bf16 is bit-equal to the bf16 rounding of y in fp32, for both kernels' store paths (ragged N)."""
    for K, N, bits in ((4096, 4096 + 64 + 4, 4), (512, 60, 3)):
        L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=N, nonzero_full_rows=True, bias=True)
        T = to_torch(L)
        xb, xt = bf16(make_activations(K, 6, seed=N))
        with Mode(lib, 1):
            for i in (0, 1, 5):
                y16 = fused_dt(lib, L, T, xt[i], y_dtype=torch.bfloat16, bias=T["bias"])
                y32 = fused_dt(lib, L, T, xt[i], bias=T["bias"])
                assert y16.dtype == torch.bfloat16 and torch.equal(y16, y32.bfloat16()), (K, N, i)
                check(y16, L, xb[i:i + 1], bias=L["bias"], y_dtype="bfloat16")
        with Mode(lib, 0):
            check(fused_dt(lib, L, T, xt[5], y_dtype=torch.bfloat16, bias=T["bias"]), L, xb[5:6], bias=L["bias"], y_dtype="bfloat16")


@pytest.mark.parametrize("bits", [3, 4])
def test_fp16_and_fp32_x_through_the_dtype_entry_are_the_old_entry(lib, bits):
    """sqllm_lutgemv_fused is sqllm_lutgemv_fused_dt with the fp16 / fp32 codes: the same bits in the deterministic mode."""
    K, N = 4096, 4096 + 40
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=70 + bits, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = torch.from_numpy(make_activations(K, 6, seed=70)[5]).cuda()
    with Mode(lib, 1):
        for xin, y_dtype in ((x.half(), torch.float32), (x.half(), torch.float16), (x, torch.float32), (x, torch.float16)):
            new = fused_dt(lib, L, T, xin, y_dtype, bias=T["bias"])
            old = fused_dt(lib, L, T, xin, y_dtype, bias=T["bias"], old=True)
            assert torch.equal(new, old), (xin.dtype, y_dtype)


def test_fp16_table_mode_keeps_the_exact_codebook_for_bf16(lib):
    """Under SQLLM_LUT_FP16_PAIR, bf16 x still runs the exact table: the exact-codebook bound holds element by element."""
    K, N = 4096, 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=81, nonzero_full_rows=True)
    L["lookup_table"][:, 1] += 1e-4  # centroids fp16 cannot hold exactly
    T = to_torch(L)
    xb, xt = bf16(make_activations(K, 6, seed=81))
    lib.sqllm_set_lut_mode(1)
    try:
        got = torch.stack([fused_dt(lib, L, T, xt[i]) for i in (0, 1, 5)])
    finally:
        lib.sqllm_set_lut_mode(0)
    check(got, L, xb[[0, 1, 5]])


# ---- a few rows, C ABI ----------------------------------------------------------------------------------------------------------
M_ROWS = [1, 2, 3, 7, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65, 79]
ROW_SHAPES = [(4096, 12288, 4), (4096, 12288, 3), (512, 132, 3), (512, 132, 4)]
_rows_cache = {}


def rows_layer(shape):
    if shape not in _rows_cache:
        _rows_cache.clear()
        K, N, bits = shape
        L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True, bias=True)
        xb, xt = bf16(make_activations(K, M_ROWS[-1], seed=K + bits))
        want = orc.forward_f64(L, xb, mul_init=L["bias"][None, :])
        _rows_cache[shape] = (L, to_torch(L), xb, xt, want, abs_sum(L, xb, L["bias"]))
    return _rows_cache[shape]


@pytest.mark.parametrize("shape,M", [(s, m) for s in ROW_SHAPES for m in M_ROWS],
                         ids=[f"w{s[2]}_{s[0]}x{s[1]}-M{m}" for s in ROW_SHAPES for m in M_ROWS])
def test_rows_c_abi_vs_oracle(lib, shape, M):
    L, T, xb, xt, want, S = rows_layer(shape)
    got = rows_dt(lib, L, T, xt[:M].contiguous(), bias=T["bias"]).cpu().numpy()
    assert bound_ratio(got, want[:M], S[:M]) <= 1.0
    assert rel_err(got, want[:M]) < TIGHT_TOL
    if M > 2:  # the all-zero row: exactly the bias
        assert np.array_equal(got[2], L["bias"])


@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("K,N", [(K, 132) for K in (32, 96, 160, 4128, 22016)] + [(160, N) for N in (4, 60, 64, 68, 131072)])
def test_rows_in_and_out_features_at_the_edges(lib, K, N, bits):
    L = orc.make_layer(bits, K, N, sparsity=0.01, topX=3, seed=K * 7 + N + bits, nonzero_full_rows=True)
    T = to_torch(L)
    xb, xt = bf16(make_activations(K, 9, seed=K + N))
    got = rows_dt(lib, L, T, xt).cpu().numpy()
    check(got, L, xb)
    assert np.array_equal(got[2], np.zeros(N, np.float32))  # the all-zero row: exactly zero


@pytest.mark.parametrize("case", ONE_ROW_CASES[-12:], ids=[_cid(c) for c in ONE_ROW_CASES[-12:]])
def test_rows_outlier_edge_cases(lib, case):
    L, off = _edge_layer(case)
    T = _torch_layer(L, off)
    xb, xt = bf16(make_activations(L["infeatures"], 17, seed=off + 5))
    check(rows_dt(lib, L, T, xt, bias=T["bias"]), L, xb, bias=L["bias"])


def test_rows_reproducible_and_independent_of_the_other_rows(lib):
    """Two calls give the same bits; a row's bits do not depend on M, on its position or on the other rows."""
    L, T, xb, xt, _, _ = rows_layer((4096, 12288, 4))
    other, _ = bf16(make_activations(4096, 79, seed=99))
    run = lambda xx: rows_dt(lib, L, T, torch.from_numpy(np.ascontiguousarray(xx)).cuda().bfloat16(), bias=T["bias"]).cpu().numpy()
    base = run(xb)
    assert np.array_equal(base.view(np.uint32), run(xb).view(np.uint32))
    for M in (2, 4, 5, 9, 17, 33, 64, 79):  # every row-group size
        keep = [0, 1, 2, 3, 5][:M]
        xn = other[:M].copy()
        pos = np.random.default_rng(M).permutation(M)[:len(keep)]  # the kept rows at new positions among new neighbours
        xn[pos] = xb[keep]
        y = run(xn)
        assert np.array_equal(y[pos].view(np.uint32), base[keep].view(np.uint32)), M
    bf = rows_dt(lib, L, T, xt, y_dtype=torch.bfloat16, bias=T["bias"])
    assert torch.equal(bf, torch.from_numpy(base).cuda().bfloat16())  # bf16 y: the fp32 value, rounded once
    assert np.array_equal(run(xb[2:3])[0], L["bias"])


@pytest.mark.parametrize("bits", [3, 4])
def test_rows_fp16_x_through_the_dtype_entry_is_the_old_entry(lib, bits):
    K, N = 4096, 4096 + 44
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=90 + bits, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x16 = torch.from_numpy(make_activations(K, 40, seed=90)).cuda().half()
    for y_dtype in (torch.float32, torch.float16):
        new = rows_dt(lib, L, T, x16, y_dtype, bias=T["bias"])
        old = rows_dt(lib, L, T, x16, y_dtype, bias=T["bias"], old=True)
        assert torch.equal(new, old), y_dtype


# ---- graphs and streams (through quant_cuda) -----------------------------------------------------------------------------------------
def _lay(T, bits, bias=None):
    return (T["qweight"], T["lookup_table"], bits, bias, T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])


def test_graph_capture_and_replay_with_new_inputs(qc, lib):
    K, N = 4096, 4096
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=9, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    _, x = bf16(make_activations(K, 16, seed=1))
    x2b, x2 = bf16(make_activations(K, 16, seed=2))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up on the capture stream: sizes its fused-path workspace
        qc.lutgemv_fused(x[5], *_lay(T, 3, T["bias"]))
        qc.lutgemv_rows_bf16(x, *_lay(T, 3))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with Mode(lib, 1):
        with torch.cuda.stream(s):  # the deterministic mode's workspace, sized before the capture
            qc.lutgemv_fused(x[5], *_lay(T, 3, T["bias"]))
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(g, stream=s):
            one = qc.lutgemv_fused(x[5], *_lay(T, 3, T["bias"]))
            few = qc.lutgemv_rows_bf16(x, *_lay(T, 3))
        x.copy_(x2)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(one, qc.lutgemv_fused(x2[5], *_lay(T, 3, T["bias"])))
    assert torch.equal(few, qc.lutgemv_rows_bf16(x2, *_lay(T, 3)))
    check(one, L, x2b[5:6], bias=L["bias"], y_dtype="bfloat16")
    check(few, L, x2b, y_dtype="bfloat16")


def test_three_streams_at_once(qc):
    """One-row bf16, few-row bf16 and few-row fp16 calls on three streams with no synchronisation between them."""
    Ls = [orc.make_layer(4, 4096, 4096, sparsity=0.0045, topX=10, seed=81 + i, nonzero_full_rows=True, bias=True) for i in range(3)]
    Ts = [to_torch(L) for L in Ls]
    xs = [make_activations(4096, 8, seed=81 + i) for i in range(3)]
    (xb0, xg0), (xb1, xg1) = bf16(xs[0]), bf16(xs[1])
    xg2 = torch.from_numpy(xs[2]).cuda().half()
    streams = [torch.cuda.Stream() for _ in range(3)]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    out = {}
    with torch.cuda.stream(streams[0]):
        out["one"] = [qc.lutgemv_fused(xg0[i], *_lay(Ts[0], 4, Ts[0]["bias"])) for i in range(8)]
    with torch.cuda.stream(streams[1]):
        out["rows bf16"] = [qc.lutgemv_rows_bf16(xg1, *_lay(Ts[1], 4)) for _ in range(4)]
    with torch.cuda.stream(streams[2]):
        out["rows fp16"] = qc.lutgemv_rows(xg2, *_lay(Ts[2], 4))
    torch.cuda.synchronize()
    for s in streams:
        with torch.cuda.stream(s):
            assert not qc.workspace_error()
    check(torch.stack(out["one"]), Ls[0], xb0, bias=Ls[0]["bias"], y_dtype="bfloat16")
    for y in out["rows bf16"]:
        assert torch.equal(y, out["rows bf16"][0])
    check(out["rows bf16"][0], Ls[1], xb1, y_dtype="bfloat16")
    check(out["rows fp16"], Ls[2], xs[2], y_dtype="float16")


# ---- QuantLinearLUT ----------------------------------------------------------------------------------------------------------------
SPIED = ("lutgemv_fused", "lutgemv_rows_bf16", "lutgemv_rows", "lutgemm_fused")


@pytest.fixture
def spy(qc, monkeypatch):
    calls = []
    for n in SPIED:
        real = getattr(qc, n)
        monkeypatch.setattr(qc, n, (lambda real, n: lambda *a, **kw: (calls.append((n, tuple(a[0].shape), a[0].dtype)), real(*a, **kw))[1])(real, n))
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
    R, T = QuantLinearLUT.BF16_ROWS_MAX, QuantLinearLUT.BF16_TC_MIN_ROWS
    assert 2 <= R < T
    K = N = 1024
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=12, nonzero_full_rows=True)
    m = _module(L)
    x = torch.from_numpy(make_activations(K, T, seed=12)).cuda()
    want = {(1, torch.bfloat16): "lutgemv_fused", (2, torch.bfloat16): "lutgemv_rows_bf16", (R, torch.bfloat16): "lutgemv_rows_bf16",
            (T, torch.bfloat16): "lutgemm_fused", (1, torch.float16): "lutgemv_fused", (8, torch.float16): "lutgemv_rows",
            (1, torch.float32): "lutgemv_fused", (8, torch.float32): None, (64, torch.float16): "lutgemm_fused"}
    for (M, dt), route in want.items():
        del spy[:]
        _run(m, x[:M].to(dt).reshape(1, M, K))
        assert [c[0] for c in spy] == ([route] if route else []), (M, dt, spy)
        if dt != torch.bfloat16:
            assert all(c[0] != "lutgemv_rows_bf16" for c in spy)
    del spy[:]
    for M in (1, 2, R, T):
        _run(m, x[:M].bfloat16().reshape(1, M, K), fused=False)
    assert spy == []


@pytest.mark.parametrize("bias_on", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("M", [1, 2, 63])
def test_module_output_matches_the_unfused_branch(bias_on, M):
    """dtype, shape and (within the bound) values of the use_fused = False branch: 1 row in bf16 with the bias inside the sum, more
    rows bf16 without a bias, fp32 with one (out.to(bf16) + bias)."""
    K, N = 4096, 1000
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=13, nonzero_full_rows=True, bias=True)
    m = _module(L, bias=bias_on)
    xb, xt = bf16(make_activations(K, M, seed=13))
    bias = m.bias.cpu().numpy() if bias_on else None
    x = xt.reshape(1, M, K)
    y, y_b = _run(m, x), _run(m, x, fused=False)
    want_dtype = torch.float32 if bias_on and M > 1 else torch.bfloat16
    assert y.dtype == y_b.dtype == want_dtype and y.shape == y_b.shape == (1, M, N)
    inside = M == 1
    want = orc.forward_f64(L, xb, mul_init=bias[None, :] if (bias_on and inside) else None)
    b = bias.astype(np.float64)[None, :] if (bias_on and not inside) else 0.0
    r, eta = OUT_ROUNDING["bfloat16"]
    for got in (y, y_b):
        assert bound_ratio(got[0].float().cpu().numpy(), want + b, abs_sum(L, xb, bias), want, r, eta=eta) <= 1.0


def test_misaligned_bf16_views_give_the_same_bits(lib, spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K, N = 4096, 1024
    m = _module(orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=14, nonzero_full_rows=True), bias=True)
    with Mode(lib, 1):  # one row: the deterministic summation, so that bits can be compared
        for M in (1, 2, QuantLinearLUT.BF16_ROWS_MAX):
            _, xa = bf16(make_activations(K, M, seed=14))
            want = _run(m, xa)
            for off in (1, 3, 7):
                buf = torch.zeros(M * K + 8, device="cuda", dtype=torch.bfloat16)
                xv = buf[off:off + M * K].view(M, K)
                xv.copy_(xa)
                assert xv.is_contiguous() and xv.data_ptr() % 16
                assert torch.equal(_run(m, xv), want), (M, off)
                assert torch.equal(xv, xa)
    assert {c[0] for c in spy} == {"lutgemv_fused", "lutgemv_rows_bf16"}


@pytest.mark.parametrize("M", [1, 9])
def test_stacked_qkv_group_in_bf16(spy, M):
    from squeezellm_b200.fusion import fuse_siblings
    K = 512
    Ls = [orc.make_layer(4, K, n, sparsity=0.01, topX=3, seed=20 + n, nonzero_full_rows=True) for n in (256, 128, 192)]
    block = torch.nn.Module()
    for name, L in zip(("q_proj", "k_proj", "v_proj"), Ls):
        setattr(block, name, _module(L))
    assert len(fuse_siblings(block)) == 1
    xb, xt = bf16(make_activations(K, M, seed=21))
    x = xt.reshape(1, M, K)
    outs = [block.q_proj(x), block.k_proj(x), block.v_proj(x)]
    torch.cuda.synchronize()
    assert [(c[0], c[2]) for c in spy] == [("lutgemv_fused" if M == 1 else "lutgemv_rows_bf16", torch.bfloat16)]
    for y, L in zip(outs, Ls):
        assert y.dtype == torch.bfloat16 and y.shape == (1, M, L["outfeatures"])
        check(y[0], L, xb, y_dtype="bfloat16")


def test_grad_forward_is_bit_identical_and_dx_is_bf16(lib, spy):
    K, N = 4096, 2048
    m = _module(orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=90, nonzero_full_rows=True))
    with Mode(lib, 1):
        for M in (1, 8):
            _, xt = bf16(make_activations(K, M, seed=90))
            with torch.no_grad():
                y0 = m(xt.reshape(1, M, K))
            x = xt.reshape(1, M, K).clone().requires_grad_(True)
            y = m(x)
            assert y.grad_fn is not None and torch.equal(y.detach(), y0)
            y.float().sum().backward()
            assert x.grad is not None and x.grad.dtype == torch.bfloat16 and x.grad.shape == x.shape
    assert [c[0] for c in spy] == ["lutgemv_fused"] * 2 + ["lutgemv_rows_bf16"] * 2


def test_train_codebook_forward_is_the_plain_forward(spy):
    K, N, M = 1024, 512, 8
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=4, seed=91, nonzero_full_rows=True)
    plain, trained = _module(L, bias=True), _module(L, bias=True)
    trained.train_codebook(lookup_table=True, vals=True, full_rows=True, bias=True)
    _, xt = bf16(make_activations(K, M, seed=91))
    with torch.no_grad():
        y0 = plain(xt)
    y1 = trained(xt)
    assert y1.grad_fn is not None and torch.equal(y1.detach(), y0)
    y1.float().sum().backward()
    assert trained.lookup_table.grad is not None
    assert [c[0] for c in spy] == ["lutgemv_rows_bf16"] * 2


def test_graphed_decode_step_over_a_7b_decoder_layer(lib, spy):
    """The four launches of one 7B decoder layer (q/k/v and gate/up stacked) in bf16, captured as a CUDA graph: replayed outputs
    equal the eager ones in the deterministic mode."""
    from squeezellm_b200.runtime import GraphedDecodeStep
    shapes = [(4096, 12288), (4096, 4096), (4096, 22016), (11008, 4096)]
    mods = [_module(orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=K + N, nonzero_full_rows=True)) for K, N in shapes]

    def step(x):
        qkv, gu = mods[0](x), mods[2](x)
        o = mods[1](qkv[..., :4096].contiguous())
        d = mods[3](gu[..., :11008].contiguous())
        return torch.cat([qkv.reshape(-1), o.reshape(-1), gu.reshape(-1), d.reshape(-1)])

    xs = [bf16(make_activations(4096, 6, seed=s)[5:6].reshape(1, 1, 4096))[1] for s in (1, 2)]
    with Mode(lib, 1):
        runner = GraphedDecodeStep(step, xs[0], warmup=2)
        for x in xs:
            runner.x_dev.copy_(x)
            y = runner.replay().clone()
            torch.cuda.synchronize()
            assert torch.equal(y, step(x))
    assert {c[0] for c in spy} == {"lutgemv_fused"}


def test_exchange_and_sequence_reject_bf16(qc):
    K, N = 512, 256
    T = to_torch(orc.make_layer(4, K, N, sparsity=0.01, topX=3, seed=3, nonzero_full_rows=True))
    x = torch.zeros(K, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="x must be fp16 or fp32"):
        qc.lutgemv_fused_exchange(x, *_lay(T, 4), 0, 0, 0, 0, 0, 1, 0, 1, N)
    item = _lay(T, 4) + (-1, 0, x, 1, N)
    with pytest.raises(RuntimeError, match="x_ext must be fp16"):
        qc.sequence_create([item], [], "exact")
    with pytest.raises(RuntimeError, match="x must be fp16 or fp32"):
        qc.lutgemv_rows(x.reshape(1, K).repeat(2, 1), *_lay(T, 4))
    with pytest.raises(RuntimeError, match="lutgemv_rows_bf16: x must be bf16"):
        qc.lutgemv_rows_bf16(x.reshape(1, K).repeat(2, 1).half(), *_lay(T, 4))
