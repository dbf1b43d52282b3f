"""Every QuantLinearLUT.forward route against the fp64 oracle, element by element, with the condition-aware bound of tests/util.py
(bound_ratio) next to the old rel_err, on prefill-like activations (util.make_activations: rows from 1e-3 to 1e2, massive channels,
an all-zero row, a one-entry row).

Routes (QuantLinearLUT.forward; the quant_cuda binding each call reaches, as a spy on the extension records it):
  * 1 row, fp16 / bf16 / fp32 x -> "lutgemv_fused" (bias inside the sum);  1 row with use_fused = False -> "symbols" (the
    reference's 1-row symbols onto a copy of the bias).
  * fp16 x of 2 to ROWS_MAX (63) rows -> "lutgemv_rows";  TC_MIN_ROWS (64) rows or more -> "lutgemm_fused".
  * bf16 x of 2 to BF16_ROWS_MAX (79) rows -> "lutgemv_rows_bf16";  BF16_TC_MIN_ROWS (80) rows or more -> "lutgemm_fused".
  * fp32 x of 2 to FP32_TC_MIN_ROWS - 1 (127) rows -> "symbols_batched" (the _batched symbols);  128 rows or more ->
    "lutgemm_fused_f32".
  * 2 rows or more with use_fused = False -> "symbols_batched".
Every route but the 1-row ones rounds the sum to x's dtype and adds the bias afterwards (out.to(dtype) + bias).
Also: the output dtype and shape the reference's quant.py gives, the input left unchanged, the same rows through every route,
bitwise row independence of the tensor-core kernel, three streams and a graph replay at once, and inputs that are not 16-byte
aligned."""
import numpy as np
import pytest
import torch

from test_error_bound_host import SHAPES
from test_prefill_tc_gpu import abi_call
from util import OUT_ROUNDING, REL_TOL, abs_layer, TIGHT_TOL, abs_sum, bound_ratio, load_lib, make_activations, orc, rel_err, to_torch

pytestmark = pytest.mark.gpu

SMALL_M = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129]
LARGE_M = [2048, 2049]  # fp16 and fp32 x on the 7B shapes; with fp32 x 2049 rows run csr_batched_kernel's second pass over the batch
LARGE_SHAPES = SHAPES[:4]  # 7B q/k/v stacked, o, gate/up stacked, down
# rows checked at M > 129: besides 0..128, both sides of 2016 / 2048 and the last (partial) 128-row tile
SAMPLE_ROWS = [777, 1919, 1920, 2015, 2016, 2017, 2047, 2048]
DTYPES = {"fp16": torch.float16, "fp32": torch.float32, "bf16": torch.bfloat16}
# rel_err limits kept beside the bound: the output is rounded to x's dtype, and bf16's own rounding (2^-9) is above REL_TOL
OLD_TOL = {"fp32": TIGHT_TOL, "fp16": REL_TOL, "bf16": 2.0 ** -8}
BF16_GROWTH =1.0 + 2.0 ** -8  # |bf16(v)| <= (1 + 2^-9) |v|: S of the fp16-exact rows, so grown, bounds S of their bf16 roundings


@pytest.fixture
def record(request):
    """Attach a measured number to the test's report (a --junitxml file lists it as a property)."""
    return lambda name, value: request.node.user_properties.append((name, value))


def route(M, dtype, fused):
    """The route the table above names for M rows of x in `dtype` (every layer here fits the fused launches).  The row counts are
    the table's, not QuantLinearLUT's thresholds: a changed threshold fails here until the table, and the cases it picks, follow."""
    if M == 1:
        return "lutgemv_fused" if fused else "symbols"
    if not fused:
        return "symbols_batched"
    if M >= {"fp16": 64, "bf16": 80, "fp32": 128}[dtype]:
        return "lutgemm_fused_f32" if dtype == "fp32" else "lutgemm_fused"
    if M <= {"fp16": 63, "bf16": 79}.get(dtype, 0):
        return "lutgemv_rows" if dtype == "fp16" else "lutgemv_rows_bf16"
    return "symbols_batched"


# routes whose results are the same bits on every call, whatever the alignment of x: no atomics
REPRODUCIBLE = {"lutgemv_rows", "lutgemv_rows_bf16", "lutgemm_fused", "lutgemm_fused_f32"}


def binding_route(name):
    """The route a quant_cuda binding name belongs to."""
    if name.startswith("vecquant"):
        return "symbols_batched" if name.endswith("_batched") else "symbols"
    return name


@pytest.fixture
def spy(monkeypatch):
    """The quant_cuda forward bindings QuantLinearLUT.forward calls, in order (a list of names; clear it between calls)."""
    from squeezellm_b200 import quant
    calls = []
    for n in dir(quant.quant_cuda):
        if n.startswith(("lutgemv", "lutgemm", "vecquant")):
            real = getattr(quant.quant_cuda, n)
            monkeypatch.setattr(quant.quant_cuda, n, (lambda real, n: lambda *a, **kw: (calls.append(n), real(*a, **kw))[1])(real, n))
    return calls


def taken(spy, M, dtype, fused):
    """The one route the last call reached; it must be the one the table names."""
    assert len(spy) == 1, spy
    rt = binding_route(spy[0])
    assert rt == route(M, dtype, fused), (spy[0], M, dtype, fused)
    del spy[:]
    return rt


def _cases():
    out = []
    for K, N, bits in SHAPES:
        for dtype in DTYPES:
            ms = SMALL_M + (LARGE_M if (K, N, bits) in LARGE_SHAPES and dtype != "bf16" else [])
            for M in ms:
                for fused in (True, False):
                    if not fused and route(M, dtype, True) == "symbols_batched":  # the unfused branch takes the same route
                        continue
                    for bias in (True, False):
                        out.append(pytest.param((K, N, bits), M, dtype, bias, fused,
                                                id=f"w{bits}_{K}x{N}-M{M}-{dtype}-{'bias' if bias else 'nobias'}-"
                                                   f"{'fused' if fused else 'unfused'}"))
    return out


class LayerData:
    """One layer on the GPU as two modules (with and without bias, same weight tensors), its activations and the oracle on the
    rows that the cases of this layer check."""

    def __init__(self, K, N, bits):
        from squeezellm_b200.quant import QuantLinearLUT
        self.L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=K + N + bits, nonzero_full_rows=True, bias=True)
        large = (K, N, bits) in LARGE_SHAPES
        self.x = make_activations(K, 2049 if large else SMALL_M[-1], seed=K + bits)
        self.rows = list(range(SMALL_M[-1])) + (SAMPLE_ROWS if large else [])
        self.pos = {r: i for i, r in enumerate(self.rows)}
        xr = self.x[self.rows]
        self.want = {"fp16": orc.forward_f64(self.L, xr)}
        self.S = {"fp16": abs_sum(self.L, xr)}
        xb = torch.from_numpy(self.x[:SMALL_M[-1]]).bfloat16().float().numpy()
        self.want["bf16"] = orc.forward_f64(self.L, xb)
        self.S["bf16"] = self.S["fp16"][:SMALL_M[-1]] * BF16_GROWTH
        self.want["fp32"], self.S["fp32"] = self.want["fp16"], self.S["fp16"]  # the same fp16-exact values
        T = to_torch(self.L)
        self.bias = T["bias"]
        self.modules = {}
        for has_bias in (True, False):
            self.modules[has_bias] = QuantLinearLUT.from_buffers(bits, T if has_bias else dict(T, bias=None))

    def check_rows(self, M):
        return [r for r in self.rows if r < M]


_layer_cache = {}


def layer_data(shape):
    if shape not in _layer_cache:
        _layer_cache.clear()
        torch.cuda.empty_cache()
        _layer_cache[shape] = LayerData(*shape)
    return _layer_cache[shape]


def expected(D, dtype, rows, bias, bias_inside):
    """want, S and the rounded quantity on `rows` for x of `dtype`, with or without bias."""
    idx = [D.pos[r] for r in rows]
    want, S = D.want[dtype][idx], D.S[dtype][idx]
    if not bias:
        return want, S, want
    b = D.L["bias"].astype(np.float64)[None, :]
    return want + b, S + np.abs(b), (want + b if bias_inside else want)


def run_module(m, x, fused):
    from squeezellm_b200.quant import QuantLinearLUT
    QuantLinearLUT.use_fused = fused
    try:
        y = m(x)
    finally:
        QuantLinearLUT.use_fused = True
    torch.cuda.synchronize()
    return y


def check(got, D, dtype, rows, bias, rt, record=None):
    """The bound and the old metric on got [len(rows), N] (numpy) computed by route rt from x of dtype."""
    want, S, rounded = expected(D, dtype, rows, bias, bias_inside=rt in ("lutgemv_fused", "symbols"))
    r, eta = OUT_ROUNDING[str(DTYPES[dtype]).split(".")[1]]
    ratio = bound_ratio(got, want, S, rounded, r, eta=eta)
    if record is not None:
        record("route", rt)
        record("bound_ratio", ratio)
    assert ratio <= 1.0, (rt, ratio)
    old = rel_err(got, want)
    assert old < OLD_TOL[dtype], (rt, old)
    return ratio


@pytest.mark.parametrize("shape,M,dtype,bias,fused", _cases())
def test_route_vs_oracle(record, spy, shape, M, dtype, bias, fused):
    D = layer_data(shape)
    K, N, _ = shape
    xt = torch.from_numpy(D.x[:M]).cuda().to(DTYPES[dtype]).reshape(1, M, K)
    x_before = xt.clone()
    y = run_module(D.modules[bias], xt, fused)
    rt = taken(spy, M, dtype, fused)
    assert torch.equal(xt, x_before), "forward modified its input"
    # quant.py: a 1-row input comes back in its own dtype (y.to(dtype)); a batch as out.to(dtype) + bias
    want_dtype = xt.dtype if M == 1 or not bias else torch.result_type(torch.empty(0, dtype=xt.dtype), D.bias)
    assert y.shape == (1, M, N) and y.dtype == want_dtype, (y.shape, y.dtype)
    rows = D.check_rows(M)
    got = y.reshape(M, N)[rows].float().cpu().numpy()
    check(got, D, dtype, rows, bias, rt, record)
    if M > 2:  # the all-zero row: exactly the bias, or zero
        zero = got[rows.index(2)]
        assert np.array_equal(zero, D.L["bias"] if bias else np.zeros(N, np.float32)), np.abs(zero - (D.L["bias"] if bias else 0)).max()


# ---- the same rows through every route ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [SHAPES[1], SHAPES[9]], ids=["w3_4096x4096", "w4_512x132"])
def test_same_rows_through_every_route(record, spy, shape):
    D = layer_data(shape)
    K, N, _ = shape
    M, one = 64, list(range(8))  # 64 rows as a batch; the first 8 (1e-3, 1e2, zero, one-entry rows among them) one at a time
    m = D.modules[True]
    x16 = torch.from_numpy(D.x[:M]).cuda().half()
    ratios = {}
    for fused, xin in ((True, x16), (False, x16), (True, x16.float())):
        dtype = "fp16" if xin.dtype == torch.float16 else "fp32"
        got = run_module(m, xin, fused).float().cpu().numpy()
        rt = taken(spy, M, dtype, fused)
        ratios[f"{rt}-{dtype}"] = check(got, D, dtype, list(range(M)), True, rt)
    for fused in (True, False):
        got = []
        for i in one:
            got.append(run_module(m, x16[i], fused).float().cpu().numpy())
            rt = taken(spy, 1, "fp16", fused)
        ratios[rt] = check(np.stack(got), D, "fp16", one, True, rt)
    record("bound_ratios", ratios)


# ---- tensor-core rows are independent of each other ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import ctypes
    lib = load_lib()
    lib.sqllm_lutgemm_fused.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def test_tc_row_is_independent_of_other_rows_and_of_M(lib, record):
    """A row's summation order in the tensor-core kernel depends only on its own data: its fp32 result is bit-identical whatever M
    (>= 64) is and whatever the other rows hold."""
    K, N = 4096, 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=31, nonzero_full_rows=True)
    x = make_activations(K, 200, seed=31)
    other = make_activations(K, 200, seed=32)
    fixed = [0, 1, 2, 3, 37, 63]
    late = 128  # in the second M-tile: compared where it exists
    keep = np.array(fixed + [late])
    run = lambda xx: abi_call(lib, L, torch.from_numpy(np.ascontiguousarray(xx)).cuda().half())
    base = run(x)
    variants = {f"M={M}": run(x[:M]) for M in (64, 65, 128, 129)}
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
    # fp32 output: the ratio is the accumulation error alone, not the rounding to fp16
    want = orc.forward_f64(L, x)
    ratio = bound_ratio(base, want, abs_sum(L, x))
    record("bound_ratios", {"tc fp32 out": ratio})
    assert ratio <= 1.0


# ---- several streams at once ----------------------------------------------------------------------------------------------------
def test_three_streams_and_a_graph_replay_at_once(record):
    """lutgemv_fused, lutgemm_fused and a batched call on three streams with no synchronisation between them, then a CUDA graph of
    lutgemv_fused replayed on its capture stream while eager lutgemv_fused calls run on another: the fused path's workspace is
    per (device, stream), so none of them may disturb another."""
    from squeezellm_b200.quant import quant_cuda as qc
    Ls = [orc.make_layer(4, 4096, 4096, sparsity=0.0045, topX=10, seed=41, nonzero_full_rows=True, bias=True),
          orc.make_layer(3, 4096, 12288, sparsity=0.0045, topX=10, seed=42, nonzero_full_rows=True),
          orc.make_layer(4, 11008, 4096, sparsity=0.0045, topX=10, seed=43, nonzero_full_rows=True),
          orc.make_layer(3, 4096, 4096, sparsity=0.0045, topX=10, seed=44, nonzero_full_rows=True, bias=True)]
    Ts = [to_torch(L) for L in Ls]
    args = lambda T, bits: (T["qweight"], T["lookup_table"], bits, T.get("bias"), T["rows"], T["cols"], T["vals"], T["full_rows"],
                            T["full_row_indices"])
    xs = [make_activations(4096, 4, seed=41), make_activations(4096, 128, seed=42), make_activations(11008, 9, seed=43),
          make_activations(4096, 4, seed=44)]
    xg = [torch.from_numpy(v).cuda() for v in xs]
    xg[0], xg[1], xg[3] = xg[0].half(), xg[1].half(), xg[3].half()
    gx = xg[3][1].clone()
    streams = [torch.cuda.Stream() for _ in range(5)]
    main = torch.cuda.current_stream()
    for s in streams:
        s.wait_stream(main)
    # the graph: warm up on its capture stream (allocates that stream's workspace), capture, then replay below
    sg = streams[3]
    with torch.cuda.stream(sg):
        qc.lutgemv_fused(gx, *args(Ts[3], 3))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=sg):
        gy = qc.lutgemv_fused(gx, *args(Ts[3], 3))
    sg.wait_stream(main)
    out = {}
    with torch.cuda.stream(streams[0]):
        out["gemv"] = [qc.lutgemv_fused(xg[0][i], *args(Ts[0], 4)) for i in range(4)]
    with torch.cuda.stream(streams[1]):
        out["tc"] = qc.lutgemm_fused(xg[1], *args(Ts[1], 3))
    with torch.cuda.stream(streams[2]):
        y = torch.zeros((9, 4096), device="cuda")
        qc.vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(Ts[2]["rows"], Ts[2]["cols"], Ts[2]["vals"], xg[2], Ts[2]["full_rows"],
                                                              Ts[2]["full_row_indices"], y, 4096, Ts[2]["qweight"], Ts[2]["lookup_table"])
        out["batched"] = y
    with torch.cuda.stream(sg):
        g.replay()
    with torch.cuda.stream(streams[4]):
        out["eager beside graph"] = [qc.lutgemv_fused(xg[3][i], *args(Ts[3], 3)) for i in (0, 2, 3)]
    torch.cuda.synchronize()
    for s in streams:
        with torch.cuda.stream(s):
            assert not qc.workspace_error()
    ratios = {}

    def bound(name, got, L, x, y_dtype):  # every output here is one rounding of the whole sum (bias included)
        b = L.get("bias")
        want = orc.forward_f64(L, x, mul_init=None if b is None else b[None, :])
        r, eta = OUT_ROUNDING[y_dtype]
        ratios[name] = bound_ratio(got, want, abs_sum(L, x, b), want, r, eta=eta)
        assert ratios[name] <= 1.0, (name, ratios[name])

    bound("gemv", torch.stack(out["gemv"]).float().cpu().numpy(), Ls[0], xs[0], "float16")
    bound("tc", out["tc"].float().cpu().numpy(), Ls[1], xs[1], "float16")
    bound("batched", out["batched"].cpu().numpy(), Ls[2], xs[2], "float32")
    bound("graph replay", gy.float().cpu().numpy()[None], Ls[3], xs[3][1:2], "float16")
    bound("eager beside graph", torch.stack(out["eager beside graph"]).float().cpu().numpy(), Ls[3], xs[3][[0, 2, 3]], "float16")
    record("bound_ratios", ratios)


# ---- x that is not 16-byte aligned -----------------------------------------------------------------------------------------------
MISALIGNED = [("fp16", M, off) for M in (1, 5, 64) for off in range(1, 8)] + [("fp32", M, off) for M in (1, 5, 64) for off in range(1, 4)] + \
             [("bf16", M, off) for M in (1, 5, 80) for off in range(1, 8)] + [("fp32", 128, off) for off in range(1, 4)]


@pytest.mark.parametrize("dtype,M,offset", MISALIGNED, ids=[f"{d}-M{m}-off{o}" for d, m, o in MISALIGNED])
def test_misaligned_x(record, spy, dtype, M, offset):
    """A contiguous view that starts `offset` elements into its storage computes what the aligned input computes: bit-identical
    on the routes without atomics (REPRODUCIBLE), within the bound elsewhere (their cross-CTA sums use atomics)."""
    shape = SHAPES[1]
    D = layer_data(shape)
    K, N, _ = shape
    m = D.modules[True]
    xa = torch.from_numpy(D.x[:M]).cuda().to(DTYPES[dtype])
    buf = torch.zeros(M * K + 8, device="cuda", dtype=xa.dtype)
    xv = buf[offset:offset + M * K].view(1, M, K)
    xv.copy_(xa.reshape(1, M, K))
    assert xv.is_contiguous() and xv.data_ptr() % 16
    y = run_module(m, xv, True)
    assert torch.equal(xv, xa.reshape(1, M, K))
    rt = taken(spy, M, dtype, True)
    if rt in REPRODUCIBLE:
        assert torch.equal(y, run_module(m, xa.reshape(1, M, K), True))
    got = y.reshape(M, N).float().cpu().numpy()
    check(got, D, dtype, list(range(M)), True, rt, record)


# ---- CSR columns outside [0, in_features) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,fused", [("fp32", True), ("fp16", False)], ids=["fp32-fused", "fp16-unfused"])
def test_out_of_range_csr_columns_are_ignored_on_the_batched_route(spy, dtype, fused):
    """The _batched symbols skip CSR entries whose column lies outside [0, in_features), as every fused route does: x sits at the
    start of a NaN-filled buffer, so a gather past its end would turn the output NaN (or fault at the end of an allocation)."""
    from backward_ref import dense_w_f64
    from squeezellm_b200.quant import QuantLinearLUT
    K, N, M = 1024, 512, 5
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=10, seed=77, nonzero_full_rows=True)
    L["cols"] = L["cols"].copy()
    L["cols"][0], L["cols"][-1] = K + 9, -3
    T = to_torch(L)
    m = QuantLinearLUT.from_buffers(4, T)
    x = torch.from_numpy(make_activations(K, M, seed=78)).cuda()
    buf = torch.full((M * K + 4 * K,), float("nan"), device="cuda")
    xt = buf[:M * K].view(M, K)
    xt.copy_(x)
    if dtype == "fp16":
        buf = buf.half()
        xt = buf[:M * K].view(M, K)
    y = run_module(m, xt, fused)
    taken(spy, M, dtype, fused)
    W = dense_w_f64(L)  # ignores the out-of-range entries
    x64 = xt.double().cpu().numpy()
    r, eta = OUT_ROUNDING[str(DTYPES[dtype]).split(".")[1]]
    ratio = bound_ratio(y.float().cpu().numpy(), x64 @ W, np.abs(x64) @ np.abs(dense_w_f64(abs_layer(L))), None, r, eta=eta)
    assert ratio <= 1.0, ratio
