"""The tensor-core LUT-GEMM (`sqllm_lutgemm_fused`, `quant_cuda.lutgemm_fused`, csrc/lutgemm_tc.cuh) that runs fp16 inputs of
QuantLinearLUT.TC_MIN_ROWS or more rows: every parity shape and a range of row counts against the fp64 oracle, numerics stress
(tiny and huge weights, outliers far above the codebook, many and duplicate dense rows, unsorted CSR rows, a partial last
K-chunk), the reference kernels' stored outputs, determinism, CUDA-graph replay and the module routing."""
import ctypes
import os

import numpy as np
import pytest
import torch

from test_gpu_parity import BATCHED_SHAPES, IDS, SHAPES, batched_id, batched_inputs, ref_comparable
from util import GOLDEN, Args, REL_TOL, TIGHT_TOL, load_lib, orc, quant_layer, rel_err, sample_idx, to_torch

pytestmark = pytest.mark.gpu

M_MAX = 200
ORACLE_ROWS = [0, 1, 7, 16, 33, 63, 64, 65, 100, 127, 128, 140, 160, 199]  # both M-tiles of every M below, and every tail


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    lib.sqllm_lutgemm_fused.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def abi_call(lib, L, x16, y_half=False, bias=None):
    """sqllm_lutgemm_fused on the layer dict L (numpy) and fp16 x [M, K] (torch, cuda) -> y [M, N] (fp32 unless y_half)."""
    T = to_torch(L)
    M, N = x16.shape[0], L["outfeatures"]
    y = torch.empty((M, N), device="cuda", dtype=torch.float16 if y_half else torch.float32)
    a = Args(bits=L["bits"], in_features=L["infeatures"], out_features=N, batch=M,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T.get("rows") is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T.get("full_rows") is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    b = None if bias is None else torch.from_numpy(bias).cuda()
    rc = lib.sqllm_lutgemm_fused(ctypes.byref(a), x16.data_ptr(), y.data_ptr(), int(y_half), None if b is None else b.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    return y.float().cpu().numpy()


def check_rows(got, L, x, rows, tol, mul_init=None):
    """got [M, N] against the oracle on the given rows (rows are independent, so only those rows are computed)."""
    want = orc.forward_f64(L, x[rows], mul_init=mul_init)
    e = rel_err(got[rows], want)
    assert e < tol, e
    return want


_cache = {}


def parity_case(shape):
    """Layer, M_MAX fp16-exact rows of x and the oracle on ORACLE_ROWS, shared by the row counts of one shape."""
    if shape not in _cache:
        _cache.clear()
        bits, K, N, sp, topx, nz, skew = shape
        L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=K + 3 * N + bits, skew=skew, nonzero_full_rows=nz)
        if topx and sp == 0:
            L["full_rows"] = L["full_row_indices"] = None
        x = orc.make_vec(K, batch=M_MAX, seed=K + N)
        _cache[shape] = (L, x, orc.forward_f64(L, x[ORACLE_ROWS]))
    return _cache[shape]


@pytest.mark.parametrize("M", [1, 17, 64, 129, 200])
@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_c_abi_vs_oracle(lib, shape, M):
    L, x, want = parity_case(shape)
    got = abi_call(lib, L, torch.from_numpy(x[:M]).cuda().half())
    sel = [i for i, r in enumerate(ORACLE_ROWS) if r < M]
    e = rel_err(got[[ORACLE_ROWS[i] for i in sel]], want[sel])
    assert e < TIGHT_TOL, e


@pytest.mark.parametrize("shape", [(4, 4096, 12288, 0.0045, 10, True, True), (4, 4096, 22016, 0.0045, 10, True, False),
                                   (4, 11008, 4096, 0.0045, 10, True, False)], ids=["qkv", "gate_up", "down"])
def test_c_abi_vs_oracle_2048_rows(lib, shape):
    """A 2048-token prefill on the 7B shapes: all columns of the first and last M-tile's edge rows and a fixed spread of rows."""
    bits, K, N, sp, topx, nz, skew = shape
    L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=7, skew=skew, nonzero_full_rows=nz)
    M = 2048
    x = orc.make_vec(K, batch=M, seed=11)
    bias = np.random.default_rng(3).standard_normal(N).astype(np.float32)
    got = abi_call(lib, L, torch.from_numpy(x).cuda().half(), bias=bias)
    rows = sorted(set([0, 1, 63, 64, 127, 128, 1023, 1919, 1920, 2046, 2047] + list(range(5, M, 397))))
    check_rows(got, L, x, rows, TIGHT_TOL, mul_init=bias[None, :])


# ---- numerics stress ----------------------------------------------------------------------------------------------------------
def _stress_x(K, M=70, seed=0):
    return orc.make_vec(K, batch=M, seed=seed)


def _all_rows(lib, L, x, tol=TIGHT_TOL):
    got = abi_call(lib, L, torch.from_numpy(x).cuda().half())
    want = orc.forward_f64(L, x)
    assert rel_err(got, want) < tol, rel_err(got, want)
    return got, want


def test_tiny_and_large_centroids_side_by_side(lib):
    """Channels with centroids around 1e-6 next to channels around 1e-1: each group within TIGHT_TOL of its own magnitude."""
    L = orc.make_layer(4, 512, 256, sparsity=0.01, topX=4, seed=1, nonzero_full_rows=True)
    L["lookup_table"][0::2] *= 5e-5
    L["lookup_table"][1::2] *= 5.0
    tiny = np.arange(0, 256, 2)
    tiny = tiny[~np.isin(tiny, L["full_row_indices"])]
    hit = np.repeat(np.arange(256), np.diff(L["rows"]))
    L["vals"][np.isin(hit, tiny)] *= 5e-5  # the outliers of the tiny channels are tiny too
    x = _stress_x(512)
    got, want = _all_rows(lib, L, x)
    assert rel_err(got[:, tiny], want[:, tiny]) < TIGHT_TOL


def test_outlier_a_million_times_the_codebook(lib):
    L = orc.make_layer(3, 1024, 192, sparsity=0.005, seed=2)
    c = 37
    e = L["rows"][c]
    assert L["rows"][c + 1] > e
    L["vals"][e] = 1e6 * np.abs(L["lookup_table"][c]).max()
    x = _stress_x(1024)
    got, want = _all_rows(lib, L, x)
    others = np.arange(192) != c
    assert rel_err(got[:, others], want[:, others]) < TIGHT_TOL
    assert rel_err(got[:, c], want[:, c]) < TIGHT_TOL


def test_all_128_dense_rows_on_channel_0(lib):
    L = orc.make_layer(4, 1024, 256, sparsity=0.005, topX=128, seed=3, nonzero_full_rows=True)
    L["full_row_indices"][:] = 0
    L["full_rows"] /= 128.0  # one channel sums all of them: keep its magnitude that of the others
    x = _stress_x(1024)
    got, want = _all_rows(lib, L, x)
    assert rel_err(got[:, 0], want[:, 0]) < TIGHT_TOL


def test_topx_300_with_duplicates_and_ignored_indices(lib):
    """More dense rows than any other path takes; some channels get several; indices outside [0, N) are ignored."""
    K, N = 512, 384
    L = orc.make_layer(4, K, N, sparsity=0.01, topX=300, seed=4, nonzero_full_rows=True)
    rng = np.random.default_rng(4)
    fri = rng.integers(0, N, size=300).astype(np.int32)
    fri[:20] = 5
    L["full_rows"][:, :20] /= 20.0
    fri[290], fri[291], fri[292] = -1, N, N + 1000
    L["full_row_indices"] = fri
    x = _stress_x(K)
    got = abi_call(lib, L, torch.from_numpy(x).cuda().half())
    keep = (fri >= 0) & (fri < N)
    L2 = dict(L, full_rows=np.ascontiguousarray(L["full_rows"][:, keep]), full_row_indices=np.ascontiguousarray(fri[keep]))
    want = orc.forward_f64(L2, x)
    assert rel_err(got, want) < TIGHT_TOL


def test_unsorted_csr_rows(lib):
    """Shuffled column indices within each CSR row: same result as the sorted rows and the oracle."""
    L = orc.make_layer(4, 2048, 320, sparsity=0.02, seed=5, skew=True)
    rng = np.random.default_rng(5)
    U = dict(L, cols=L["cols"].copy(), vals=L["vals"].copy())
    for c in range(320):
        e0, e1 = L["rows"][c], L["rows"][c + 1]
        perm = rng.permutation(e1 - e0) + e0
        U["cols"][e0:e1], U["vals"][e0:e1] = L["cols"][perm], L["vals"][perm]
    assert not np.array_equal(U["cols"], L["cols"])
    x = _stress_x(2048)
    xt = torch.from_numpy(x).cuda().half()
    got_u, got_s = abi_call(lib, U, xt), abi_call(lib, L, xt)
    want = orc.forward_f64(L, x)
    assert rel_err(got_u, want) < TIGHT_TOL
    assert rel_err(got_u, got_s) < TIGHT_TOL


@pytest.mark.parametrize("bits,K,N", [(4, 160, 200), (3, 96, 60), (4, 4128, 136)])
def test_partial_last_k_chunk_and_empty_csr(lib, bits, K, N):
    """in_features a multiple of 32 but not of 64, a CSR with no entries, odd and ragged widths."""
    L = orc.make_layer(bits, K, N, sparsity=0.0, topX=3, seed=K, nonzero_full_rows=True)
    L["rows"] = np.zeros(N + 1, dtype=np.int32)
    L["cols"] = np.zeros(0, dtype=np.int32)
    L["vals"] = np.zeros(0, dtype=np.float32)
    _all_rows(lib, L, _stress_x(K, M=131))


# ---- through quant_cuda ------------------------------------------------------------------------------------------------------
def test_module_fp16_output_vs_oracle_and_bit_identical(qc):
    K, N, M = 4096, 4096, 100
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=8, nonzero_full_rows=True, bias=True)
    T = to_torch(L)
    x = orc.make_vec(K, batch=M, seed=8)
    xt = torch.from_numpy(x).cuda().half()
    args = (xt, T["qweight"], T["lookup_table"], 4, T["bias"], T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])
    y1, y2 = qc.lutgemm_fused(*args), qc.lutgemm_fused(*args)
    torch.cuda.synchronize()
    assert y1.dtype == torch.float16 and y1.shape == (M, N)
    assert torch.equal(y1, y2)
    want = orc.forward_f64(L, x, mul_init=L["bias"][None, :])
    assert rel_err(y1.float().cpu().numpy(), want) < REL_TOL


@pytest.mark.parametrize("batch", [16, 64])
@pytest.mark.parametrize("shape", [s for s in BATCHED_SHAPES if ref_comparable(s)], ids=batched_id)
def test_module_vs_reference_kernels(qc, shape, batch):
    """The reference's own batched kernels on the same inputs (golden outputs); x is fp16-exact there."""
    g = np.load(os.path.join(GOLDEN, "reference_outputs.npz"))
    key = f"b{batch}__{batched_id(shape)}"
    L, x = batched_inputs(shape, batch)
    T = to_torch(L)
    y = qc.lutgemm_fused(torch.from_numpy(x).cuda().half(), T["qweight"], T["lookup_table"], shape[0], None,
                         T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])
    got = y.float().cpu().numpy().reshape(-1)
    assert rel_err(got[sample_idx(got.size)], g[key], b_absmax=float(g[key + "__absmax"])) < REL_TOL


def test_graph_capture_and_replay_with_new_inputs(qc):
    K, N, M = 4096, 4096, 256
    L = orc.make_layer(3, K, N, sparsity=0.0045, topX=10, seed=9, nonzero_full_rows=True)
    T = to_torch(L)
    x = torch.from_numpy(orc.make_vec(K, batch=M, seed=1)).cuda().half()
    x2 = torch.from_numpy(orc.make_vec(K, batch=M, seed=2)).cuda().half()
    args = lambda xx: (xx, T["qweight"], T["lookup_table"], 3, None, T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        qc.lutgemm_fused(*args(x))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = qc.lutgemm_fused(*args(x))
    x.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, qc.lutgemm_fused(*args(x2)))


# ---- QuantLinearLUT routing ---------------------------------------------------------------------------------------------------
def _module(L):
    return quant_layer(L, bias=None).cuda()


@pytest.fixture
def spy(qc, monkeypatch):
    calls = []
    real = qc.lutgemm_fused

    def wrapped(*a, **kw):
        calls.append(a[0].shape)
        return real(*a, **kw)
    monkeypatch.setattr(qc, "lutgemm_fused", wrapped)
    return calls


def test_module_routing(spy):
    from squeezellm_b200.quant import QuantLinearLUT
    K = N = 4096
    L = orc.make_layer(4, K, N, sparsity=0.0045, topX=10, seed=12, nonzero_full_rows=True)
    m = _module(L)
    x = orc.make_vec(K, batch=2048, seed=12)
    y = m(torch.from_numpy(x).cuda().half().reshape(1, 2048, K))
    assert spy == [(2048, K)]
    assert y.shape == (1, 2048, N) and y.dtype == torch.float16
    rows = [0, 1, 127, 128, 1000, 2047]
    assert rel_err(y[0].float().cpu().numpy()[rows], orc.forward_f64(L, x[rows])) < REL_TOL
    few = QuantLinearLUT.TC_MIN_ROWS - 1
    xs = torch.from_numpy(x[:few]).cuda()
    for xin in (xs.half(), torch.from_numpy(x[:64]).cuda(), torch.from_numpy(x[:64]).cuda().bfloat16()):
        m(xin.reshape(1, -1, K))
    QuantLinearLUT.use_fused = False
    try:
        m(torch.from_numpy(x[:64]).cuda().half())
    finally:
        QuantLinearLUT.use_fused = True
    assert spy == [(2048, K)]


def test_sibling_group_members_get_their_slices(spy):
    from squeezellm_b200.fusion import fuse_siblings
    from squeezellm_b200.quant import QuantLinearLUT
    K, M = 512, QuantLinearLUT.TC_MIN_ROWS
    Ls = [orc.make_layer(4, K, n, sparsity=0.01, topX=3, seed=20 + n, nonzero_full_rows=True) for n in (256, 128, 192)]
    block = torch.nn.Module()
    for name, L, n in zip(("q_proj", "k_proj", "v_proj"), Ls, (256, 128, 192)):
        setattr(block, name, _module(L))
    assert len(fuse_siblings(block)) == 1
    x = orc.make_vec(K, batch=M, seed=21)
    xt = torch.from_numpy(x).cuda().half().reshape(1, M, K)
    outs = [block.q_proj(xt), block.k_proj(xt), block.v_proj(xt)]
    assert spy == [(M, K)]
    for y, L in zip(outs, Ls):
        assert rel_err(y[0].float().cpu().numpy(), orc.forward_f64(L, x)) < REL_TOL
