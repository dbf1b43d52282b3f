"""Dense rows (topX), wide layers and unaligned outlier arrays on the GPU, against the fp64 oracle.

Every kernel has two dense-row branches: topX <= 32 (a lane is one (row slot, dense row) pair; rows that feed the same output channel
travel combined) and a general one (a lane per row, one word per row, the owner's list built with a shared-memory atomic).  Stacking
siblings (fusion.py) adds up their dense rows, so the general branch is what a q/k/v group with topX >= 11 per member runs.  Also here:
the finishers' path for CTAs that own more than 8 strips (wide layers), the 4-byte staging of CSR arrays that are not 16-byte aligned,
and the module's fall-back to the 12 symbols for layers the fused launch does not take.

Metric and tolerances of tests/util.py: TIGHT_TOL for fp32 outputs, REL_TOL for fp16 outputs; the fp16 pair table is checked with
fp32 y through the C ABI against the oracle on the fp16-rounded codebook."""
import ctypes

import numpy as np
import pytest
import torch

from util import Args, REL_TOL, TIGHT_TOL, late_owned_strips, load_lib, orc, rel_err, to_torch

pytestmark = pytest.mark.gpu

PATTERNS = ["distinct", "chan0", "one-strip", "edges", "mixed"]


def _fri(pattern, topX, N, rng):
    """Output channels of the dense rows.  All of them stay in [0, N) (the oracle does not bounds-check them)."""
    if pattern == "distinct":
        return rng.choice(N, size=topX, replace=False)
    if pattern == "chan0":  # what a checkpoint without dense rows loads as (llama.py:182, strict=False)
        return np.zeros(topX, dtype=np.int64)
    if pattern == "one-strip":  # every row in one strip, with duplicates: the owner lists all topX rows (128 fill its list exactly)
        lo = (N // 64) // 2 * 64
        return lo + rng.integers(0, min(64, N - lo), size=topX)
    if pattern == "edges":  # column 0 and the last column (of a ragged last strip when N % 64 != 0)
        f = rng.integers(0, N, size=topX)
        f[0::3] = 0
        f[1::3] = N - 1
        return f
    assert pattern == "mixed"  # unique channels over all strips plus a few channels that several rows feed
    nu = min((topX + 1) // 2, N)
    uniq = rng.choice(N, size=nu, replace=False)
    dup = rng.choice(uniq[:max(1, topX // 8)], size=topX - nu)
    return rng.permutation(np.concatenate([uniq, dup]))


def _layer(bits, K, N, topX, pattern, sparsity=0.01, seed=0, bias=True):
    rng = np.random.default_rng(seed + 1)
    # (make_layer draws topX distinct channels: more dense rows than channels get their values here)
    L = orc.make_layer(bits, K, N, sparsity=sparsity, topX=topX if topX <= N else 0, seed=seed, nonzero_full_rows=True, bias=bias)
    if topX > N:
        L["full_rows"] = (rng.standard_normal((K, topX)) * 0.05).astype(np.float32)
    if topX:
        fri = _fri(pattern, topX, N, rng)
        L["full_row_indices"] = fri.astype(np.int32)
        fr = L["full_rows"]
        if pattern == "chan0":  # as loaded from a checkpoint without dense rows the rows are zero; the first 16 carry values here
            fr[:, 16:] = 0.0
        # m non-zero dense rows on one channel: each scaled by 1/m, so that the channel's dense-row sum keeps the size of one row's.
        # Unscaled, 17 rows of ~1.6 each that cancel to ~0.01 leave fp32 rounding of ~5e-6 (3e-4 of the 1 % floor) whatever the kernel
        # does; and the accumulate symbols add every (CTA, row) part into the channel with its own fp32 rounding (128 rows: ~16K of them).
        m = np.bincount(fri[fr.any(axis=0)], minlength=N)[fri]
        L["full_rows"] = (fr / np.maximum(m, 1)[None, :]).astype(np.float32)
    return L


def _lut16(L):
    L16 = dict(L)
    L16["lookup_table"] = L["lookup_table"].astype(np.float16).astype(np.float32)
    return L16


def _accumulate(qc, L, T, x):
    """The reference's batch-1 hybrid symbol: y (fp32, zero) += layer(x)."""
    y = torch.zeros(L["outfeatures"], device="cuda")
    fn = getattr(qc, f"vecquant{L['bits']}matmul_spmv_hybrid_nuq_perchannel")
    fn(T["rows"], T["cols"], T["vals"], x, T["full_rows"], T["full_row_indices"], y, L["outfeatures"], T["qweight"], T["lookup_table"])
    return y


def _fused(qc, T, x):
    y = qc.lutgemv_fused(x, T["qweight"], T["lookup_table"], T["bits"], T.get("bias"), T.get("rows"), T.get("cols"), T.get("vals"),
                         T.get("full_rows"), T.get("full_row_indices"))
    torch.cuda.synchronize()
    assert not qc.workspace_error(), "a bounded in-kernel wait of the fused path gave up"
    return y


@pytest.fixture(scope="module")
def lib():
    lib = load_lib()
    yield lib
    lib.sqllm_set_lut_mode(0)


def _pair_abi(lib, T, x_half):
    """fp16 pair-table mode through the C ABI with fp32 y (no output rounding)."""
    N = T["outfeatures"]
    a = Args(bits=T["bits"], in_features=T["infeatures"], out_features=N, batch=1,
             qweight=T["qweight"].data_ptr(), lookup_table=T["lookup_table"].data_ptr())
    if T["rows"] is not None:
        a.rows, a.cols, a.vals = T["rows"].data_ptr(), T["cols"].data_ptr(), T["vals"].data_ptr()
    if T["full_rows"] is not None:
        a.full_rows, a.full_row_indices, a.topX = T["full_rows"].data_ptr(), T["full_row_indices"].data_ptr(), T["full_rows"].shape[1]
    nbytes = lib.sqllm_workspace_bytes(T["bits"], T["infeatures"], N, a.topX)
    assert nbytes > 0
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    y = torch.empty(N, dtype=torch.float32, device="cuda")
    bias = T.get("bias")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib.sqllm_set_lut_mode(1)
    try:
        rc = lib.sqllm_lutgemv_fused(ctypes.byref(a), ctypes.c_void_p(x_half.data_ptr()), 1, ctypes.c_void_p(y.data_ptr()), 0,
                                     ctypes.c_void_p(bias.data_ptr() if bias is not None else 0), ctypes.c_void_p(ws.data_ptr()),
                                     ctypes.c_size_t(nbytes), st)
    finally:
        lib.sqllm_set_lut_mode(0)
    assert rc == 0, lib.sqllm_last_error()
    torch.cuda.synchronize()
    assert lib.sqllm_workspace_error(ctypes.c_void_p(ws.data_ptr()), st) == 0
    return y.cpu().numpy()


def _every_mode(lib, L, pair_table=True, accumulate=True):
    """Accumulate symbol, fused (fp32 x, fp16 x, fp16 pair table, deterministic) against the oracle."""
    from squeezellm_b200.quant import quant_cuda as qc
    K = L["infeatures"]
    T = to_torch(L)
    x = orc.make_vec(K, seed=7)  # fp16-representable
    xf = torch.from_numpy(x).cuda().reshape(-1)
    want = orc.forward_f64(L, x, mul_init=L["bias"][None, :])
    if accumulate:
        wacc = orc.forward_f64(L, x)
        assert rel_err(_accumulate(qc, L, T, xf).cpu().numpy(), wacc) < TIGHT_TOL, "accumulate symbol"
    assert rel_err(_fused(qc, T, xf).cpu().numpy(), want) < TIGHT_TOL, "fused, fp32 x"
    yh = _fused(qc, T, xf.half())
    assert yh.dtype == torch.float16 and rel_err(yh.float().cpu().numpy(), want) < REL_TOL, "fused, fp16 x"
    if pair_table:
        # layers narrower than one strip keep the exact codebook in the fp16 table mode
        want16 = orc.forward_f64(_lut16(L), x, mul_init=L["bias"][None, :]) if L["outfeatures"] >= 64 else want
        assert rel_err(_pair_abi(lib, T, xf.half()), want16) < TIGHT_TOL, "fused, fp16 pair table"
    qc.set_deterministic(True)
    try:
        y1, y2 = _fused(qc, T, xf), _fused(qc, T, xf)
    finally:
        qc.set_deterministic(False)
    assert torch.equal(y1, y2), "the deterministic mode must be bit-reproducible"
    assert rel_err(y1.cpu().numpy(), want) < TIGHT_TOL, "fused, deterministic"


# ---------------------------------------------------------------------------------------------------------------------------------
# A. topX across both branches of every dense-row site
TOPX = [1, 16, 17, 31, 32, 33, 64, 100, 128]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("topx", TOPX)
def test_dense_rows_every_mode(lib, topx, pattern):
    """K = 1024, N = 1000 (15 strips and a ragged 40-column one); w4 and w3."""
    for bits in (4, 3):
        _every_mode(lib, _layer(bits, 1024, 1000, topx, pattern, seed=topx * 10 + bits))


@pytest.mark.parametrize("pattern", ["chan0", "one-strip", "edges", "mixed"])
@pytest.mark.parametrize("topx", [1, 17, 33, 128])
def test_dense_rows_narrow_layer_every_mode(lib, topx, pattern):
    """N = 60 < 64: one ragged strip in every mode; in the deterministic mode the round-1 kernel's hybrid_totals (tp <= 16 split)."""
    _every_mode(lib, _layer(4, 512, 60, topx, pattern, sparsity=0.02, seed=topx + 500))


@pytest.mark.parametrize("topx", [129, 256])
def test_dense_rows_accumulate_symbols_beyond_the_fused_limit(topx):
    """The 12 symbols have no topX limit of their own (v2, N < 64 included)."""
    from squeezellm_b200.quant import quant_cuda as qc
    for bits, K, N, pattern in ((4, 1024, 1000, "mixed"), (3, 512, 1000, "one-strip"), (4, 512, 60, "mixed")):
        L = _layer(bits, K, N, topx, pattern, seed=topx + N)
        x = orc.make_vec(K, seed=3)
        y = _accumulate(qc, L, to_torch(L), torch.from_numpy(x).cuda().reshape(-1))
        assert rel_err(y.cpu().numpy(), orc.forward_f64(L, x)) < TIGHT_TOL


@pytest.mark.parametrize("B", [3, 13])
@pytest.mark.parametrize("topx", [1, 17, 33, 128, 129, 256])
def test_dense_rows_batched(topx, B):
    """The batched symbols (dense_rows_batched_kernel takes up to 256 rows); B = 13 has a partial second batch tile."""
    from squeezellm_b200.quant import quant_cuda as qc
    for bits, pattern in ((4, "mixed"), (3, "chan0"), (4, "one-strip")):
        K, N = 512, 1000
        L = _layer(bits, K, N, topx, pattern, seed=topx * 3 + B + bits)
        T = to_torch(L)
        x = orc.make_vec(K, batch=B, seed=B)
        y = torch.zeros((B, N), device="cuda")
        fn = getattr(qc, f"vecquant{bits}matmul_spmv_hybrid_nuq_perchannel_batched")
        fn(T["rows"], T["cols"], T["vals"], torch.from_numpy(x).cuda(), T["full_rows"], T["full_row_indices"], y, N, T["qweight"], T["lookup_table"])
        assert rel_err(y.cpu().numpy(), orc.forward_f64(L, x)) < TIGHT_TOL, f"w{bits} {pattern}"


def test_dense_row_limits_fail_with_their_message():
    from squeezellm_b200.quant import quant_cuda as qc
    lim = qc.fused_limits()
    assert lim["max_topx"] == 128 and lim["max_out_features"] == 262144
    L = _layer(4, 512, 256, 129, "mixed", seed=1)
    T = to_torch(L)
    x = torch.from_numpy(orc.make_vec(512, seed=1)).cuda().reshape(-1)
    with pytest.raises(RuntimeError, match="fused path supports topX <= 128"):
        _fused(qc, T, x)
    item = (T["qweight"], T["lookup_table"], 4, None, T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"],
            -1, 0, x.half(), 1, 256)
    with pytest.raises(RuntimeError, match="topX <= 128"):
        qc.sequence_create([item], [], "exact")
    L = _layer(4, 512, 256, 257, "mixed", seed=2)
    T = to_torch(L)
    y = torch.zeros((3, 256), device="cuda")
    with pytest.raises(RuntimeError, match="batched path supports topX <= 256"):
        qc.vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(T["rows"], T["cols"], T["vals"], torch.zeros((3, 512), device="cuda"),
                                                              T["full_rows"], T["full_row_indices"], y, 256, T["qweight"], T["lookup_table"])


@pytest.mark.parametrize("topx", [33, 64])
def test_dense_rows_llama_qkv_shape(lib, topx):
    """LLaMA-7B q/k/v stacked (4096 x 12288) with as many dense rows as three stacked members of topX 11 / 22 carry."""
    L = _layer(4, 4096, 12288, topx, "mixed", sparsity=0.0045, seed=topx)
    _every_mode(lib, L)


# ---------------------------------------------------------------------------------------------------------------------------------
# B. QuantLinearLUT falls back to the 12 symbols for layers the fused launch does not take
def _module(L):
    from squeezellm_b200.quant import QuantLinearLUT
    sparse = L.get("rows") is not None
    topx = int(L["full_rows"].shape[1]) if L.get("full_rows") is not None else 0
    m = QuantLinearLUT(L["bits"], L["infeatures"], L["outfeatures"], L.get("bias") is not None, include_sparse=sparse,
                       numvals=len(L["vals"]) if sparse else 0, topX=topx)
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray) and k in sd}, strict=False)
    return m.cuda()


@pytest.mark.parametrize("K,N,topx", [(64, 262208, 4), (512, 1000, 129)], ids=["out262208", "topx129"])
def test_module_forward_beyond_the_fused_limits(K, N, topx):
    L = _layer(4, K, N, topx, "mixed", sparsity=0.002, seed=N, bias=False)
    m = _module(L)
    x = orc.make_vec(K, seed=9)
    y = m(torch.from_numpy(x).cuda().half().reshape(1, 1, K))
    torch.cuda.synchronize()
    assert y.shape == (1, 1, N) and y.dtype == torch.float16
    assert rel_err(y.float().cpu().numpy(), orc.forward_f64(L, x)) < REL_TOL


def test_decode_sequence_rejects_what_the_fused_launch_does_not_take():
    from squeezellm_b200.runtime import DecodeSequence
    for K, N, topx, msg in ((512, 256, 129, "topX <= 128"), (64, 262208, 4, "out_features=262208 exceeds 262144")):
        m = _module(_layer(4, K, N, topx, "mixed", sparsity=0.002, seed=5, bias=False))
        seq = DecodeSequence(K, "cuda")
        seq.matvec(m, seq.input)
        with pytest.raises(RuntimeError, match=msg):
            seq.compile(outputs=[])


# ---------------------------------------------------------------------------------------------------------------------------------
# C. Wide layers: CTAs that own more than 8 strips
@pytest.mark.parametrize("bits,K,N", [(4, 128, 131072), (3, 256, 262144)], ids=["w4-128x131072", "w3-256x262144"])
def test_wide_layer_dense_rows_in_late_owned_strips(lib, bits, K, N):
    from squeezellm_b200.quant import quant_cuda as qc
    late = late_owned_strips(bits, K, N, qc.sm_count())
    assert len(late) > 0, "no CTA owns more than 8 strips: the shape no longer covers that branch"
    rng = np.random.default_rng(N)
    topx = 128
    L = orc.make_layer(bits, K, N, sparsity=0.001, topX=topx, seed=bits, nonzero_full_rows=True, bias=True)
    f = rng.choice(late, size=100) * 64 + rng.integers(0, 64, size=100)  # late-owned strips, some of them several times
    f = np.concatenate([f, f[:12], [0, N - 1], rng.integers(0, N, size=topx - 114)])
    L["full_row_indices"] = rng.permutation(f).astype(np.int32)
    _every_mode(lib, L)


# ---------------------------------------------------------------------------------------------------------------------------------
# D. CSR arrays that are not 16-byte aligned (staged with 4-byte copies on another chunk grid)
def _csr_with_long_row(K, N, long_len, rng):
    counts = rng.integers(0, 9, size=N)
    counts[N // 3] = long_len  # longer than a staging chunk (v2: 256, round 1: 1024 elements)
    rows = np.zeros(N + 1, dtype=np.int32)
    rows[1:] = np.cumsum(counts)
    cols = np.concatenate([np.sort(rng.choice(K, size=c, replace=False)) for c in counts]).astype(np.int32)
    vals = (rng.standard_normal(len(cols)) * 0.1).astype(np.float32)
    return rows, cols, vals


def _shifted(t, off):
    """A contiguous view of t that starts `off` elements into a larger buffer (16-byte aligned only when off % 4 == 0)."""
    buf = torch.zeros(t.numel() + off + 4, dtype=t.dtype, device=t.device)
    v = buf[off:off + t.numel()]
    v.copy_(t)
    return v


@pytest.mark.parametrize("N", [1000, 60], ids=["v2", "narrow"])
def test_unaligned_outlier_arrays(lib, N):
    from squeezellm_b200.quant import quant_cuda as qc
    bits, K, topx = 4, 2048, 10
    rng = np.random.default_rng(N)
    L = orc.make_layer(bits, K, N, topX=topx, seed=N, nonzero_full_rows=True, bias=True)
    L["rows"], L["cols"], L["vals"] = _csr_with_long_row(K, N, 1500, rng)
    T = to_torch(L)
    x = orc.make_vec(K, seed=4)
    xf = torch.from_numpy(x).cuda().reshape(-1)
    want, wacc = orc.forward_f64(L, x, mul_init=L["bias"][None, :]), orc.forward_f64(L, x)
    aligned = {"acc": _accumulate(qc, L, T, xf).cpu().numpy(), "fused": _fused(qc, T, xf).cpu().numpy()}
    for off_r, off_c, off_v in ((1, 2, 3), (2, 3, 1), (3, 1, 2)):
        U = dict(T)
        U["rows"], U["cols"], U["vals"] = _shifted(T["rows"], off_r), _shifted(T["cols"], off_c), _shifted(T["vals"], off_v)
        assert U["cols"].data_ptr() % 16 and U["vals"].data_ptr() % 16
        ya = _accumulate(qc, L, U, xf).cpu().numpy()
        yf = _fused(qc, U, xf).cpu().numpy()
        assert rel_err(ya, wacc) < TIGHT_TOL and rel_err(ya, aligned["acc"]) < TIGHT_TOL, "accumulate symbol"
        assert rel_err(yf, want) < TIGHT_TOL and rel_err(yf, aligned["fused"]) < TIGHT_TOL, "fused"
        qc.set_deterministic(True)
        try:
            yd = _fused(qc, U, xf).cpu().numpy()
        finally:
            qc.set_deterministic(False)
        assert rel_err(yd, want) < TIGHT_TOL, "fused, deterministic"
        if N >= 64:
            y16 = _pair_abi(lib, U, xf.half())
            assert rel_err(y16, orc.forward_f64(_lut16(L), x, mul_init=L["bias"][None, :])) < TIGHT_TOL, "fused, fp16 pair table"
