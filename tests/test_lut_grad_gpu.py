"""Codebook training on the GPU (`sqllm_lut_grad`, `quant_cuda.lut_grad`, csrc/lut_grad.cuh and lut_grad_tc.cuh, and
QuantLinearLUT.train_codebook): the gradients of the codebook, the CSR values and the dense rows against the fp64 truth
(tests/lut_grad_ref.py) per element, at every route-test shape and row counts on both sides of every chunk boundary, in every
dtype pair on both kernels; outlier and dense-row patterns; in_features and out_features at the edges of the tiles and slabs;
bitwise reproducibility, CUDA-graph replay and several streams; and the module level: autograd of all four tensors, dx unchanged
by codebook training, a teacher-student run, and in-place modification between forward and backward.

The bound is that of the forward kernels (tests/util.py, bound_ratio): |got - want| <= e S with e = 2^-20 and S the same bucketing
applied to |x|^T |dy|; the outputs are fp32, so r = eta = 0.  Every output is a sum of exact (tensor cores) or once-rounded (CUDA
cores) products, added in fp32 in chunks of 64 (32) rows, then over the chunks, then over the 32-input groups of a bin, then over
the S CTAs of a cluster: the argument of tests/util.py for the forward's fp32 sums applies unchanged.

x and dy hold values exact in fp16, bf16 and fp32 alike (bf16(fp16(v)): below 2^-14 fp16's spacing 2^-24 is at least bf16's, above
it bf16's 8 significant bits fit fp16's 11), so one truth serves every dtype pair."""
import numpy as np
import pytest
import torch

from lut_grad_ref import dense_w_torch, lut_grad_f64
from test_error_bound_host import SHAPES
from util import bound_ratio, make_activations, orc, quant_layer, to_torch

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
PAIRS = [(F16, F16), (BF16, BF16), (F32, F32), (F16, F32)]
M_ALL = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129]
SEVEN_B = {(4096, 12288, 4), (4096, 4096, 3), (4096, 22016, 4), (11008, 4096, 3)}
KEYS = ("lookup_table", "vals", "full_rows")


def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def paths(xt, dt):
    """The kernels that take this dtype pair: tensor cores for fp16/fp16 and bf16/bf16, CUDA cores for all."""
    return ("tc", "cuda") if xt == dt and xt != F32 else ("cuda",)


def exact_rows(n, M, seed):
    """make_activations rows (1e-3 .. 1e2 scales, massive channels, row 2 all zero, row 3 one non-zero) rounded to bf16(fp16(v)):
    exact in all three dtypes.  fp32 cuda tensor."""
    a = torch.from_numpy(make_activations(n, M, seed=seed)) if n >= 16 else \
        torch.from_numpy(np.random.default_rng(seed).standard_normal((M, n)) * (10.0 ** np.linspace(-3, 2, M))[:, None])
    return a.cuda().half().bfloat16().float()


def call(L, T, x, dy, path="auto", want=KEYS):
    """quant_cuda.lut_grad on layer L (T: its torch tensors) -> {key: tensor} for the keys the layer has and `want` lists."""
    has = {"lookup_table": True, "vals": T.get("rows") is not None, "full_rows": T.get("full_rows") is not None}
    w = {k: k in want and has[k] for k in KEYS}
    out = qc().lut_grad(x, dy, T["qweight"], T["lookup_table"], L["bits"], T.get("rows"), T.get("cols"), T.get("vals"),
                        T.get("full_rows"), T.get("full_row_indices"), want_lut=w["lookup_table"], want_vals=w["vals"],
                        want_full_rows=w["full_rows"], path=path)
    return {k: o for k, o in zip(KEYS, out) if w[k]}


def check(got, truth, what=""):
    want, S = truth
    for k, v in got.items():
        ratio = bound_ratio(v.double().cpu().numpy(), want[k], S[k])
        assert ratio <= 1.0, (what, k, ratio)


def _layer(K, N, bits, seed, topX=10, sparsity=0.0045):
    return orc.make_layer(bits, K, N, sparsity=sparsity, topX=topX, seed=seed, nonzero_full_rows=topX > 0)


KN = sorted({(k, n) for k, n, _ in SHAPES})
ALL_SHAPES = [(k, n, b) for k, n in KN for b in (3, 4)]


# ---- every route-test shape, every row count, every dtype pair, both kernels -------------------------------------------------
@pytest.mark.parametrize("K,N,bits", ALL_SHAPES, ids=[f"w{b}_{k}x{n}" for k, n, b in ALL_SHAPES])
def test_per_element_all_rows(K, N, bits):
    L = _layer(K, N, bits, seed=K + N + bits)
    T = to_torch(L)
    Mmax = 2048 if (K, N) in {(k, n) for k, n, _ in SEVEN_B} else max(M_ALL)
    x, dy = exact_rows(K, Mmax, seed=K), exact_rows(N, Mmax, seed=N + 1)
    for M in M_ALL + ([2048] if Mmax == 2048 else []):
        truth = lut_grad_f64(L, x[:M], dy[:M], device="cuda")
        for xt, dt in PAIRS:
            xm, dm = x[:M].to(xt).contiguous(), dy[:M].to(dt).contiguous()
            got = {}
            for path in paths(xt, dt):
                got[path] = call(L, T, xm, dm, path=path)
                check(got[path], truth, (M, xt, dt, path))
            auto = "tc" if xt == dt and xt != F32 and M >= 8 else "cuda"  # SQLLM_LUT_GRAD_TC_MIN_ROWS = 8
            a = call(L, T, xm, dm)
            assert all(torch.equal(a[k], got[auto][k]) for k in a)


# ---- outliers and dense rows -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("topX", [1, 33, 128, 300])
@pytest.mark.parametrize("bits", [3, 4])
def test_dense_rows(bits, topX):
    K, N = 1024, 640
    L = _layer(K, N, bits, seed=topX + bits, topX=topX, sparsity=0.01)
    fri = np.random.default_rng(topX).integers(0, N, size=topX).astype(np.int32)
    if topX >= 33:
        fri[:5] = fri[0]          # duplicates: each gets the full G
        fri[5] = 0                # channel 0
        fri[6] = N - 1            # the last channel
        fri[7] = N + 3            # out of range: 0
        fri[8] = -2
    L["full_row_indices"] = fri
    T = to_torch(L)
    for M in (1, 9, 65):
        x, dy = exact_rows(K, M, seed=M), exact_rows(N, M, seed=M + 7)
        truth = lut_grad_f64(L, x, dy, device="cuda")
        for xt, dt in PAIRS:
            for path in paths(xt, dt):
                got = call(L, T, x.to(xt), dy.to(dt), path=path)
                check(got, truth, (M, xt, dt, path))
                if topX >= 33:
                    fr = got["full_rows"]
                    assert (fr[:, 7] == 0).all() and (fr[:, 8] == 0).all()
                    assert all(torch.equal(fr[:, j], fr[:, 0]) for j in range(1, 5))


@pytest.mark.parametrize("path", ["tc", "cuda"])
def test_all_dense_rows_on_channel_0(path):
    K, N = 512, 132
    L = _layer(K, N, 4, seed=3, topX=40)
    L["full_row_indices"] = np.zeros(40, dtype=np.int32)
    x, dy = exact_rows(K, 9, seed=4), exact_rows(N, 9, seed=5)
    got = call(L, to_torch(L), x.half(), dy.half(), path=path)
    check(got, lut_grad_f64(L, x, dy, device="cuda"))
    assert all(torch.equal(got["full_rows"][:, j], got["full_rows"][:, 0]) for j in range(40))


@pytest.mark.parametrize("path", ["tc", "cuda"])
def test_csr_edges(path):
    """Empty CSR, no sparse buffers, one 3000-entry row with a duplicated and out-of-range columns, shuffled rows (each entry's
    gradient moves with it, bit for bit), CSR arrays and x / dy starting 1-3 elements into a buffer."""
    K, N, bits, M = 4096, 132, 4, 17
    x, dy = exact_rows(K, M, seed=5), exact_rows(N, M, seed=6)
    xt = dt = F16 if path == "tc" else F32
    xm, dm = x.to(xt), dy.to(dt)
    base = _layer(K, N, bits, seed=6, topX=0, sparsity=0.01)
    empty = dict(base, rows=np.zeros(N + 1, dtype=np.int32), cols=np.zeros(0, dtype=np.int32), vals=np.zeros(0, dtype=np.float32))
    got = call(empty, to_torch(empty), xm, dm, path=path)
    assert got["vals"].numel() == 0
    check(got, lut_grad_f64(empty, x, dy, device="cuda"))
    assert call(empty, to_torch(empty), xm, dm, path=path, want=("vals",))["vals"].numel() == 0
    none = dict(base, rows=None, cols=None, vals=None)
    check(call(none, to_torch(none), xm, dm, path=path), lut_grad_f64(none, x, dy, device="cuda"))
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
    truth = lut_grad_f64(big, x, dy, device="cuda")
    sorted_g = call(big, to_torch(big), xm, dm, path=path)
    check(sorted_g, truth)
    dv = sorted_g["vals"]
    assert dv[rows[3]] == 0 and dv[rows[4]] == 0 and dv[rows[70] + 1] == dv[rows[70]]
    perm = np.arange(len(cols))
    for c in range(N):
        perm[rows[c]:rows[c + 1]] = rows[c] + rng.permutation(rows[c + 1] - rows[c])
    shuffled = dict(big, cols=cols[perm], vals=vals[perm])
    shuf_g = call(shuffled, to_torch(shuffled), xm, dm, path=path)
    assert torch.equal(shuf_g["vals"], dv[torch.from_numpy(perm).cuda()])
    assert torch.equal(shuf_g["lookup_table"], sorted_g["lookup_table"])
    for off in (1, 2, 3):
        T = to_torch(big)
        for k in ("rows", "cols", "vals"):
            buf = torch.zeros(T[k].numel() + off, dtype=T[k].dtype, device="cuda")
            buf[off:] = T[k]
            T[k] = buf[off:]
        xb = torch.zeros(M * K + off, dtype=xt, device="cuda")
        xb[off:] = xm.reshape(-1)
        db = torch.zeros(M * N + off, dtype=dt, device="cuda")
        db[off:] = dm.reshape(-1)
        got = call(big, T, xb[off:].view(M, K), db[off:].view(M, N), path=path)
        assert all(torch.equal(got[k], sorted_g[k]) for k in got)


TILE_KN = [(k, n) for k in (32, 96, 160, 4128, 22016) for n in (4, 60, 68, 132, 131072) if (k, n) != (22016, 131072)]


@pytest.mark.parametrize("K,N", TILE_KN, ids=[f"{k}x{n}" for k, n in TILE_KN])
@pytest.mark.parametrize("bits", [3, 4])
def test_tiling_edges(bits, K, N):
    L = _layer(K, N, bits, seed=K * 7 + N, topX=min(3, N), sparsity=0.02 if K * N < 1 << 24 else 0.0005)
    T = to_torch(L)
    for M in (1, 9, 130):
        x, dy = exact_rows(K, M, seed=M + K), exact_rows(N, M, seed=M + N)
        truth = lut_grad_f64(L, x, dy, device="cuda")
        for xt, dt in ((F16, F16), (BF16, BF16), (F16, F32)):
            for path in paths(xt, dt):
                check(call(L, T, x.to(xt), dy.to(dt), path=path), truth, (M, xt, dt, path))


# ---- reproducibility, graphs, streams ----------------------------------------------------------------------------------------
def test_two_calls_bit_identical():
    K, N, bits = 4096, 4096, 3
    L = _layer(K, N, bits, seed=11)
    T = to_torch(L)
    x, dy = exact_rows(K, 300, seed=12), exact_rows(N, 300, seed=13)
    for xt, dt in PAIRS:
        for path in paths(xt, dt):
            a = call(L, T, x.to(xt), dy.to(dt), path=path)
            b = call(L, T, x.to(xt), dy.to(dt), path=path)
            assert all(torch.equal(a[k], b[k]) for k in a), (xt, dt, path)


@pytest.mark.parametrize("path", ["tc", "cuda"])
def test_cuda_graph_replay(path):
    K, N, bits, M = 4096, 4096, 4, 200
    L = _layer(K, N, bits, seed=13)
    T = to_torch(L)
    sx, sd = exact_rows(K, M, seed=1).bfloat16(), exact_rows(N, M, seed=2).bfloat16()
    call(L, T, sx, sd, path=path)  # warm-up (sets the kernel's shared-memory limit outside the capture)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = call(L, T, sx, sd, path=path)
    for seed in (15, 16):
        x, dy = exact_rows(K, M, seed=seed), exact_rows(N, M, seed=seed + 1)
        sx.copy_(x)
        sd.copy_(dy)
        g.replay()
        torch.cuda.synchronize()
        fresh = call(L, T, x.bfloat16(), dy.bfloat16(), path=path)
        assert all(torch.equal(out[k], fresh[k]) for k in out)
        check({k: v.clone() for k, v in out.items()}, lut_grad_f64(L, x, dy, device="cuda"))


def test_three_streams_at_once():
    K, N = 4096, 4096
    layers = [_layer(K, N, b, seed=20 + i) for i, b in enumerate((4, 3, 4))]
    Ts = [to_torch(L) for L in layers]
    ins = [(exact_rows(K, m, seed=m).to(xt), exact_rows(N, m, seed=m + 1).to(dt))
           for m, xt, dt in ((5, F16, F16), (40, F16, F32), (130, BF16, BF16))]
    alone = [call(L, T, x, d) for L, T, (x, d) in zip(layers, Ts, ins)]
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = []
    torch.cuda.synchronize()
    for L, T, (x, d), s in zip(layers, Ts, ins, streams):
        with torch.cuda.stream(s):
            outs.append(call(L, T, x, d))
    torch.cuda.synchronize()
    for o, a in zip(outs, alone):
        assert all(torch.equal(o[k], a[k]) for k in o)


# ---- module level ------------------------------------------------------------------------------------------------------------
def _module(L, bias=False):
    K, N = L["infeatures"], L["outfeatures"]
    return quant_layer(L, bias=np.random.default_rng(K).standard_normal(N).astype(np.float32) if bias else None).cuda()


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("dtype", [F16, BF16, F32], ids=["f16", "bf16", "f32"])
def test_autograd_of_all_four_tensors(dtype, bias):
    """Gradients of lookup_table, vals, full_rows (and bias) through QuantLinearLUT.forward against torch's fp64 autograd through
    the dense restatement of W, within the bound of the truth's condition S; dx within the input gradient's bound."""
    K, N = 1024, 512
    L = _layer(K, N, 4, seed=40, sparsity=0.01)
    L["cols"][0] = K + 9  # one out-of-range CSR column: its gradient is 0
    m = _module(L, bias)
    params = m.train_codebook(lookup_table=True, vals=True, full_rows=True, bias=bias)
    for shape in ((K,), (1, 1, K), (5, K), (2, 40, K), (96, K)):
        M = int(np.prod(shape[:-1]))
        x = exact_rows(K, M, seed=41).to(dtype).reshape(shape).requires_grad_()
        y = m(x)
        g = exact_rows(N, M, seed=42).to(y.dtype).reshape(y.shape)
        grads = torch.autograd.grad(y, [x] + params, g)
        assert grads[0].dtype == x.dtype and grads[0].shape == x.shape
        assert all(gp.shape == p.shape and gp.dtype == p.dtype for gp, p in zip(grads[1:], params))
        # fp64 autograd through the dense restatement
        P = [p.detach().double().requires_grad_() for p in params]
        xd = x.detach().double().reshape(-1, K)
        yd = xd @ dense_w_torch(L, P[0], P[1], P[2])
        if bias:
            yd = yd + P[3]
        want = torch.autograd.grad(yd, P, g.double().reshape(-1, N))
        _, S = lut_grad_f64(L, xd, g.reshape(-1, N), device="cuda")
        for i, k in enumerate(KEYS):
            assert bound_ratio(grads[1 + i].double().cpu().numpy(), want[i].cpu().numpy(), S[k]) <= 1.0, (shape, k)
        assert grads[2][0] == 0
        if bias:
            Sb = g.double().reshape(-1, N).abs().sum(0).cpu().numpy()
            assert bound_ratio(grads[4].double().cpu().numpy(), want[3].cpu().numpy(), Sb) <= 1.0


def test_dx_bit_identical_with_and_without_codebook_training():
    from squeezellm_b200.quant import quant_cuda
    quant_cuda.set_deterministic(True)  # the one-row forward in its reproducible mode
    try:
        K, N = 2048, 1024
        L = _layer(K, N, 3, seed=50)
        plain, trained = _module(L, bias=True), _module(L, bias=True)
        trained.train_codebook(lookup_table=True, vals=True, full_rows=True, bias=True)
        for shape, dtype in (((K,), F16), ((5, K), F16), ((3, 40, K), BF16), ((130, K), F16), ((64, K), F32)):
            x = exact_rows(K, int(np.prod(shape[:-1])), seed=51).to(dtype).reshape(shape)
            xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
            ya, yb = plain(xa), trained(xb)
            g = torch.randn(ya.shape, device="cuda").to(ya.dtype)
            if dtype == F16 or len(shape) == 1:  # reproducible forward routes
                assert torch.equal(ya.detach(), yb.detach())
            (dxa,) = torch.autograd.grad(ya, xa, g)
            (dxb,) = torch.autograd.grad(yb, xb, g)
            assert torch.equal(dxa, dxb), shape
    finally:
        quant_cuda.set_deterministic(False)


def test_one_lut_grad_launch_for_the_requested_tensors(monkeypatch):
    """One lut_grad launch for the requested tensors; a layer whose only trained tensor is the bias makes none, and dx alone
    still goes through lutgemm_t exactly once."""
    from squeezellm_b200 import quant
    K, N = 1024, 256
    L = _layer(K, N, 4, seed=55)
    calls = []
    for n in ("lut_grad", "lutgemm_t"):
        real = getattr(quant.quant_cuda, n)
        monkeypatch.setattr(quant.quant_cuda, n, (lambda real, n: lambda *a, **kw: (calls.append((n, kw.get("want_lut"), kw.get(
            "want_vals"), kw.get("want_full_rows"))), real(*a, **kw))[1])(real, n))
    m = _module(L, bias=True)
    m.train_codebook(lookup_table=False, bias=True)
    x = torch.randn(70, K, device="cuda", dtype=F16)
    m(x).float().sum().backward()
    assert calls == [] and m.bias.grad is not None
    m.train_codebook(lookup_table=True, full_rows=True)
    m(x).float().sum().backward()
    assert calls == [("lut_grad", True, False, True)]
    calls.clear()
    xg = x.clone().requires_grad_()
    m(xg).float().sum().backward()
    assert sorted(c[0] for c in calls) == ["lut_grad", "lutgemm_t"]


def test_teacher_student_adam_on_the_codebook():
    """A student with the teacher's indices and outliers and a perturbed codebook: 100 Adam steps (lr 1e-3) on the codebook alone,
    full batch of 256 fp16 rows, lower the mean squared output error by at least 100x (an fp64 run of the same problem gains about
    6e4x; the fp16 outputs put a floor near 1e-6 of the initial error)."""
    torch.manual_seed(0)
    K, N = 1024, 512
    L = _layer(K, N, 4, seed=90, topX=4)
    teacher = _module(L)
    S = dict(L, lookup_table=L["lookup_table"] + 0.01 * np.random.default_rng(92).standard_normal(L["lookup_table"].shape).astype(np.float32))
    student = _module(S)
    opt = torch.optim.Adam(student.train_codebook(), lr=1e-3)
    x = torch.randn(256, K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(91)).half()
    with torch.no_grad():
        yt = teacher(x).float()
    losses = []
    for _ in range(100):
        loss = ((student(x).float() - yt) ** 2).mean()
        losses.append(loss.item())
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert losses[-1] * 100 <= losses[0], (losses[0], losses[-1])
    assert torch.equal(student.qweight, teacher.qweight)  # the indices stay fixed


def test_in_place_modification_between_forward_and_backward_raises():
    K, N = 1024, 512
    m = _module(_layer(K, N, 4, seed=81))
    (lut,) = m.train_codebook()
    x = torch.randn(8, K, device="cuda", dtype=F16)
    y = m(x)
    with torch.no_grad():
        lut.mul_(2.0)  # e.g. an optimizer step before this graph's backward
    with pytest.raises(RuntimeError, match="modified or replaced"):
        y.float().sum().backward()
