"""quant_cuda.sample (sqllm_sample) on the GPU against the numpy contract (tests/sample_ref.py), draw by draw.

The sweep: fp32 / fp16 / bf16 logits, V in {1, 3, 4, 5, 31999, 32000, 32001, 128256, 151936, 262144}, 79 rows per launch at random
positions, each row with its own (temperature, top_k, top_p, seed, logit kind) from the grid below; fp16 and bf16 rows give many exact
ties.  A greedy row must be bitwise torch.argmax.  A sampled row's token i is checked in fp64:

  * top-k is exact (the kernel and the reference compare the same fp32 z), so only the top-p boundary can move.  The kernel's masses are
    m_j = expf(fl(z_j - z_max)) rounded to multiples of 2^-44: relative error <= |z_j - z_max| 2^-24 (the subtraction) + 2^-23 (expf,
    2 ulp), plus 2^-45 absolute.  Summed over tokens with weights p_j, sum p_j |z_j - z_max| <= H(p) <= ln V, so every normalised mass
    above a token, and the total, is off by at most e = ln(V) 2^-24 + 2^-23 + V 2^-45 relative; the ratio by 2e.  SLACK = 2 (2e): the
    kernel's kept set K lies between K- (M < top_p - SLACK) and K+ (M < top_p + SLACK).  i must be in K+.
  * The score s_j = z_j + g_j in fp32: g's inner logf is 1 ulp (relative 2^-23), which the outer log turns into 2^-23 absolute, the
    outer logf adds 1 ulp of |g| and the sum 1/2 ulp of |z| + |g|: err_j <= 2^-23 (1 + |g_j|) + 2^-24 (|z_j| + |g_j|); doubled for
    margin, e_j = 2^-22 (1 + |g_j|) + 2^-23 (|z_j| + |g_j|).  The kernel's argmax over K holds s_i >= max over K- of s_j - delta with
    delta = e_i + max over K- of e_j (both scores may be off, in opposite directions).
The worst ratio of the shortfall to delta and the number of draws that fell in the slack (i outside K-, or not the fp64 argmax over
K-) are recorded.  Besides: a row's token is bitwise the same alone (R = 1), among 8 and among 79 rows; idle rows are not written; a
graph that advances pos replays the eager tokens of successive positions; reruns, a view with row stride V + 1 and an odd element
offset, and three streams at once are bitwise equal; rows holding NaN or +inf give ids in [0, V)."""
import math

import numpy as np
import pytest
import torch

import sample_ref as ref

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
VOCABS = [1, 3, 4, 5, 31999, 32000, 32001, 128256, 151936, 262144]
TEMPS = [0.0, 1e-3, 0.7, 1.0, 5.0]
TOPP = [1.0, 0.999, 0.9, 0.5, 1e-6]
KINDS = ["normal1", "normal30", "neginf", "equal", "dominant"]
R = 79


def topks(V):
    return [0, 1, 2, 50, V - 1, V, V + 7]


def make_row(kind, V, rng):
    if kind == "normal1":
        x = rng.normal(size=V)
    elif kind == "normal30":
        x = rng.normal(size=V) * 30
    elif kind == "neginf":
        x = rng.normal(size=V) * 3
        for _ in range(4):  # stretches of -inf, never the whole row
            a = int(rng.integers(0, V))
            x[a:a + max(1, V // 8)] = -np.inf
        x[int(rng.integers(0, V))] = 1.0
    elif kind == "equal":
        x = np.full(V, 0.25)
    else:  # dominant
        x = rng.normal(size=V)
        x[int(rng.integers(0, V))] = 25.0
    return x.astype(np.float32)


def make_batch(V, dt, rows, seed):
    """logits [rows, V] (dt, on the GPU) and the per-row parameters, cycling through the grid from an offset of `seed`."""
    rng = np.random.default_rng(seed)
    grid = [(t, k, p, kind) for t in TEMPS for k in topks(V) for p in TOPP for kind in KINDS]
    off = int(rng.integers(0, len(grid)))
    P = [grid[(off + 11 * b) % len(grid)] for b in range(rows)]
    x = torch.from_numpy(np.stack([make_row(kind, V, rng) for (_, _, _, kind) in P])).to(dt).cuda()
    par = dict(pos=torch.tensor(rng.integers(0, 1 << 20, rows), dtype=torch.int32),
               temperature=torch.tensor([p[0] for p in P], dtype=torch.float32),
               top_k=torch.tensor([p[1] for p in P], dtype=torch.int32),
               top_p=torch.tensor([p[2] for p in P], dtype=torch.float32),
               seed=torch.tensor(rng.integers(0, 2 ** 63 - 1, rows, dtype=np.int64), dtype=torch.int64))
    return x, {k: v.cuda() for k, v in par.items()}


def run(x, par, out=None):
    from squeezellm_b200.quant import quant_cuda
    out = torch.full((x.shape[0],), -7, dtype=torch.int64, device=x.device) if out is None else out
    quant_cuda.sample(x, par["pos"], par["temperature"], par["top_k"], par["top_p"], par["seed"], out)
    return out


def check_row(x, t, k, p, pos, seed, tok):
    """None for a greedy row (checked by the caller), else (in_slack, shortfall / delta)."""
    V = x.size
    z, _, M = ref.row(x, t, k, p)
    e = 2 * (math.log(V) * 2.0 ** -24 + 2.0 ** -23 + V * 2.0 ** -45)
    slack = 2 * 2 * e
    kminus, kplus = ref.kept(M, z, p, -slack), ref.kept(M, z, p, slack)
    if not kminus.any():  # the maximum is always kept
        kminus = ref.kept(M, z, 0.0)
    assert kplus[tok], f"token {tok} outside the kept set (M={M[tok]:.9g}, top_p={p}, top_k={k}, t={t})"
    g = ref.gumbel(V, pos, seed)
    s = z.astype(np.float64) + g
    err = 2.0 ** -22 * (1 + np.abs(g)) + 2.0 ** -23 * (np.abs(z.astype(np.float64)) + np.abs(g))
    sm = np.where(kminus, s, -np.inf)
    best = int(np.argmax(sm))
    delta = err[tok] + err[kminus].max()
    short = sm[best] - s[tok]
    assert short <= delta, f"token {tok} scores {s[tok]:.9g}, the kept maximum {best} {sm[best]:.9g}: {short:.3g} > delta {delta:.3g}"
    return (not kminus[tok] or best != tok), max(short, 0.0) / delta


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("V", VOCABS)
def test_sweep(record, dtype, V):
    x, par = make_batch(V, DTYPES[dtype], R, seed=V * 3 + len(dtype))
    tok = run(x, par).cpu().numpy()
    xs = x.float().cpu().numpy()
    am = x.argmax(dim=1).cpu().numpy()
    pc = {k: v.cpu().numpy() for k, v in par.items()}
    worst, in_slack, sampled = 0.0, 0, 0
    for b in range(R):
        t, k, p = float(pc["temperature"][b]), int(pc["top_k"][b]), float(pc["top_p"][b])
        assert 0 <= tok[b] < V
        if ref.greedy(xs[b], t):
            assert tok[b] == am[b], f"row {b}: greedy token {tok[b]}, torch.argmax {am[b]}"
            continue
        slk, ratio = check_row(xs[b], t, k, p, int(pc["pos"][b]), int(pc["seed"][b]), int(tok[b]))
        sampled += 1
        in_slack += slk
        worst = max(worst, ratio)
    record("sampled_rows", sampled)
    record("worst_ratio_to_delta", worst)
    record("draws_in_slack", in_slack)
    print(f"{dtype} V={V}: {sampled} sampled rows, worst shortfall / delta {worst:.3g}, {in_slack} draws in the slack")


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("V", [5, 32000, 151936])
def test_row_independent_of_the_batch(dtype, V):
    """Each row alone (R = 1) and in a batch of 8 gives bitwise its token in the batch of 79 next to random rows."""
    x, par = make_batch(V, DTYPES[dtype], R, seed=V + 1)
    full = run(x, par)
    for b in (0, 3, 40, 78):
        one = run(x[b:b + 1], {k: v[b:b + 1] for k, v in par.items()})
        assert one.item() == full[b].item()
    x2, par2 = make_batch(V, DTYPES[dtype], 8, seed=V + 2)
    x2[5] = x[40]
    par2 = {k: v.clone() for k, v in par2.items()}
    for k in par2:
        par2[k][5] = par[k][40]
    assert run(x2, par2)[5].item() == full[40].item()


def test_idle_rows_untouched():
    x, par = make_batch(32000, torch.float16, 16, seed=3)
    par["pos"][::3] = -1
    par["pos"][1] = -(2 ** 31)
    out = run(x, par)
    idle = (par["pos"] < 0).cpu()
    assert (out.cpu()[idle] == -7).all() and (out.cpu()[~idle] >= 0).all()
    ref_out = run(x, {**par, "pos": par["pos"].clamp(min=0)})
    assert torch.equal(out[~idle.cuda()], ref_out[~idle.cuda()])


@pytest.mark.parametrize("V", [32000, 128256])
def test_graph_replay_advances_the_position(V):
    """A graph of [sample, pos += 1] replayed n times gives the eager tokens at positions p, p + 1, ..., p + n - 1."""
    x, par = make_batch(V, torch.bfloat16, 8, seed=9)
    par["temperature"].fill_(0.8)
    start = par["pos"].clone()
    out = torch.zeros(8, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(x, par, out)
    torch.cuda.current_stream().wait_stream(s)
    par["pos"].copy_(start)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        run(x, par, out)
        par["pos"].add_(1)
    par["pos"].copy_(start)
    got = []
    for _ in range(6):
        g.replay()
        got.append(out.clone())
    torch.cuda.synchronize()
    for n in range(6):
        want = run(x, {**par, "pos": start + n})
        assert torch.equal(got[n], want)
    assert len({tuple(t.tolist()) for t in got}) > 1  # the position changes the draw


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_rerun_strided_view_and_streams(dtype):
    V = 32001
    x, par = make_batch(V, DTYPES[dtype], 12, seed=21)
    a = run(x, par)
    assert torch.equal(run(x, par), a)
    buf = torch.full((12 * (V + 1) + 3,), float("nan"), dtype=x.dtype, device="cuda")
    view = buf[3:3 + 12 * (V + 1)].view(12, V + 1)[:, :V]  # row stride V + 1, an odd element offset
    view.copy_(x)
    assert view.stride() == (V + 1, 1) and view.storage_offset() == 3
    assert torch.equal(run(view, par), a)
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = [torch.zeros(12, dtype=torch.int64, device="cuda") for _ in streams]
    torch.cuda.synchronize()
    for st, o in zip(streams, outs):
        with torch.cuda.stream(st):
            run(x, par, o)
    torch.cuda.synchronize()
    for o in outs:
        assert torch.equal(o, a)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_nan_and_inf_rows_give_valid_ids(dtype):
    V = 40000
    rows = []
    rng = np.random.default_rng(2)
    for kind in range(8):
        x = rng.normal(size=V).astype(np.float32)
        if kind == 0:
            x[123] = np.nan
        elif kind == 1:
            x[:] = np.nan
        elif kind == 2:
            x[777] = np.inf
        elif kind == 3:
            x[:] = -np.inf
        elif kind == 4:
            x[::2] = np.inf
        elif kind == 5:
            x[5], x[39999] = np.nan, np.inf
        elif kind == 6:
            x[:] = np.inf
        else:
            x[:100] = -np.inf
        rows.append(x)
    x = torch.from_numpy(np.stack(rows)).to(DTYPES[dtype]).cuda()
    n = x.shape[0]
    for t, k, p in ((0.0, 0, 1.0), (1.0, 0, 1.0), (0.7, 50, 0.9), (1e-3, 0, 0.5)):
        par = dict(pos=torch.arange(n, dtype=torch.int32, device="cuda"), temperature=torch.full((n,), t, device="cuda"),
                   top_k=torch.full((n,), k, dtype=torch.int32, device="cuda"), top_p=torch.full((n,), p, device="cuda"),
                   seed=torch.arange(n, dtype=torch.int64, device="cuda"))
        out = run(x, par).cpu()
        assert ((out >= 0) & (out < V)).all(), out
        am = x.argmax(dim=1).cpu()
        for b in (2, 3, 4, 6):  # no NaN: greedy by the rule, bitwise torch.argmax
            assert out[b] == am[b]
