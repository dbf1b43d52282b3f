"""quant_cuda.attn_verify (csrc/attn_verify.cuh) on the GPU: T new tokens at device positions pos .. pos+T-1, against fp64 truth from
the kernel's own inputs per element, and against T successive attn_decode calls bitwise for what it stores.

Per call, with the cache slots from pos on filled with NaN (so any read of a slot the call did not write would show in the output):
  * k_cache and v_cache (and a guard band after them) bitwise equal to what T successive attn_decode calls at pos .. pos+T-1 leave:
    the same k' bits, v unchanged, every other slot untouched, NaN past pos + T still NaN;
  * every output element within the bound of test_attn_decode_gpu.out_bound (DESIGN section 3.17) with its own token's position p_t.
Shapes: (n_heads, n_kv) in test_attn_decode_gpu.HEADS (g = n_heads / n_kv from 1 to 16 and 71: where g does not divide 8, a chunk of
8 rows can start inside a token, and padding rows fill the last chunk; 71 x 1 at T = 16 is 142 clusters, so S = 1), head_dim 64 and
128, fp16 and bf16, T in {1, 2, 5, 8, 16}, pos at 0, 1, 63 - T/2, 64, 64 S - 1, 64 S (S: the split count), 4095 - T and
capacity - T.  Besides: one dominant score (+-1e4) and all-equal scores (also at g = 7 and 71); row t unchanged when the qkv rows
after t change, also to inf or NaN (also at g = 7, with token t split by a chunk edge); the launched split count within 1 .. 8; reruns
and a graph replay that advances the device pos bitwise equal to eager calls; pos < 0 and pos + T > capacity write nothing."""
import pytest
import torch

from test_attn_decode_gpu import CAP, DTYPES, E_SCORE, E_SUM, HEADS, U, rope_tables, rotary64
from util import OUT_ROUNDING

pytestmark = pytest.mark.gpu

TOKENS = [1, 2, 5, 8, 16]


def _quant_cuda():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


class VCase:
    """Inputs of one call: qkv [T, ...], caches [n_kv, CAP, d] inside a buffer with a guard band after them, tables, pos."""

    def __init__(self, nh, nkv, d, dt, pos, T, seed=0, cap=CAP, mode="random"):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.d, self.dt, self.cap, self.pos, self.T = nh, nkv, d, dt, cap, pos, T
        self.scale = d ** -0.5
        n = nkv * cap * d
        self.kbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.vbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.kc, self.vc = self.kbuf[:n].view(nkv, cap, d), self.vbuf[:n].view(nkv, cap, d)
        if 0 <= pos < cap:
            self.kc[:, pos:] = float("nan")
            self.vc[:, pos:] = float("nan")
        self.qkv = torch.randn(T, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.cos, self.sin = rope_tables(cap, d)
        if mode == "equal":      # q = 0: every score 0, the output is the mean of V
            self.qkv[:, :nh * d] = 0
        elif mode == "dominant":  # K rows at scores +1e4 (one) and -1e4 (one) for token 0 against every head of KV head 0's group
            for h in range(1, nh // nkv):
                self.qkv[0, h * d:(h + 1) * d] = self.qkv[0, :d]
            c, s = self.cos[pos].double(), self.sin[pos].double()
            q = rotary64(self.qkv[0, :d].double(), c, s)[0]
            kd = q * (1e4 / (self.scale * float((q * q).sum())))
            self.kc[0, pos // 2] = kd.to(dt)
            self.kc[0, pos // 3] = (-kd).to(dt)
        self.pos_t = torch.tensor([pos], dtype=torch.int32, device="cuda")
        self.out = torch.full((T, nh * d), 7.0, dtype=dt, device="cuda")

    def run(self):
        _quant_cuda().attn_verify(self.qkv, self.pos_t, self.cos, self.sin, self.kc, self.vc, self.out, self.nh, self.nkv, self.scale)

    def run_decode(self):
        """T successive attn_decode calls at pos .. pos+T-1 on this case's caches."""
        qc = _quant_cuda()
        out = torch.empty(self.nh * self.d, dtype=self.dt, device="cuda")
        for t in range(self.T):
            p = torch.tensor([self.pos + t], dtype=torch.int32, device="cuda")
            qc.attn_decode(self.qkv[t].contiguous(), p, self.cos, self.sin, self.kc, self.vc, out, self.nh, self.nkv, self.scale)


def out_bound(case):
    """(want, bound) of the output, fp64 [T, n_heads, d], from the cache as the call left it: token t attends to slots 0 .. pos + t."""
    nh, nkv, d, pos, T = case.nh, case.nkv, case.d, case.pos, case.T
    g, P = nh // nkv, pos + T
    c, s = case.cos[pos:P].double()[:, None], case.sin[pos:P].double()[:, None]
    q = case.qkv[:, :nh * d].double().view(T, nh, d)
    qr, qmag = rotary64(q, c, s)
    qr, qmag = qr.view(T, nkv, g, d), qmag.view(T, nkv, g, d)
    K, V = case.kc[:, :P].double(), case.vc[:, :P].double()
    mask = torch.arange(P, device="cuda")[None, :] > (pos + torch.arange(T, device="cuda"))[:, None]  # [T, P]
    z = case.scale * torch.einsum("tkgd,kpd->tkgp", qr, K)
    A = case.scale * torch.einsum("tkgd,kpd->tkgp", qmag, K.abs())
    m = mask[:, None, None, :]
    z, A = z.masked_fill(m, -torch.inf), A.masked_fill(m, 0)
    p = torch.softmax(z, dim=-1)
    want = torch.einsum("tkgp,kpd->tkgd", p, V).reshape(T, nh, d)
    PV = torch.einsum("tkgp,kpd->tkgd", p, V.abs()).reshape(T, nh, d)
    eps = (torch.expm1(E_SCORE * A.amax(dim=-1, keepdim=True)) + E_SUM).reshape(T, nh, 1)
    r, eta = OUT_ROUNDING[str(case.dt).split(".")[1]]
    return want, r * want.abs() + eta + (1 + r) * 2 * eps * PV


def check_call(case):
    """Runs the case and the same inputs through T attn_decode calls; all the per-call checks; returns the output's bound ratio."""
    twin = VCase(case.nh, case.nkv, case.d, case.dt, case.pos, case.T)
    twin.kbuf.copy_(case.kbuf)
    twin.vbuf.copy_(case.vbuf)
    twin.qkv.copy_(case.qkv)
    case.run()
    twin.run_decode()
    assert torch.equal(case.kbuf.view(torch.int16), twin.kbuf.view(torch.int16)), "k_cache differs from T attn_decode calls"
    assert torch.equal(case.vbuf.view(torch.int16), twin.vbuf.view(torch.int16)), "v_cache differs from T attn_decode calls"
    if case.pos + case.T < case.cap:
        assert torch.isnan(case.kc[:, case.pos + case.T:].float()).all(), "a slot past pos + T was written"
    got = case.out.double().view(case.T, case.nh, case.d)
    assert torch.isfinite(got).all(), "non-finite output: a NaN slot at or past pos + T was read"
    want, bound = out_bound(case)
    err = (got - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def positions(nh, nkv, T, d, dt):
    S = _quant_cuda().attn_verify_splits(nh, nkv, T, d, dt)
    return sorted({p for p in (0, 1, 63 - T // 2, 64, 64 * S - 1, 64 * S, 4095 - T, CAP - T) if 0 <= p <= CAP - T})


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nh,nkv", HEADS, ids=[f"{a}x{b}" for a, b in HEADS])
def test_against_fp64_and_decode(record, nh, nkv, d, dtype):
    worst = 0.0
    for T in TOKENS:
        for i, pos in enumerate(positions(nh, nkv, T, d, DTYPES[dtype])):
            case = VCase(nh, nkv, d, DTYPES[dtype], pos, T, seed=100 * T + i)
            ratio = check_call(case)
            assert ratio <= 1.0, (T, pos, ratio)
            worst = max(worst, ratio)
    record("bound_ratio", worst)


@pytest.mark.parametrize("mode", ["dominant", "equal"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64), (28, 4, 128), (71, 1, 64)])
def test_extreme_scores(record, nh, nkv, d, dtype, mode):
    worst = 0.0
    for pos in (2, 700, 4090):
        case = VCase(nh, nkv, d, DTYPES[dtype], pos, 5, seed=pos, mode=mode)
        ratio = check_call(case)
        assert ratio <= 1.0, (pos, ratio)
        worst = max(worst, ratio)
        if mode == "dominant":  # token 0's output is the dominant row's V, to the output's rounding
            kv0 = case.vc[0, pos // 2].double()
            got = case.out[0].double().view(nh, d)[:nh // nkv]
            assert ((got - kv0).abs() <= 2 * OUT_ROUNDING[str(case.dt).split(".")[1]][0] * kv0.abs() + 1e-6).all()
    record("bound_ratio", worst)


@pytest.mark.parametrize("nh,nkv,d", [(32, 32, 128), (32, 8, 128), (8, 2, 64), (28, 4, 128)])
def test_row_ignores_later_rows(nh, nkv, d):
    """At g = 7, token t = 2's rows 14 .. 20 straddle the chunk edge at 16, and chunk 2 holds rows of token 3 as well."""
    T, t, pos = 8, 2, 777
    a = VCase(nh, nkv, d, torch.float16, pos, T, seed=4)
    b = VCase(nh, nkv, d, torch.float16, pos, T, seed=4)
    b.qkv[t + 1:] = torch.randn_like(b.qkv[t + 1:].float()).half()
    a.run()
    b.run()
    assert torch.equal(a.out[:t + 1].view(torch.int16), b.out[:t + 1].view(torch.int16))
    assert torch.equal(a.kc[:, :pos + t + 1].view(torch.int16), b.kc[:, :pos + t + 1].view(torch.int16))
    assert not torch.equal(a.out[t + 1:], b.out[t + 1:])


@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("nh,nkv,d", [(32, 32, 128), (8, 2, 64), (28, 4, 128)])
def test_row_ignores_non_finite_later_rows(nh, nkv, d, bad):
    """A later token's k and v that overflowed (inf) or are NaN leave the earlier rows' outputs bitwise as they were.  At g = 7, token
    t = 3's rows 21 .. 27 straddle the chunk edge at 24, and chunk 3 holds rows of token 4 as well."""
    T, t, pos = 8, 3, 300
    a = VCase(nh, nkv, d, torch.float16, pos, T, seed=6)
    b = VCase(nh, nkv, d, torch.float16, pos, T, seed=6)
    b.qkv[t + 1:, nh * d:] = float(bad)
    a.run()
    b.run()
    assert torch.isfinite(b.out[:t + 1].float()).all()
    assert torch.equal(a.out[:t + 1].view(torch.int16), b.out[:t + 1].view(torch.int16))


def test_launch_splits_keep_every_cluster_resident():
    """The launched S is in 1 .. 8 for every instance, and at one token it is at most the decode kernel's."""
    qc = _quant_cuda()
    for nh, nkv in HEADS + [(32, 4), (64, 8)]:
        for T in TOKENS:
            for d in (64, 128):
                for dt in DTYPES.values():
                    S = qc.attn_verify_splits(nh, nkv, T, d, dt)
                    assert 1 <= S <= 8
    assert qc.attn_verify_splits(32, 32, 1) <= qc.attn_decode_splits(32, 32)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_bitwise_reproducible(dtype):
    case = VCase(32, 8, 128, DTYPES[dtype], 3001, 8, seed=5)
    outs = []
    for _ in range(5):
        case.run()
        outs.append((case.out.clone(), case.kc[:, 3001:3009].clone()))
    for o, k in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0][0].view(torch.int16))
        assert torch.equal(k.view(torch.int16), outs[0][1].view(torch.int16))


@pytest.mark.parametrize("nh,nkv,d", [(32, 32, 128), (8, 2, 64)])
def test_graph_replay_advances_pos_on_device(nh, nkv, d):
    """N verify steps of one captured call + pos += T, each with new qkv, bitwise equal to N eager calls at the same positions."""
    N, T, p0 = 6, 4, 250
    dt = torch.float16
    g = torch.Generator(device="cuda").manual_seed(9)
    qkvs = torch.randn(N, T, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
    eager = VCase(nh, nkv, d, dt, p0, T, seed=1)
    graphed = VCase(nh, nkv, d, dt, p0, T, seed=1)
    outs_e, outs_g = [], []
    for i in range(N):
        eager.qkv.copy_(qkvs[i])
        eager.pos_t.fill_(p0 + T * i)
        eager.run()
        outs_e.append(eager.out.clone())
    qc = _quant_cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        qc.attn_verify(graphed.qkv, graphed.pos_t, graphed.cos, graphed.sin, graphed.kc, graphed.vc, graphed.out, nh, nkv, graphed.scale)
        graphed.pos_t.add_(T)
    for i in range(N):
        graphed.qkv.copy_(qkvs[i])
        graph.replay()
        outs_g.append(graphed.out.clone())
    torch.cuda.synchronize()
    assert int(graphed.pos_t) == p0 + N * T
    for a, b in zip(outs_e, outs_g):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(eager.kbuf.view(torch.int16), graphed.kbuf.view(torch.int16))
    assert torch.equal(eager.vbuf.view(torch.int16), graphed.vbuf.view(torch.int16))


@pytest.mark.parametrize("pos", [CAP - 4 + 1, CAP, -1])
def test_positions_outside_the_cache_write_nothing(pos):
    case = VCase(8, 2, 128, torch.float16, pos, 4, seed=2)
    before_k, before_v, before_out = case.kbuf.clone(), case.vbuf.clone(), case.out.clone()
    case.run()
    torch.cuda.synchronize()
    assert torch.equal(case.kbuf.view(torch.int16), before_k.view(torch.int16))  # the cache and the guard band after it
    assert torch.equal(case.vbuf.view(torch.int16), before_v.view(torch.int16))
    assert torch.equal(case.out.view(torch.int16), before_out.view(torch.int16))


def test_the_stored_k_is_one_rounding_of_the_fp64_rotary():
    case = VCase(32, 8, 128, torch.bfloat16, 900, 16, seed=8)
    case.run()
    r, eta = OUT_ROUNDING["bfloat16"]
    for t in range(case.T):
        p = case.pos + t
        kn = case.qkv[t, 32 * 128:40 * 128].double().view(8, 128)
        k64, kmag = rotary64(kn, case.cos[p].double(), case.sin[p].double())
        got = case.kc[:, p].double()
        assert ((got - k64).abs() <= r * k64.abs() + eta + (1 + r) * 4 * U * kmag).all(), t
