"""quant_cuda.attn_extend (csrc/attn_extend.cuh) on the GPU against fp64 truth built from the kernel's own inputs, per element.

Per call, with the cache slots before `start` random and the slots from `start` on NaN (so any read past the chunk shows in the output):
  * the stored cache bitwise equal to what T successive attn_decode calls at start .. start+T-1 leave (k' and v at the chunk's slots,
    every other slot and the guard band after the cache unchanged: the NaN slots past start + T stay NaN);
  * every output element within the bound of `out_bound`, reported as its ratio (<= 1 passes).
Shapes: (n_heads, n_kv) in test_attn_decode_gpu.HEADS (g = n_heads / n_kv from 1 to 16 and 71: where g does not divide 64,
a 64-row query tile of a group can start inside a token), head_dim 64 and 128, fp16 and bf16, (start, T) from one token at 0 to 2048 tokens
at 0, across the 64-key blocks and with a few tokens on a long history; scores at +-1e4 and all-equal scores (also at g = 7 and 71);
two calls bitwise equal; out row t independent of the qkv rows after t (also at g = 7, with token t split by a tile edge); a
CUDA-graph replay bitwise equal to the eager call; T = 1 against attn_decode.

The bound.  For token t at p = start + t and head h, with z_j = scale q'.K_j (natural-log units), A_j = scale sum_d |q'-terms| |K_jd|
(the rotary's terms summed in magnitude, as in test_attn_decode_gpu) and the fp64 softmax weights w_j:
  * score error |dz_j| <= E_SCORE A_j + E_ABS scale sum_d |K_jd|:
      - q' = hi + lo + r with hi = dt(x), lo = dt(x - hi) at x = q'/4: |r| <= u_dt^2 |x| (+ half a subnormal of lo in fp16), u_dt = 2^-11
        (fp16) or 2^-8 (bf16): U_SPLIT = 2^-22 or 2^-16 of each |q'_d|, and in fp16 E_ABS = 4 * 2^-25 = 2^-23 per unit of |K_jd|;
      - K is exact in the dtype and every hi/lo x K product is exact in fp32; the tensor cores add the 2 D / 16 <= 16 partial MMAs of a
        score in fp32 (rounded or truncated: <= 2^-23 of the magnitudes each, 2^-19 together), then the fp32 rotary (3 u), the /4 and
        the base-2 scale (2 u): below 2^-18 in all.  E_SCORE = U_SPLIT + 2^-17 leaves a factor of two.
  * weight and sum error E_SUM (relative to sum_j w_j |V_j|): P = hi + lo in the dtype (U_SPLIT of each weight, plus in fp16 half a
    subnormal absolute, ETA_P = 2^-25 of each |V_j| since every weight is <= 1 and the final sum >= 1); exp2f (2 ulp); the fp32 chains
    of the online softmax: the tensor-core accumulation of O over 2 MMAs per 16 keys (2^-22 each, truncation included), the running
    sum over a lane's keys, the 4-lane and cluster combines and the final division - at most 2 ceil((p + 1) / 16) + 64 steps of 2^-22.
  * out = round(sum w V / sum w): |out - want| <= r |want| + eta + (1 + r) (2 eps sum_j w_j |V_j| + ETA_P sum_j |V_j|), with
    eps = expm1(max_j |dz_j|) + E_SUM, the factor 2 for the numerator and the denominator (r, eta: util.OUT_ROUNDING)."""
import math

import numpy as np
import pytest
import torch

from test_attn_decode_gpu import HEADS
from util import OUT_ROUNDING

pytestmark = pytest.mark.gpu

CAP = 4160
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
CHUNKS = [(0, 1), (0, 17), (0, 64), (0, 65), (63, 2), (64, 64), (100, 300), (4000, 8), (0, 2048), (CAP - 5, 5)]
U_SPLIT = {torch.float16: 2.0 ** -22, torch.bfloat16: 2.0 ** -16}
E_ABS = {torch.float16: 2.0 ** -23, torch.bfloat16: 0.0}
ETA_P = {torch.float16: 2.0 ** -25, torch.bfloat16: 0.0}


def _quant_cuda():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def rope_tables(cap, d, identity=False):
    if identity:  # cos 1, sin 0: q' = q at every position
        return torch.ones(cap, d // 2, device="cuda"), torch.zeros(cap, d // 2, device="cuda")
    inv = 1.0 / (10000.0 ** (np.arange(0, d, 2, dtype=np.float64) / d))
    ang = np.arange(cap, dtype=np.float64)[:, None] * inv[None, :]
    return (torch.from_numpy(np.cos(ang)).float().cuda(), torch.from_numpy(np.sin(ang)).float().cuda())


def rotary64(x, c, s):
    """rotate-half rotary of x [..., d] in fp64 with fp64 tables c, s [..., d/2]; also the |terms| sum."""
    h = x.shape[-1] // 2
    a, b = x[..., :h], x[..., h:]
    rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1)
    mag = torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], dim=-1)
    return rot, mag


class Case:
    """Inputs of one call: qkv [T, ...], caches [n_kv, cap, d] inside a buffer with a guard band after them, tables, start."""

    def __init__(self, nh, nkv, d, dt, start, T, seed=0, cap=CAP, mode="random"):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.d, self.dt, self.cap, self.start, self.T = nh, nkv, d, dt, cap, start, T
        self.scale = 1.0 / math.sqrt(d)
        n = nkv * cap * d
        self.kbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.vbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.kc, self.vc = self.kbuf[:n].view(nkv, cap, d), self.vbuf[:n].view(nkv, cap, d)
        self.kc[:, start:] = float("nan")
        self.vc[:, start:] = float("nan")
        self.qkv = torch.randn(T, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.cos, self.sin = rope_tables(cap, d, identity=mode == "dominant")
        if mode == "equal":      # q = 0: every score 0, the output is the mean of V[0..p]
            self.qkv[:, :nh * d] = 0
        elif mode == "dominant":  # K rows at scores +1e4 (one) and -1e4 (one) against every head of KV head 0's group, every token
            q = self.qkv[0, :d].clone()
            for h in range(nh // nkv):
                self.qkv[:, h * d:(h + 1) * d] = q
            q = q.double()
            kd = q * (1e4 / (self.scale * float((q * q).sum())))
            self.kc[0, start // 2] = kd.to(dt)
            self.kc[0, start // 3] = (-kd).to(dt)
        self.out = torch.full((T, nh * d), 7.0, dtype=dt, device="cuda")

    def run(self, out=None, qkv=None):
        _quant_cuda().attn_extend(self.qkv if qkv is None else qkv, self.start, self.cos, self.sin, self.kc, self.vc,
                                  self.out if out is None else out, self.nh, self.nkv, self.scale)


def out_bound(case, TB=64):
    """(want, bound) of the output, fp64 [T, n_heads, d], from the cache as the call left it."""
    nh, nkv, d, start, T, dt = case.nh, case.nkv, case.d, case.start, case.T, case.dt
    L = start + T
    kv_of = torch.arange(nh, device="cuda") // (nh // nkv)
    K = case.kc[:, :L].double()[kv_of]        # [nh, L, d]
    V = case.vc[:, :L].double()[kv_of]
    Ka, Va = K.abs(), V.abs()
    Ksum = case.scale * Ka.sum(-1)            # [nh, L]
    q = case.qkv[:, :nh * d].double().view(T, nh, d)
    c = case.cos[start:L].double()[:, None, :]
    s = case.sin[start:L].double()[:, None, :]
    qr, qmag = rotary64(q, c, s)              # [T, nh, d]
    r, eta = OUT_ROUNDING[str(dt).split(".")[1]]
    e_score = U_SPLIT[dt] + 2.0 ** -17
    wants, bounds = [], []
    j = torch.arange(L, device="cuda")
    for t0 in range(0, T, TB):
        t1 = min(T, t0 + TB)
        p = start + torch.arange(t0, t1, device="cuda")                 # [tb]
        masked = j[None, :] > p[:, None]                                 # [tb, L]
        z = case.scale * torch.einsum("thd,hjd->htj", qr[t0:t1], K).masked_fill(masked, -math.inf)
        A = case.scale * torch.einsum("thd,hjd->htj", qmag[t0:t1], Ka).masked_fill(masked, 0.0)
        dz = e_score * A + E_ABS[dt] * Ksum[:, None, :].masked_fill(masked, 0.0)
        w = torch.softmax(z, dim=-1)
        want = torch.einsum("htj,hjd->htd", w, V)
        PV = torch.einsum("htj,hjd->htd", w, Va)
        Vsum = torch.einsum("tj,hjd->htd", (~masked).double(), Va)
        e_sum = U_SPLIT[dt] + 2.0 ** -22 * (2 * torch.ceil((p + 1) / 16.0).double() + 64)   # [tb]
        eps = torch.expm1(dz.max(dim=-1).values) + e_sum[None, :]         # [nh, tb]
        bound = r * want.abs() + eta + (1 + r) * (2 * eps[..., None] * PV + ETA_P[dt] * Vsum)
        wants.append(want.transpose(0, 1))
        bounds.append(bound.transpose(0, 1))
    return torch.cat(wants), torch.cat(bounds)


def ratio(case, out=None):
    got = (case.out if out is None else out).double().view(case.T, case.nh, case.d)
    assert torch.isfinite(got).all(), "non-finite output: a NaN slot at or past start + T was read"
    want, bound = out_bound(case)
    err = (got - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def decode_cache(case, kbuf, vbuf):
    """kbuf / vbuf (copies of the caches before the call) after T successive attn_decode calls at start .. start+T-1."""
    n = case.nkv * case.cap * case.d
    kc, vc = kbuf[:n].view(case.nkv, case.cap, case.d), vbuf[:n].view(case.nkv, case.cap, case.d)
    out = torch.empty(case.nh * case.d, dtype=case.dt, device="cuda")
    pos = torch.empty(1, dtype=torch.int32, device="cuda")
    for t in range(case.T):
        pos.fill_(case.start + t)
        _quant_cuda().attn_decode(case.qkv[t], pos, case.cos, case.sin, kc, vc, out, case.nh, case.nkv, case.scale)
    return out


def check_cache(case, before_k, before_v):
    """The caches as the call left them: bitwise what attn_decode stores at start .. start+T-1, everything else unchanged."""
    n = case.nkv * case.cap * case.d
    mask = torch.ones(case.kbuf.numel(), dtype=torch.bool, device="cuda")
    mask[:n].view(case.nkv, case.cap, case.d)[:, case.start:case.start + case.T] = False
    assert torch.equal(case.kbuf.view(torch.int16)[mask], before_k.view(torch.int16)[mask]), "a k slot outside the chunk changed"
    assert torch.equal(case.vbuf.view(torch.int16)[mask], before_v.view(torch.int16)[mask]), "a v slot outside the chunk changed"
    kd, vd = before_k.clone(), before_v.clone()
    decode_cache(case, kd, vd)
    assert torch.equal(case.kbuf.view(torch.int16), kd.view(torch.int16)), "stored k differs from attn_decode's"
    assert torch.equal(case.vbuf.view(torch.int16), vd.view(torch.int16)), "stored v differs from attn_decode's"
    v_new = case.qkv[:, (case.nh + case.nkv) * case.d:].reshape(case.T, case.nkv, case.d).transpose(0, 1)
    assert torch.equal(case.vc[:, case.start:case.start + case.T].view(torch.int16), v_new.view(torch.int16)), "stored v not bit-exact"


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nh,nkv", HEADS, ids=[f"{a}x{b}" for a, b in HEADS])
def test_against_fp64(record, nh, nkv, d, dtype):
    worst = 0.0
    for i, (start, T) in enumerate(CHUNKS):
        case = Case(nh, nkv, d, DTYPES[dtype], start, T, seed=i)
        before_k, before_v = case.kbuf.clone(), case.vbuf.clone()
        case.run()
        check_cache(case, before_k, before_v)
        rt = ratio(case)
        assert rt <= 1.0, (start, T, rt)
        worst = max(worst, rt)
    record("bound_ratio", worst)


@pytest.mark.parametrize("mode", ["dominant", "equal"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64), (28, 4, 128), (71, 1, 64)])
def test_extreme_scores(record, nh, nkv, d, dtype, mode):
    worst = 0.0
    for start, T in ((5, 5), (700, 64), (4000, 100)):
        case = Case(nh, nkv, d, DTYPES[dtype], start, T, seed=start, mode=mode)
        before_k, before_v = case.kbuf.clone(), case.vbuf.clone()
        case.run()
        check_cache(case, before_k, before_v)
        rt = ratio(case)
        assert rt <= 1.0, (start, T, rt)
        worst = max(worst, rt)
        if mode == "dominant":  # every token's output of group 0 is the dominant row's V, to the output's rounding
            kv0 = case.vc[0, start // 2].double()
            got = case.out.double().view(T, nh, d)[:, :nh // nkv]
            assert ((got - kv0).abs() <= 2 * OUT_ROUNDING[str(case.dt).split(".")[1]][0] * kv0.abs() + 1e-6).all()
    record("bound_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("start,T", [(4000, 8), (100, 300)])
def test_bitwise_reproducible(dtype, start, T):
    case = Case(32, 8, 128, DTYPES[dtype], start, T, seed=5)
    outs = []
    for _ in range(3):
        case.run()
        outs.append((case.out.clone(), case.kbuf.clone()))
    for o, k in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0][0].view(torch.int16))
        assert torch.equal(k.view(torch.int16), outs[0][1].view(torch.int16))


@pytest.mark.parametrize("nh,nkv,d,start,T", [(32, 8, 128, 100, 300), (8, 2, 64, 4000, 8), (32, 32, 128, 0, 130),
                                               (28, 4, 128, 100, 55)])
def test_causal(nh, nkv, d, start, T):
    """Changing the qkv rows after t leaves out rows 0..t bitwise unchanged.  At g = 7 and T = 55, t = 27: token 27's rows 189 .. 195
    straddle the tile edge at 192, so tile 3 holds heads of token 27 and of every token after it."""
    case = Case(nh, nkv, d, torch.float16, start, T, seed=3)
    case.run()
    first = case.out.clone()
    t = T // 2
    g = torch.Generator(device="cuda").manual_seed(11)
    case.qkv[t + 1:] = torch.randn(T - t - 1, case.qkv.shape[1], generator=g, device="cuda").to(case.dt)
    case.run()
    assert torch.equal(case.out[:t + 1].view(torch.int16), first[:t + 1].view(torch.int16))
    assert not torch.equal(case.out[t + 1:].view(torch.int16), first[t + 1:].view(torch.int16))


@pytest.mark.parametrize("nh,nkv,d,start,T", [(32, 8, 128, 4000, 8), (8, 2, 64, 64, 64)])
def test_graph_replay_equals_eager(nh, nkv, d, start, T):
    eager = Case(nh, nkv, d, torch.bfloat16, start, T, seed=1)
    graphed = Case(nh, nkv, d, torch.bfloat16, start, T, seed=1)
    eager.run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        graphed.run()
    graphed.out.fill_(7.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.out.view(torch.int16), graphed.out.view(torch.int16))
    assert torch.equal(eager.kbuf.view(torch.int16), graphed.kbuf.view(torch.int16))
    assert torch.equal(eager.vbuf.view(torch.int16), graphed.vbuf.view(torch.int16))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (32, 32, 64), (8, 2, 128)])
def test_one_token_agrees_with_decode(nh, nkv, d, dtype):
    """T = 1 at several positions: the same stored k / v as attn_decode, and an output within the bound of attn_decode's."""
    for start in (0, 63, 1000, CAP - 1):
        case = Case(nh, nkv, d, DTYPES[dtype], start, 1, seed=start)
        kd, vd = case.kbuf.clone(), case.vbuf.clone()
        case.run()
        dec = decode_cache(case, kd, vd)
        assert torch.equal(case.kbuf.view(torch.int16), kd.view(torch.int16))
        _, bound = out_bound(case)
        diff = (case.out.double().view(1, nh, d) - dec.double().view(1, nh, d)).abs()
        assert (diff <= 2 * bound).all(), float((diff / bound).max())


def test_splits_rule_on_the_device():
    qc = _quant_cuda()
    sm = qc.sm_count()
    assert qc.attn_extend_splits(32, 8, 8, 4000) == max(1, min(8, sm // 8, (4008 + 63) // 64))
    assert qc.attn_extend_splits(32, 8, 2048, 0) == 1
    assert qc.attn_extend_splits(32, 8, 0, 0) == 0
