"""quant_cuda.attn_decode (csrc/attn_decode.cuh) on the GPU against fp64 truth built from the kernel's own inputs, per element.

Per call, with the cache slots past `pos` filled with NaN (so any read of them would show in the output):
  * the stored k within one rounding to the dtype (plus the fp32 rotary's terms) of the fp64 rotary of qkv's k;
  * the stored v bit-exact, every other cache slot bitwise unchanged;
  * the output within the bound of `out_bound`, reported as its ratio (<= 1 passes) like util.bound_ratio.
Shapes: (n_heads, n_kv) in HEADS, with query heads per KV head g in {1, 2, 3, 4, 5, 6, 7, 8, 12, 16, 71} (every instance G in
{1, 2, 4, 8}, padding rows for g = 3, 5, 6, 7, a group over several clusters for g > 8), head_dim 64 and 128, fp16 and bf16, pos at 0,
1, both sides of the first two split boundaries, 4095 and capacity - 1; one dominant score (+-1e4) and all-equal scores (also at g = 7
and at g = 71, whose group 0 spans nine clusters); repeated runs bitwise equal; N steps replayed in a CUDA graph that advances pos on
the device bitwise equal to N eager calls (also at g = 12, where only the first cluster of a group appends); pos = capacity writes
nothing."""
import math

import numpy as np
import pytest
import torch

from util import OUT_ROUNDING

pytestmark = pytest.mark.gpu

CAP = 4160
# (n_heads, n_kv) of every kernel test of the four attention kernels: g = n_heads / n_kv at 1 and 4 (G = 1, 4), 2 (G = 2), 3, 5, 6
# and 7 (padding rows in G = 4 or 8, and one token's heads split across verify chunks of 8 rows and extend tiles of 64), 8 (G = 8 with
# U = 2), 12 and 16 (a group over two clusters, the last one partial at 12) and the MQA 71 x 1 (nine clusters, the last of 7 heads)
HEADS = [(32, 32), (32, 8), (8, 2), (4, 4), (16, 8), (24, 8), (40, 8), (12, 2), (28, 4), (64, 8), (48, 4), (32, 2), (71, 1)]
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
U = 2.0 ** -24
E_SCORE = 2.0 ** -19  # fp32 terms of a score, relative to scale * sum_d |q-rotary terms| |k_d|: the rotary, the 8-term FMA chain, the
#                      4-step shuffle sum, the base-2 scale (about 16 roundings; 32 u leaves a factor of two)
E_SUM = 2.0 ** -18    # fp32 terms of the softmax's sums and weighted sum along one chain: the positions of a lane's slot, the xor tree,
#                      the warp and rank combines, exp2f and the final division (at most ~40 roundings at 4160 positions; 64 u)


def _quant_cuda():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def rope_tables(cap, d):
    inv = 1.0 / (10000.0 ** (np.arange(0, d, 2, dtype=np.float64) / d))
    ang = np.arange(cap, dtype=np.float64)[:, None] * inv[None, :]
    return (torch.from_numpy(np.cos(ang)).float().cuda(), torch.from_numpy(np.sin(ang)).float().cuda())


def rotary64(x, c, s):
    """rotate-half rotary of x [..., d] in fp64 with fp64 tables of the fp32 values c, s [d/2]; also the |terms| sum."""
    h = x.shape[-1] // 2
    a, b = x[..., :h], x[..., h:]
    rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1)
    mag = torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], dim=-1)
    return rot, mag


class Case:
    """Inputs of one call: qkv, caches [n_kv, CAP, d] inside a buffer with a guard band after them, tables, pos."""

    def __init__(self, nh, nkv, d, dt, pos, seed=0, cap=CAP, mode="random"):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.d, self.dt, self.cap, self.pos = nh, nkv, d, dt, cap, pos
        self.scale = 1.0 / math.sqrt(d)
        n = nkv * cap * d
        self.kbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.vbuf = torch.randn(n + 4096, generator=g, device="cuda").to(dt)
        self.kc, self.vc = self.kbuf[:n].view(nkv, cap, d), self.vbuf[:n].view(nkv, cap, d)
        if pos + 1 < cap:
            self.kc[:, pos + 1:] = float("nan")
            self.vc[:, pos + 1:] = float("nan")
        self.qkv = torch.randn((nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.cos, self.sin = rope_tables(cap, d)
        if mode == "equal":      # q = 0: every score 0, the output is the mean of V
            self.qkv[:nh * d] = 0
        elif mode == "dominant" and pos >= 2:  # K rows at scores +1e4 (one) and -1e4 (one) against every head of KV head 0's group
            for h in range(1, nh // nkv):  # every head of the group gets head 0's q, so the same dominant score
                self.qkv[h * d:(h + 1) * d] = self.qkv[:d]
            q = self.q64()[0]
            kd = q * (1e4 / (self.scale * float((q * q).sum())))
            self.kc[0, pos // 2] = kd.to(dt)
            self.kc[0, pos // 3] = (-kd).to(dt)
        self.pos_t = torch.tensor([pos], dtype=torch.int32, device="cuda")
        self.out = torch.full((nh * d,), 7.0, dtype=dt, device="cuda")

    def q64(self):
        if 0 <= self.pos < self.cap:
            c, s = self.cos[self.pos].double(), self.sin[self.pos].double()
        else:
            c = s = torch.zeros(self.d // 2, dtype=torch.float64, device="cuda")
        q = self.qkv[:self.nh * self.d].double().view(self.nh, self.d)
        return rotary64(q, c, s)[0]

    def run(self):
        _quant_cuda().attn_decode(self.qkv, self.pos_t, self.cos, self.sin, self.kc, self.vc, self.out, self.nh, self.nkv, self.scale)


def out_bound(case):
    """(want, bound) of the output, fp64 [n_heads, d], from the cache as the call left it (slot pos: the stored k and v)."""
    nh, nkv, d, pos = case.nh, case.nkv, case.d, case.pos
    c, s = case.cos[pos].double(), case.sin[pos].double()
    q = case.qkv[:nh * d].double().view(nh, d)
    qr, qmag = rotary64(q, c, s)
    kv_of = torch.arange(nh, device="cuda") // (nh // nkv)
    K = case.kc[:, :pos + 1].double()[kv_of]          # [nh, T, d]
    V = case.vc[:, :pos + 1].double()[kv_of]
    z = case.scale * torch.einsum("hd,htd->ht", qr, K)
    A = case.scale * torch.einsum("hd,htd->ht", qmag, K.abs())
    p = torch.softmax(z, dim=-1)
    want = torch.einsum("ht,htd->hd", p, V)
    PV = torch.einsum("ht,htd->hd", p, V.abs())
    eps = torch.expm1(E_SCORE * A.max(dim=-1, keepdim=True).values) + E_SUM
    r, eta = OUT_ROUNDING[str(case.dt).split(".")[1]]
    return want, r * want.abs() + eta + (1 + r) * 2 * eps * PV


def check_call(case, before_k, before_v):
    """All the per-call checks; returns the output's bound ratio."""
    nh, nkv, d, pos, dt = case.nh, case.nkv, case.d, case.pos, case.dt
    r, eta = OUT_ROUNDING[str(dt).split(".")[1]]
    kn = case.qkv[nh * d:(nh + nkv) * d].double().view(nkv, d)
    k64, kmag = rotary64(kn, case.cos[pos].double(), case.sin[pos].double())
    got_k = case.kc[:, pos].double()
    assert ((got_k - k64).abs() <= r * k64.abs() + eta + (1 + r) * 4 * U * kmag).all(), "stored k beyond one rounding"
    assert torch.equal(case.vc[:, pos].view(torch.int16), case.qkv[(nh + nkv) * d:].view(nkv, d).view(torch.int16)), "stored v not bit-exact"
    mask = torch.ones(case.kbuf.numel(), dtype=torch.bool, device="cuda")
    mask[:nkv * case.cap * d].view(nkv, case.cap, d)[:, pos] = False
    assert torch.equal(case.kbuf.view(torch.int16)[mask], before_k.view(torch.int16)[mask]), "a k slot other than pos changed"
    assert torch.equal(case.vbuf.view(torch.int16)[mask], before_v.view(torch.int16)[mask]), "a v slot other than pos changed"
    got = case.out.double().view(nh, d)
    assert torch.isfinite(got).all(), "non-finite output: a NaN slot past pos was read"
    want, bound = out_bound(case)
    err = (got - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def positions(nh, nkv):
    S = _quant_cuda().attn_decode_splits(nh, nkv)
    return sorted({0, 1, 63, 64, 65, 64 * S - 1, 64 * S, 64 * S + 1, 4095, CAP - 1})


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nh,nkv", HEADS, ids=[f"{a}x{b}" for a, b in HEADS])
def test_against_fp64(record, nh, nkv, d, dtype):
    worst = 0.0
    for i, pos in enumerate(positions(nh, nkv)):
        case = Case(nh, nkv, d, DTYPES[dtype], pos, seed=i)
        before_k, before_v = case.kbuf.clone(), case.vbuf.clone()
        case.run()
        ratio = check_call(case, before_k, before_v)
        assert ratio <= 1.0, (pos, ratio)
        worst = max(worst, ratio)
    record("bound_ratio", worst)


@pytest.mark.parametrize("mode", ["dominant", "equal"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64), (28, 4, 128), (71, 1, 64)])
def test_extreme_scores(record, nh, nkv, d, dtype, mode):
    worst = 0.0
    for pos in (2, 700, 4095):
        case = Case(nh, nkv, d, DTYPES[dtype], pos, seed=pos, mode=mode)
        before_k, before_v = case.kbuf.clone(), case.vbuf.clone()
        case.run()
        ratio = check_call(case, before_k, before_v)
        assert ratio <= 1.0, (pos, ratio)
        worst = max(worst, ratio)
        if mode == "dominant":  # the output is the dominant row's V, to the output's rounding
            kv0 = case.vc[0, pos // 2].double()
            got = case.out.double().view(nh, d)[:nh // nkv]
            assert ((got - kv0).abs() <= 2 * OUT_ROUNDING[str(case.dt).split(".")[1]][0] * kv0.abs() + 1e-6).all()
    record("bound_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_bitwise_reproducible(dtype):
    case = Case(32, 8, 128, DTYPES[dtype], 3001, seed=5)
    outs = []
    for _ in range(5):
        case.run()
        outs.append((case.out.clone(), case.kc[:, 3001].clone()))
    for o, k in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0][0].view(torch.int16))
        assert torch.equal(k.view(torch.int16), outs[0][1].view(torch.int16))


@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64), (48, 4, 128)])
def test_graph_replay_advances_pos_on_device(nh, nkv, d):
    """N steps of one captured call + pos += 1, each with new qkv, bitwise equal to N eager calls at the same positions."""
    N, p0 = 12, 250
    dt = torch.float16
    g = torch.Generator(device="cuda").manual_seed(9)
    qkvs = torch.randn(N, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
    eager = Case(nh, nkv, d, dt, p0, seed=1)
    graphed = Case(nh, nkv, d, dt, p0, seed=1)
    outs_e, outs_g = [], []
    for i in range(N):
        eager.qkv.copy_(qkvs[i])
        eager.pos_t.fill_(p0 + i)
        eager.run()
        outs_e.append(eager.out.clone())
    qc = _quant_cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        qc.attn_decode(graphed.qkv, graphed.pos_t, graphed.cos, graphed.sin, graphed.kc, graphed.vc, graphed.out, nh, nkv, graphed.scale)
        graphed.pos_t.add_(1)
    for i in range(N):
        graphed.qkv.copy_(qkvs[i])
        graph.replay()
        outs_g.append(graphed.out.clone())
    torch.cuda.synchronize()
    assert int(graphed.pos_t) == p0 + N
    for a, b in zip(outs_e, outs_g):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(eager.kbuf.view(torch.int16), graphed.kbuf.view(torch.int16))
    assert torch.equal(eager.vbuf.view(torch.int16), graphed.vbuf.view(torch.int16))


@pytest.mark.parametrize("pos", [CAP, CAP + 5, -1])
def test_pos_outside_the_cache_writes_nothing(pos):
    case = Case(8, 2, 128, torch.float16, pos, seed=2)
    before_k, before_v, before_out = case.kbuf.clone(), case.vbuf.clone(), case.out.clone()
    case.run()
    torch.cuda.synchronize()
    assert torch.equal(case.kbuf.view(torch.int16), before_k.view(torch.int16))  # the cache and the guard band after it
    assert torch.equal(case.vbuf.view(torch.int16), before_v.view(torch.int16))
    assert torch.equal(case.out.view(torch.int16), before_out.view(torch.int16))


def test_module_rejects_mismatched_cuda_tensors():
    case = Case(8, 2, 64, torch.float16, 5)
    with pytest.raises(RuntimeError, match="k_cache, v_cache and out must have qkv's dtype"):
        _quant_cuda().attn_decode(case.qkv, case.pos_t, case.cos, case.sin, case.kc, case.vc, case.out.float().half().to(torch.bfloat16),
                                  8, 2, 0.125)
    with pytest.raises(RuntimeError, match="rope_cos must be a CUDA tensor"):
        _quant_cuda().attn_decode(case.qkv, case.pos_t, case.cos.cpu(), case.sin, case.kc, case.vc, case.out, 8, 2, 0.125)
