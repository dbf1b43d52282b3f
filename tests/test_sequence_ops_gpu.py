"""GPU tests of the sequence kernel's ops (sqllm_sequence_create_ops, DecodeSequence.matvec(norm=, up=, residual=)): a LLaMA decoder
layer's quantized part as one persistent launch -

    o  = o_proj(a) + h                         (h: an external residual)
    gu = gate_up(rmsnorm(o))                   (stacked gate | up; or gate and up as two items)
    d  = down(silu(gu[:I]) * gu[I:]) + o
    q  = qkv(rmsnorm(d))

Every item is exported and checked per element against fp64 truth computed from the exported values of its own sources, so errors
do not compound: |got - want| <= r |want| + eta + (1 + r) e S, with S = sum_k |W_ck| |x'_k| + |bias_c| + |res_c| plus the transform's
rounding (u_XT + its fp32 terms, transform_fp32_rel) sum_k |W_ck| |x'_k| (x' in fp64 from the sources; e, r, eta as in tests/util.py)."""
import numpy as np
import pytest
import torch

from test_sequence_gpu import _module
from util import E_ACC, OUT_ROUNDING, U32, abs_sum, bound_ratio, orc

pytestmark = pytest.mark.gpu

EPS = 1e-5
TDT = {"exact": torch.float16, "fp16": torch.float16, "bf16": torch.bfloat16}


def _round(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dt).double().numpy()


def _layer(bits, K, N, kind, seed, scale=1.0):
    """kind: "dense" (LUT only), "csr" (CSR outliers and dense rows), "rows" (dense rows only)."""
    sp, topX = {"dense": (0.0, 0), "csr": (0.0045 if K * N > 1e7 else 0.02, 4), "rows": (0.0, 33)}[kind]
    L = orc.make_layer(bits, K, N, sparsity=sp, topX=topX, seed=seed, nonzero_full_rows=topX > 0)
    L["lookup_table"] = (L["lookup_table"] * (50.0 * scale / np.sqrt(K))).astype(np.float32)   # |y| ~ |x|
    return L, _module(L, bits, K, N, topX)


def _lut_view(L, mode):
    if mode != "fp16":
        return L
    LL = dict(L)
    LL["lookup_table"] = L["lookup_table"].astype(np.float16).astype(np.float32)
    return LL


def transform_fp32_rel(transform, K):
    """Relative error of the kernel's fp32 steps before x' is rounded (in units of u = 2^-24, plus one u for the oracle's fp32 copy of
    x').  RMSNorm: S is a chain of 2 ceil(K / 4096) * 4 fmas per thread, the warp's 5-level xor tree and 16 warp sums (each rounding
    at most u of the partial sum, all terms >= 0), so S carries at most n_S u; r = 1/sqrt(S/K + eps) halves that and adds the
    division, the add, the sqrt and the reciprocal (4 u); x r and the product with the weight add 2 u.  SiLU gating: expf (2 ulp), the
    add, the division and the product with u (4 u)."""
    if transform is None:
        return 0.0
    if transform == "rms":
        n_s = 8 * -(-K // 4096) + 5 + 16
        return (n_s / 2 + 4 + 2 + 1) * U32
    assert transform == "silu"
    return (2 + 4 + 1) * U32


def _check(got, L, xp, mode, dt, bias=None, res=None, what="", transform=None):
    """got: the item's output (fp64 of its XT values); xp: the item's input after its transform ("rms", "silu" or None), in fp64 from
    the exported sources."""
    LL = _lut_view(L, mode)
    r_out, eta = OUT_ROUNDING[str(dt).split(".")[1]]
    x32 = xp.astype(np.float32).reshape(1, -1)
    want = orc.forward_f64(LL, x32, mul_init=None if bias is None else bias[None, :]).reshape(-1)
    S = abs_sum(LL, x32, bias).reshape(-1)
    if res is not None:
        want = want + res
        S = S + np.abs(res)
    if transform is not None:   # x' = round_XT(x'_true (1 + fp32 error)): u_XT + the fp32 terms of each |x'_k|, folded into e S
        rel = (1 + r_out) * transform_fp32_rel(transform, xp.size) + r_out
        S = S + rel / E_ACC * abs_sum(LL, x32).reshape(-1)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    ratio = bound_ratio(got, want, S, r=r_out, eta=eta)
    assert ratio <= 1.0, f"{what}: bound ratio {ratio:.3f}"
    return ratio


def rmsnorm64(x, w, eps):
    return w * (x / np.sqrt(np.mean(x * x) + eps))


def silu_mul64(g, u):
    with np.errstate(over="ignore"):
        return g / (1.0 + np.exp(-g)) * u


class Block:
    """The four (or five, unfused) items of a decoder layer's quantized part, their oracle layers and their op data."""

    def __init__(self, bits, H, I, Q, kind, mode, fused=True, seed=0):
        self.bits, self.H, self.I, self.Q, self.mode, self.fused = bits, H, I, Q, mode, fused
        self.dt = TDT[mode]
        rng = np.random.default_rng(seed)
        self.o, self.mo = _layer(bits, H, H, kind, seed + 1)
        if fused:
            self.gu, self.mgu = _layer(bits, H, 2 * I, kind, seed + 2)
        else:
            self.g, self.mg = _layer(bits, H, I, kind, seed + 2)
            self.u, self.mu = _layer(bits, H, I, kind, seed + 3)
        self.d, self.md = _layer(bits, I, H, kind, seed + 4)
        self.q, self.mq = _layer(bits, H, Q, kind, seed + 5)
        self.w1 = _round(1.0 + 0.1 * rng.standard_normal(H), self.dt)
        self.w2 = _round(1.0 + 0.1 * rng.standard_normal(H), self.dt)
        self.eps = EPS

    def sequence(self):
        from squeezellm_b200.runtime import DecodeSequence
        dt = self.dt
        seq = DecodeSequence(self.H, "cuda", lut_mode="fp16" if self.mode == "fp16" else "exact", dtype=dt)
        hv, self.h_t = seq.new_input(self.H)
        w1, w2 = (torch.from_numpy(w).to("cuda", dt) for w in (self.w1, self.w2))
        o = seq.matvec(self.mo, seq.input, residual=hv)
        if self.fused:
            gu = seq.matvec(self.mgu, o, norm=(w2, self.eps))
            g, u = gu[0:self.I], gu[self.I:2 * self.I]
            mid = [gu]
        else:
            g = seq.matvec(self.mg, o, norm=(w2, self.eps))
            u = seq.matvec(self.mu, o, norm=(w2, self.eps))
            mid = [g, u]
        d = seq.matvec(self.md, g, up=u, residual=o)
        q = seq.matvec(self.mq, d, norm=(w1, self.eps))
        seq.compile(outputs=[o] + mid + [d, q])
        return seq

    def set_inputs(self, seq, a, h):
        seq.x.copy_(torch.from_numpy(a).to(self.dt))
        self.h_t.copy_(torch.from_numpy(h).to(self.dt))

    def check(self, outs, a, h):
        """outs: the exported vectors (fp64 numpy); a, h: the inputs (already representable)."""
        mode, dt = self.mode, self.dt
        it = iter(outs)
        o = next(it)
        worst = [_check(o, self.o, a, mode, dt, res=h, what="o_proj + h")]
        if self.fused:
            gu = next(it)
            worst.append(_check(gu, self.gu, rmsnorm64(o, self.w2, self.eps), mode, dt, what="gate_up(rmsnorm(o))", transform="rms"))
            g, u = gu[:self.I], gu[self.I:]
        else:
            g, u = next(it), next(it)
            worst.append(_check(g, self.g, rmsnorm64(o, self.w2, self.eps), mode, dt, what="gate(rmsnorm(o))", transform="rms"))
            worst.append(_check(u, self.u, rmsnorm64(o, self.w2, self.eps), mode, dt, what="up(rmsnorm(o))", transform="rms"))
        d = next(it)
        worst.append(_check(d, self.d, silu_mul64(g, u), mode, dt, res=o, what="down(silu(g) u) + o", transform="silu"))
        q = next(it)
        worst.append(_check(q, self.q, rmsnorm64(d, self.w1, self.eps), mode, dt, what="qkv(rmsnorm(d))", transform="rms"))
        return max(worst)


def _vec(n, seed, dt, scale=1.0):
    return _round(orc.make_vec(n, seed=seed).reshape(-1) * scale, dt)


def _run(seq):
    outs = [o.clone() for o in seq.replay()]
    torch.cuda.synchronize()
    return [o.double().cpu().numpy() for o in outs]


SMALL = [(bits, mode, kind) for bits in (4, 3) for mode in ("exact", "fp16", "bf16") for kind in ("dense", "csr", "rows")]


@pytest.mark.parametrize("bits,mode,kind", SMALL, ids=[f"w{b}-{m}-{k}" for b, m, k in SMALL])
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
def test_layer_ops_ragged(bits, mode, kind, fused):
    """Small, ragged shapes: hidden 192 (three strips), intermediate 704, a 200-column last item (a ragged strip)."""
    blk = Block(bits, 192, 704, 200, kind, mode, fused=fused, seed=bits * 10)
    seq = blk.sequence()
    for rep, s in enumerate((1, 1, 2)):   # two replays of the same token, then a new one
        a, h = _vec(192, s, blk.dt), _vec(192, s + 50, blk.dt)
        blk.set_inputs(seq, a, h)
        outs = _run(seq)
        assert not seq.error(), "a bounded in-kernel wait of the sequence gave up"
        blk.check(outs, a, h)
        if rep == 1:
            assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(outs, prev)), "a replay of the same token differs"
        prev = outs


SEVEN_B = [(4, "exact"), (4, "fp16"), (4, "bf16"), (3, "exact")]


@pytest.mark.parametrize("bits,mode", SEVEN_B, ids=[f"w{b}-{m}" for b, m in SEVEN_B])
def test_layer_ops_7b_shapes(bits, mode):
    """A LLaMA-7B decoder layer: 4096 hidden, 11008 intermediate (stacked gate_up 22016, down K = 11008), stacked q/k/v 12288; CSR
    outliers (0.45 %) and dense rows."""
    blk = Block(bits, 4096, 11008, 12288, "csr", mode, seed=bits)
    seq = blk.sequence()
    a, h = _vec(4096, 3, blk.dt), _vec(4096, 4, blk.dt)
    blk.set_inputs(seq, a, h)
    outs = _run(seq)
    assert not seq.error()
    print(f"w{bits} {mode}: worst bound ratio {blk.check(outs, a, h):.3f}")


@pytest.mark.parametrize("mode", ["exact", "bf16"])
@pytest.mark.parametrize("case", ["tiny", "huge", "eps_dominates", "gates", "cancel"])
def test_layer_ops_stress(case, mode):
    """Activations from 1e-3 to 6e4, an eps that dominates the mean square, gates at +-30 and +-1e4, residuals that cancel the
    matvec (o = o_proj(a) + h with h = -round(o_proj(a)))."""
    blk = Block(4, 192, 704, 200, "csr", mode, seed=7)
    if case == "eps_dominates":
        blk.eps = 10.0
    seq = blk.sequence()
    dt = blk.dt
    a, h = _vec(192, 1, dt), _vec(192, 2, dt)
    if case == "tiny":
        a, h = _vec(192, 1, dt, 1e-3), _vec(192, 2, dt, 1e-3)
    elif case == "huge":   # a residual stream up to 6e4; o = o_proj(a) + h stays inside the fp16 range (|o_proj(a)| ~ 3)
        v = orc.make_vec(192, seed=2).reshape(-1).astype(np.float64)
        a, h = _vec(192, 1, dt), _round(v * (6e4 / np.abs(v).max()), dt)
        assert np.abs(h).max() >= 5.9e4
    elif case == "gates":   # gate outputs at +-30 and +-1e4; the up half at 1e-2, so that silu(g) u stays inside the fp16 range
        s = np.full(2 * blk.I, 1e-2, dtype=np.float32)
        s[: blk.I // 2], s[blk.I // 2: blk.I] = 30.0, 1e4
        blk.gu["lookup_table"] = (blk.gu["lookup_table"] * s[:, None]).astype(np.float32)
        blk.mgu.lookup_table.copy_(torch.from_numpy(blk.gu["lookup_table"]))   # (the outliers stay O(1))
    elif case == "cancel":
        blk.set_inputs(seq, a, np.zeros(192))
        h = -_run(seq)[0]   # o = round(o_proj(a) - round(o_proj(a))): what is left is the first rounding's error
    blk.set_inputs(seq, a, h)
    outs = _run(seq)
    assert not seq.error()
    blk.check(outs, a, h)
    if case == "cancel":
        assert np.abs(outs[0]).max() < 1e-2 * np.abs(h).max()
    if case == "gates":
        g = outs[1][: blk.I]
        assert np.abs(g).max() > 1e3


def test_layer_ops_in_cuda_graph_with_new_inputs():
    """The ops run inside a captured graph: new inputs through the static buffers, each replay checked; bit-identical to eager runs."""
    from squeezellm_b200.runtime import GraphedDecodeStep
    blk = Block(4, 192, 704, 200, "csr", "exact", seed=11)
    seq = blk.sequence()
    runner = GraphedDecodeStep(lambda x: seq.replay()[-1], seq.x, warmup=2, static_input=True)
    for s in (1, 2, 3):
        a, h = _vec(192, s, blk.dt), _vec(192, s + 9, blk.dt)
        blk.h_t.copy_(torch.from_numpy(h).to(blk.dt))
        runner(torch.from_numpy(a).to(blk.dt))
        outs = [o.double().cpu().numpy() for o in seq.outputs]
        blk.check(outs, a, h)
        blk.set_inputs(seq, a, h)
        eager = _run(seq)
        assert all(np.array_equal(x, y) for x, y in zip(outs, eager)), "graph replay and eager run differ"
    assert not seq.error()


def test_plain_matvecs_unchanged_by_the_ops_keywords():
    """A sequence without any op takes the plain kernel: the same bits with or without an all-None ops list through quant_cuda."""
    from squeezellm_b200.quant import quant_cuda as qc
    L, m = _layer(4, 256, 256, "csr", 5)
    x = torch.from_numpy(_vec(256, 1, torch.float16)).cuda().half()
    item = (m.qweight, m.lookup_table, 4, None, *m._sparse_args(), -1, 0, x, 1, 256)
    outs = []
    for ops in (None, [None]):
        y = torch.zeros(256, dtype=torch.float16, device="cuda")
        h = qc.sequence_create([item], [(0, y)], "exact", ops=ops)
        qc.sequence_run(h)
        torch.cuda.synchronize()
        qc.sequence_destroy(h)
        outs.append(y.clone())
    assert torch.equal(outs[0], outs[1])


def test_quant_cuda_range_checks_of_ops():
    """The op checks that need the items' lengths and the tensors' addresses, through quant_cuda."""
    from squeezellm_b200.quant import quant_cuda as qc
    _, m0 = _layer(4, 256, 256, "dense", 1)
    _, m1 = _layer(4, 256, 512, "dense", 2)
    x = torch.zeros(256, dtype=torch.float16, device="cuda")
    it0 = (m0.qweight, m0.lookup_table, 4, None, None, None, None, None, None, -1, 0, x, 1, 256)
    it1 = (m1.qweight, m1.lookup_table, 4, None, None, None, None, None, None, 0, 0, None, 1, 512)
    it2 = (m0.qweight, m0.lookup_table, 4, None, None, None, None, None, None, 1, 0, None, 1, 256)
    w = torch.ones(264, dtype=torch.float16, device="cuda")
    for ops, frag in [
        ([None, None, (2, None, 0.0, 1, 300, -1, 0, None)], "item 2: x2 reads [300, 556) of item 1's 512 outputs"),
        ([None, (0, None, 0.0, -1, 0, 0, 0, None), None], "item 1: residual reads [0, 512) of item 0's 256 outputs"),
        ([None, None, (1, w[4:260], 1e-6, -1, 0, -1, 0, None)], "item 2: norm_weight must be a 16-byte aligned fp16 vector"),
        ([None, None, (0, None, 0.0, -1, 0, -1, 0, w[2:258])], "item 2: res_ext must be a 16-byte aligned fp16 vector"),
    ]:
        with pytest.raises(RuntimeError, match=frag.replace("[", r"\[").replace("(", r"\(").replace(")", r"\)")):
            qc.sequence_create([it0, it1, it2], [], "exact", ops=ops)
