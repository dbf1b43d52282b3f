"""GPU tests of the Fisher information: quant_cuda.fisher_accumulate (sqllm_fisher_accumulate, csrc/fisher.cuh) against an fp64
truth per element, its reproducibility, its argument checks, and quantize.fisher_information on tiny Llama models up to a
quantized, saved and reloaded checkpoint.

Truth and bound (fp64 torch on the GPU, as in lut_grad_ref.py): per sample s, g_s = dy_s^T x_s and A_s = |dy_s|^T |x_s|; then
    F = F_old + sum_s g_s^2,     |F^ - F| <= sum_s (2 e A_s |g_s| + e^2 A_s^2) + e (F_old + F) + eta
with e = E_ACC = 2^-20: each g_s is kept to e A_s (exact 16-bit products, 64-row chunks promoted into fp32 sums), which moves
g_s^2 by at most 2 e A_s |g_s| + e^2 A_s^2; the fp32 squares, their sum and the final add round by a few u of F_old + F; eta
covers squares that fall below fp32's normal range."""
import types

import pytest
import torch

import squeezellm_b200.checkpoint as ck
import squeezellm_b200.quantize as qz
from squeezellm_b200.quant import QuantLinearLUT, quant_cuda
from util import E_ACC

pytestmark = pytest.mark.gpu
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
SHAPES_7B = [(4096, 4096), (11008, 4096), (4096, 11008)]  # [out, in]
SHAPES_RAGGED = [(8, 8), (136, 264), (1000, 520), (8, 11008)]
SEQ = [1, 17, 63, 64, 65, 129, 512, 2048]
SAMPLES = [1, 2, 5, 16]


def make_data(S, T, K, N, dtype, seed=0):
    """x [S T, K], dy [S T, N] in dtype: rows of N(0, 1) scaled by 10^U(-3, 2) (x) and 10^U(-2, 1) (dy), three x channels x100, a
    zero row; sample 1 cancels (its second half repeats the first half's x with dy negated: g_1 = 0); in bf16 sample 0's x is
    scaled by 1e6 and the last sample's dy by 1e-6, magnitudes fp16 cannot hold."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rows = S * T
    x = torch.randn(rows, K, device="cuda", generator=gen, dtype=torch.float64)
    dy = torch.randn(rows, N, device="cuda", generator=gen, dtype=torch.float64)
    x *= 10.0 ** (torch.rand(rows, 1, device="cuda", generator=gen, dtype=torch.float64) * 5 - 3)
    dy *= 10.0 ** (torch.rand(rows, 1, device="cuda", generator=gen, dtype=torch.float64) * 3 - 2)
    x[:, [min(5, K - 1), K // 2, K - 1]] *= 100.0
    x[rows // 2] = 0.0
    if S >= 2 and T >= 2:
        h = T // 2
        x[T + h:T + 2 * h] = x[T:T + h]
        dy[T + h:T + 2 * h] = -dy[T:T + h]
        if T % 2:
            x[2 * T - 1] = 0.0
    if dtype == torch.bfloat16:
        x[:T] *= 1e6
        dy[(S - 1) * T:] *= 1e-6
    else:
        x.clamp_(-60000.0, 60000.0)
    return x.to(dtype).contiguous(), dy.to(dtype).contiguous()


def truth(x, dy, T, f_old):
    """(F, bound) in fp64 for the exact 16-bit values the kernel sees."""
    rows, K = x.shape
    N = dy.shape[1]
    S = rows // T
    xd, dyd = x.double().reshape(S, T, K), dy.double().reshape(S, T, N)
    F = f_old.double().clone()
    B = torch.zeros_like(F)
    for s in range(S):
        g = dyd[s].t() @ xd[s]
        A = dyd[s].abs().t() @ xd[s].abs()
        F += g * g
        B += 2 * E_ACC * A * g.abs() + E_ACC * E_ACC * A * A
        del g, A
    B += E_ACC * (f_old.double() + F) + S * 2.0 ** -126
    return F, B


def check(got, F, B, what):
    err = (got.double() - F).abs()
    ratio = float((err / B).max())
    assert ratio <= 1.0, f"{what}: max |err| / bound = {ratio:.3g}"


def run_case(N, K, T, S, dt, seed):
    x, dy = make_data(S, T, K, N, DT[dt], seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 99)
    f_old = torch.rand(N, K, device="cuda", generator=gen) * 1e-3
    f = f_old.clone()
    quant_cuda.fisher_accumulate(x, dy, f, T)
    F, B = truth(x, dy, T, f_old)
    check(f, F, B, f"{dt} [{N}, {K}] T={T} S={S}")
    if S >= 2 and T >= 2:  # the cancelling sample contributes (almost) nothing
        f1 = torch.zeros(N, K, device="cuda")
        quant_cuda.fisher_accumulate(x[T:2 * T], dy[T:2 * T], f1, T)
        F1, B1 = truth(x[T:2 * T], dy[T:2 * T], T, torch.zeros_like(f1))
        check(f1, F1, B1, f"{dt} [{N}, {K}] T={T} cancelling sample")


RAGGED_CASES = [(N, K, T, SAMPLES[(i + j) % 4]) for i, (N, K) in enumerate(SHAPES_RAGGED) for j, T in enumerate(SEQ)]
BIG_CASES = [(N, K, T, S) for (N, K) in SHAPES_7B for (T, S) in [(2048, 2), (512, 5), (65, 16), (1, 16)]]


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("N,K,T,S", RAGGED_CASES)
def test_ragged_shapes(N, K, T, S, dt):
    run_case(N, K, T, S, dt, seed=N + K + T)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("N,K,T,S", BIG_CASES)
def test_7b_shapes(N, K, T, S, dt):
    run_case(N, K, T, S, dt, seed=T + S)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_reproducible_across_calls_streams_and_graphs(dt):
    N, K, T, S = 1000, 520, 129, 5
    x, dy = make_data(S, T, K, N, DT[dt], 7)
    f_old = torch.rand(N, K, device="cuda")
    a, b = f_old.clone(), f_old.clone()
    quant_cuda.fisher_accumulate(x, dy, a, T)
    quant_cuda.fisher_accumulate(x, dy, b, T)
    assert torch.equal(a, b)

    outs = [f_old.clone() for _ in range(3)]
    streams = [torch.cuda.Stream() for _ in range(3)]
    torch.cuda.synchronize()
    for st, o in zip(streams, outs):
        with torch.cuda.stream(st):
            quant_cuda.fisher_accumulate(x, dy, o, T)
    torch.cuda.synchronize()
    assert all(torch.equal(o, a) for o in outs)

    sx, sdy, sf = torch.zeros_like(x), torch.zeros_like(dy), torch.zeros_like(f_old)
    graph = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        quant_cuda.fisher_accumulate(sx, sdy, sf, T)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(st)
    with torch.cuda.graph(graph):
        quant_cuda.fisher_accumulate(sx, sdy, sf, T)
    x2, dy2 = make_data(S, T, K, N, DT[dt], 8)
    sx.copy_(x2)
    sdy.copy_(dy2)
    sf.copy_(f_old)
    graph.replay()
    want = f_old.clone()
    quant_cuda.fisher_accumulate(x2, dy2, want, T)
    torch.cuda.synchronize()
    assert torch.equal(sf, want)


def test_argument_checks():
    h = dict(device="cuda", dtype=torch.float16)
    x, dy, f = torch.zeros(8, 16, **h), torch.zeros(8, 24, **h), torch.zeros(24, 16, device="cuda")
    quant_cuda.fisher_accumulate(x, dy, f, 4)
    bad = [
        ((x.cpu(), dy, f, 4), "fisher_accumulate: x must be a contiguous CUDA tensor"),
        ((x, dy.cpu(), f, 4), "fisher_accumulate: dy must be a contiguous CUDA tensor"),
        ((x, dy, f.cpu(), 4), "fisher_accumulate: fisher must be a contiguous CUDA tensor"),
        ((torch.zeros(16, 8, **h).t(), dy, f, 4), "fisher_accumulate: x must be a contiguous CUDA tensor"),
        ((x.float(), dy, f, 4), "fisher_accumulate: x must be fp16 or bf16"),
        ((x, dy.bfloat16(), f, 4), "fisher_accumulate: dy must have x's dtype"),
        ((x, dy, f.half(), 4), "fisher_accumulate: fisher must be fp32"),
        ((x, dy[:4], f, 4), "fisher_accumulate: dy has 4 rows but x has 8"),
        ((x, dy, f.t().contiguous(), 4), r"fisher_accumulate: fisher must be \[out=24, in=16\]"),
        ((x.reshape(2, 4, 16), dy, f, 4), r"fisher_accumulate: x must be \[rows, in\] and dy \[rows, out\]"),
        ((x, dy, f, 3), "fisher_accumulate: seq_len=3 must be >= 1 and divide the 8 rows of x"),
        ((x, dy, f, 0), "fisher_accumulate: seq_len=0 must be >= 1"),
        ((x[:, :12].contiguous(), dy, f[:, :12].contiguous(), 4), "in_features=12 must be a positive multiple of 8"),
        ((x[:0], dy[:0], f, 4), "x must have 1 to 2\\^31-1 rows"),
    ]
    for args, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            quant_cuda.fisher_accumulate(*args)


def tiny_llama(dtype, seed=0):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=97, max_position_embeddings=64)
    torch.manual_seed(seed)
    return cfg, transformers.LlamaForCausalLM(cfg).eval().to(dtype).cuda()


def batches(B=3, T=24, n=2, seed=5):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randint(0, 97, (B, T), device="cuda", generator=gen) for _ in range(n)]


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_fisher_information_on_tiny_llama(dt, monkeypatch):
    _, model = tiny_llama(DT[dt])
    params = {n: p.detach().clone() for n, p in model.named_parameters()}
    seen = []

    def spy(x, dy, fisher, seq_len):
        before = fisher.clone()
        quant_cuda.fisher_accumulate(x, dy, fisher, seq_len)
        seen.append((x.clone(), dy.clone(), seq_len, before, fisher.clone()))

    monkeypatch.setattr(qz, "quant_cuda", types.SimpleNamespace(fisher_accumulate=spy))
    F = qz.fisher_information(model, batches())
    names = [n for n in ck.find_linear_layers(model) if n != "lm_head"]
    assert sorted(F) == sorted(f"{n}.weight" for n in names)
    assert len(seen) == 2 * len(names)
    for x, dy, T, before, after in seen:
        assert x.dtype == dy.dtype == DT[dt] and T == 24 and x.shape[0] == 72
        want, bound = truth(x, dy, T, before)
        check(after, want, bound, f"{dt} layer call")
    for n in names:
        f = F[f"{n}.weight"]
        assert f.dtype == torch.float32 and f.shape == ck.find_linear_layers(model)[n].weight.shape
        assert torch.isfinite(f).all() and bool((f > 0).any()), n
    for n, p in model.named_parameters():
        assert torch.equal(p.detach(), params[n]) and p.grad is None and p.requires_grad, n


def test_pipeline_fisher_quantize_save_load(tmp_path):
    cfg, model = tiny_llama(torch.float16)
    fisher = qz.fisher_information(model, batches())
    names = [n for n in ck.find_linear_layers(model) if n != "lm_head"]
    numvals = qz.quantize_model(model, fisher, 4, outlier_range=3.0, sensitivity=0.45)
    assert sorted(numvals) == sorted(names) and all(v > 0 for v in numvals.values())
    ids = batches(1, 12, 1)[0]
    with torch.no_grad():
        logits = model(ids).logits.float()
    assert torch.isfinite(logits).all()
    path = str(tmp_path / "model.pt")
    ck.save_checkpoint(model, path, 4)
    import transformers
    torch.manual_seed(0)
    fresh = transformers.LlamaForCausalLM(cfg).eval().half()
    ck.load_checkpoint(fresh, path)
    fresh = fresh.cuda()
    with torch.no_grad():
        assert torch.equal(fresh(ids).logits.float(), logits)


def test_fisher_weighting_lowers_the_weighted_error():
    """Dense-only 4-bit: per layer, sum F (W - dequantize())^2 with the Fisher codebook is <= that of the uniform-weight codebook
    (exact weighted k-means minimises exactly this).  A transposed F on the square layers would break it."""
    _, model = tiny_llama(torch.float16)
    fisher = qz.fisher_information(model, batches(4, 32, 2))
    for name, lin in ck.find_linear_layers(model).items():
        if name == "lm_head":
            continue
        f = fisher[f"{name}.weight"]
        w = lin.weight.detach().float()
        err = {}
        for kind, s in (("fisher", f), ("uniform", torch.ones_like(f))):
            q = qz.quantize_linear(lin, s, 4)
            err[kind] = float((f.double() * (w.double() - q.dequantize(torch.float32).double()) ** 2).sum())
        assert err["fisher"] <= err["uniform"] * (1 + 1e-6), (name, err)
