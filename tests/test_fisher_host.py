"""CPU tests of quantize.fisher_information's semantics: quant_cuda.fisher_accumulate is replaced by an fp64 torch statement of
its formula, and the model is a tiny random LlamaForCausalLM in fp64, so the Python layer (hooks, loss, sample boundaries, state
restoration) is checked exactly against per-sequence autograd.  The kernel itself is checked in test_fisher_gpu.py."""
import types

import pytest
import torch

import squeezellm_b200.quantize as qz
from squeezellm_b200.checkpoint import find_linear_layers

transformers = pytest.importorskip("transformers")


def fake_accumulate(x, dy, fisher, seq_len):
    """fisher += sum_s (dy_s^T x_s)^2 in fp64: sqllm_fisher_accumulate's formula without its rounding."""
    assert x.is_contiguous() and dy.is_contiguous() and x.shape[0] == dy.shape[0] and x.shape[0] % seq_len == 0
    assert fisher.shape == (dy.shape[1], x.shape[1])
    xs = x.double().reshape(-1, seq_len, x.shape[1])
    dys = dy.double().reshape(-1, seq_len, dy.shape[1])
    g = torch.einsum("stn,stk->snk", dys, xs)
    fisher += (g * g).sum(0).to(fisher.dtype)


@pytest.fixture
def fake(monkeypatch):
    calls = []

    def rec(x, dy, fisher, seq_len):
        calls.append((x.shape, dy.shape, seq_len))
        fake_accumulate(x, dy, fisher, seq_len)

    monkeypatch.setattr(qz, "quant_cuda", types.SimpleNamespace(fisher_accumulate=rec))
    monkeypatch.setattr(qz, "_FISHER_DTYPES", (torch.float64,))
    return calls


def tiny_llama(seed=0):
    cfg = transformers.LlamaConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=61, max_position_embeddings=32, attn_implementation="eager")
    torch.manual_seed(seed)
    return transformers.LlamaForCausalLM(cfg).double().eval()


def tokens(B, T, seed=1):
    return torch.randint(0, 61, (B, T), generator=torch.Generator().manual_seed(seed))


def per_sequence_grads(model, ids):
    """[{name: weight.grad of the loss of ids[b] alone}] for every row b (sum of its next-token cross-entropies)."""
    names = [n for n in find_linear_layers(model) if n != "lm_head"]
    lin = find_linear_layers(model)
    out = []
    for b in range(ids.shape[0]):
        model.zero_grad(set_to_none=True)
        logits = model(ids[b:b + 1]).logits
        loss = torch.nn.functional.cross_entropy(logits[0, :-1], ids[b, 1:], reduction="sum")
        loss.backward()
        out.append({n: lin[n].weight.grad.clone() for n in names})
    model.zero_grad(set_to_none=True)
    return out


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_equals_sum_of_per_sequence_squared_gradients(fake):
    model = tiny_llama()
    ids = tokens(4, 9)
    grads = per_sequence_grads(model, ids)
    F = qz.fisher_information(model, [ids])
    names = [n for n in find_linear_layers(model) if n != "lm_head"]
    assert sorted(F) == sorted(f"{n}.weight" for n in names)
    assert len(fake) == len(names) and all(c[2] == 9 and c[0][0] == 36 for c in fake)
    for n in names:
        want = sum(g[n] ** 2 for g in grads)
        assert F[f"{n}.weight"].dtype == torch.float64
        assert rel(F[f"{n}.weight"], want) < 1e-12, n
        # the square of the batch gradient is a different quantity
        assert rel((sum(g[n] for g in grads)) ** 2, want) > 0.1, n


def test_batching_does_not_change_the_result(fake):
    model = tiny_llama()
    ids = tokens(4, 7, seed=3)
    one = qz.fisher_information(model, [ids])
    four = qz.fisher_information(model, [ids[b:b + 1] for b in range(4)])
    assert sorted(one) == sorted(four)
    for k in one:
        assert rel(four[k], one[k]) < 1e-12, k


def test_layers_restricts_the_result(fake):
    model = tiny_llama()
    sel = ["model.layers.0.self_attn.q_proj", "model.layers.1.mlp.down_proj"]
    F = qz.fisher_information(model, [tokens(2, 5)], layers=sel)
    assert sorted(F) == sorted(f"{n}.weight" for n in sel)
    assert len(fake) == 2
    with pytest.raises(ValueError, match="lm_head"):
        qz.fisher_information(model, [tokens(2, 5)], layers=["lm_head"])


def _state(model):
    return ([(n, p.requires_grad, None if p.grad is None else p.grad.clone()) for n, p in model.named_parameters()],
            model.training, sum(len(m._forward_hooks) for m in model.modules()))


def _check_state(model, before):
    params, training, hooks = _state(model)
    assert training == before[1] and hooks == before[2] == 0
    for (n, rg, g), (n2, rg2, g2) in zip(before[0], params):
        assert n == n2 and rg == rg2, n
        assert (g is None and g2 is None) or torch.equal(g, g2), n


def _prepare(model):
    model.train()
    model.model.layers[0].mlp.up_proj.weight.requires_grad_(False)
    model.model.layers[1].mlp.gate_proj.weight.grad = torch.full_like(model.model.layers[1].mlp.gate_proj.weight, 0.5)


def test_state_restored_after_a_run(fake):
    model = tiny_llama()
    _prepare(model)
    before = _state(model)
    qz.fisher_information(model, [tokens(2, 6)])
    _check_state(model, before)


def test_state_restored_after_an_error_mid_backward(monkeypatch):
    n = [0]

    def boom(x, dy, fisher, seq_len):
        n[0] += 1
        if n[0] == 3:
            raise RuntimeError("fake failure")
        fake_accumulate(x, dy, fisher, seq_len)

    monkeypatch.setattr(qz, "quant_cuda", types.SimpleNamespace(fisher_accumulate=boom))
    monkeypatch.setattr(qz, "_FISHER_DTYPES", (torch.float64,))
    model = tiny_llama()
    _prepare(model)
    before = _state(model)
    with pytest.raises(RuntimeError, match="fake failure"):
        qz.fisher_information(model, [tokens(2, 6)])
    _check_state(model, before)


def test_a_layer_run_twice_raises(fake):
    model = tiny_llama()
    model.model.layers[1].mlp.down_proj = model.model.layers[0].mlp.down_proj
    before = _state(model)
    with pytest.raises(ValueError, match=r"layer model\.layers\.\d\.mlp\.down_proj ran more than once"):
        qz.fisher_information(model, [tokens(1, 4)])
    _check_state(model, before)


def test_rejections(fake, monkeypatch):
    model = tiny_llama()
    with pytest.raises(ValueError, match="T >= 2"):
        qz.fisher_information(model, [tokens(2, 1)])
    monkeypatch.setattr(qz, "_FISHER_DTYPES", (torch.float16, torch.bfloat16))
    with pytest.raises(ValueError, match=r"layer model\.layers\.0\.self_attn\.q_proj is torch.float64; fp16 or bf16"):
        qz.fisher_information(model, [tokens(2, 4)])
    monkeypatch.setattr(qz, "_FISHER_DTYPES", (torch.float64,))
    model.model.layers[0].mlp.down_proj = torch.nn.Linear(60, 32, bias=False).double()
    with pytest.raises(ValueError, match=r"layer model\.layers\.0\.mlp\.down_proj is 60 -> 32; in and out features must be multiples of 8"):
        qz.fisher_information(model, [tokens(2, 4)])


def test_rejects_non_finite(monkeypatch):
    def nan(x, dy, fisher, seq_len):
        fisher += float("nan")

    monkeypatch.setattr(qz, "quant_cuda", types.SimpleNamespace(fisher_accumulate=nan))
    monkeypatch.setattr(qz, "_FISHER_DTYPES", (torch.float64,))
    with pytest.raises(ValueError, match="layer model.layers.0.self_attn.q_proj is not finite"):
        qz.fisher_information(tiny_llama(), [tokens(1, 4)])
