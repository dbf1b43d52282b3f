"""CPU tests of runtime.SequenceDecoder's host side: every rejection (ValueError naming the reason, before any device allocation) on
models built on the CPU from HF configs, DecodeSequence's checks of the tensors it is given to read (x=, new_input(tensor=)), and the
layout of the decoder's plan: its sequences, their items and ops, and which buffer feeds which."""
import pytest
import torch

from util import orc

transformers = pytest.importorskip("transformers")

from squeezellm_b200 import checkpoint as ck  # noqa: E402
from squeezellm_b200.quant import QuantLinearLUT  # noqa: E402
from squeezellm_b200.runtime import AttnPlan, DecodeSequence, SeqPlan, SequenceDecoder, decoder_plan  # noqa: E402

SMALL = dict(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1, vocab_size=128,
             max_position_embeddings=64)


def quantized(cls="LlamaForCausalLM", cfg_cls="LlamaConfig", dtype=torch.float16, bits=4, quant_head=False, skip=(), **kw):
    """A model of `cls` on the CPU whose linear layers (but those in `skip`) are QuantLinearLUT layers of `bits` bits
    (oracle.make_layer, no outliers)."""
    torch.manual_seed(0)
    model = getattr(transformers, cls)(getattr(transformers, cfg_cls)(**dict(SMALL, **kw))).to(dtype).eval()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    quant = [n for n in ck.find_linear_layers(model) if (quant_head or n != "lm_head") and n not in skip]
    for i, name in enumerate(sorted(quant)):
        lin = model.get_submodule(name)
        L = orc.make_layer(bits, lin.in_features, lin.out_features, sparsity=0.0, topX=0, seed=i, bias=lin.bias is not None)
        del state[name + ".weight"]
        for k in ("qweight", "lookup_table", "bias"):
            if L.get(k) is not None:
                state[f"{name}.{k}"] = torch.from_numpy(L[k])
    ck.load_quantized(model, state, bits, skip=tuple(n for n in ck.find_linear_layers(model) if n not in quant))
    return model


def test_a_cpu_model_is_rejected_before_anything_is_stacked():
    model = quantized()
    with pytest.raises(ValueError, match=r"the model must be on one GPU \(its tensors are on \['cpu'\]\)"):
        SequenceDecoder(model, 32)
    assert all(m._sibling_group is None for m in model.modules() if isinstance(m, QuantLinearLUT))


def _mixed_bits():
    model = quantized()
    m3 = quantized(bits=3)
    model.model.layers[1].mlp.down_proj = m3.model.layers[1].mlp.down_proj
    return model


def _trained():
    model = quantized()
    model.model.layers[0].self_attn.o_proj.train_codebook(lookup_table=True)
    return model


REJECT = [
    (lambda: transformers.GPT2LMHeadModel(transformers.GPT2Config(n_layer=1, n_embd=64, n_head=2, vocab_size=64)),
     "GPT2LMHeadModel is not supported"),
    (lambda: quantized(dtype=torch.float32), "the model is torch.float32; only float16 and bfloat16"),
    (lambda: quantized(skip=("model.layers.1.mlp.up_proj",)), "layers.1.mlp.up_proj is a Linear, not a QuantLinearLUT"),
    (_mixed_bits, r"mixed bit widths \[3, 4\]"),
    (_trained, r"layers.0.self_attn.o_proj is being trained \(train_codebook: lookup_table\)"),
    (lambda: quantized("MistralForCausalLM", "MistralConfig", sliding_window=16), r"sliding_window=16 < max_len=32"),
    (lambda: quantized("Qwen2ForCausalLM", "Qwen2Config", use_sliding_window=True, sliding_window=16, max_window_layers=0),
     "sliding-window attention is not supported"),
    (lambda: quantized(num_attention_heads=8, num_key_value_heads=2), "head_dim=32 is not 64 or 128"),
    (lambda: quantized(head_dim=256), "head_dim=256 is not 64 or 128"),
    (lambda: quantized(hidden_act="gelu"), "hidden_act='gelu' is not silu"),
]


@pytest.mark.parametrize("make,frag", REJECT, ids=["class", "fp32", "dense_layer", "mixed_bits", "trained", "mistral_window",
                                                   "qwen2_window", "head_dim_32", "head_dim_256", "act"])
def test_rejections(make, frag):
    model = make()
    with pytest.raises(ValueError, match=frag):
        SequenceDecoder(model, 32)
    with pytest.raises(ValueError, match=frag):
        decoder_plan(model, 32)


@pytest.mark.parametrize("max_len", [0, -3, 2.5])
def test_rejects_a_bad_max_len(max_len):
    with pytest.raises(ValueError, match="max_len must be a positive int"):
        SequenceDecoder(quantized(), max_len)


def test_accepts_a_mistral_window_that_covers_max_len():
    plan = decoder_plan(quantized("MistralForCausalLM", "MistralConfig", sliding_window=32), 32)
    assert len(plan) == 5


# ---- the plan ----
def _group_layer(module, name):
    return getattr(module, name)._sibling_group[0].layer


@pytest.mark.parametrize("quant_head", [False, True])
def test_plan_layout(quant_head):
    model = quantized(quant_head=quant_head, num_hidden_layers=3)
    plan = decoder_plan(model, 32)
    layers = model.model.layers
    H, I = 256, 512
    kinds = [type(s).__name__ for s in plan]
    assert kinds == ["SeqPlan", "AttnPlan", "SeqPlan", "AttnPlan", "SeqPlan", "AttnPlan", "SeqPlan"]
    pro = plan[0]
    assert (pro.name, pro.x, pro.h, pro.outputs) == ("prologue", "embed", None, ["qkv"])
    (it,) = pro.items
    assert (it.name, it.x, it.up, it.residual) == ("qkv", ("x", 0, H), None, None)
    assert it.layer is _group_layer(layers[0].self_attn, "q_proj") and it.norm is layers[0].input_layernorm
    assert it.layer.outfeatures == 256 + 2 * 128
    for i in range(3):
        attn, seq = plan[1 + 2 * i], plan[2 + 2 * i]
        assert attn == AttnPlan(i, ("prologue" if i == 0 else f"layer{i - 1}", "qkv"))
        assert isinstance(seq, SeqPlan) and seq.name == f"layer{i}" and seq.x == "attn"
        assert seq.h == ("embed" if i == 0 else (f"layer{i - 1}", "d"))
        got = [(t.name, t.x, t.up, t.residual) for t in seq.items]
        want = [("o", ("x", 0, H), None, ("h", 0, H)), ("gu", ("o", 0, H), None, None), ("d", ("gu", 0, I), ("gu", I, I), ("o", 0, H))]
        L = layers[i]
        layer_of = [L.self_attn.o_proj, _group_layer(L.mlp, "gate_proj"), L.mlp.down_proj]
        norm_of = [None, L.post_attention_layernorm, None]
        if i < 2:
            want.append(("qkv", ("d", 0, H), None, None))
            layer_of.append(_group_layer(layers[i + 1].self_attn, "q_proj"))
            norm_of.append(layers[i + 1].input_layernorm)
            assert seq.outputs == ["d", "qkv"]
        elif quant_head:
            want.append(("logits", ("d", 0, H), None, None))
            layer_of.append(model.lm_head)
            norm_of.append(model.model.norm)
            assert seq.outputs == ["logits"]
        else:
            assert seq.outputs == ["d"]
        assert got == want
        assert all(t.layer is m for t, m in zip(seq.items, layer_of))
        assert all(t.norm is n for t, n in zip(seq.items, norm_of))


# ---- DecodeSequence reading tensors it does not own ----
def test_sequence_reads_the_given_tensors():
    x = torch.zeros(64, dtype=torch.float16)
    seq = DecodeSequence(64, "cpu", x=x)
    assert seq.x is x
    h = torch.ones(128, dtype=torch.float16)
    v, t = seq.new_input(128, tensor=h)
    assert t is h and seq._ext_tensor(v) is h and (v.item, v.offset, v.length) == (-2, 0, 128)
    _, t2 = seq.new_input(32)
    assert t2.shape == (32,) and t2.dtype == torch.float16 and not t2.any()


BAD_TENSORS = [
    (lambda: torch.zeros(64, dtype=torch.bfloat16), "has dtype torch.bfloat16, the sequence's is torch.float16", ValueError),
    (lambda: torch.zeros(63, dtype=torch.float16), "must be a contiguous vector of 64 elements", ValueError),
    (lambda: torch.zeros(2, 32, dtype=torch.float16), "must be a contiguous vector of 64 elements", ValueError),
    (lambda: torch.zeros(128, dtype=torch.float16)[::2], "must be a contiguous vector of 64 elements", ValueError),
    (lambda: torch.zeros(65, dtype=torch.float16)[1:], "must be 16-byte aligned", ValueError),
    (lambda: torch.zeros(64, dtype=torch.float16, device="meta"), "is on meta, the sequence on cpu", ValueError),
    (lambda: [0.0] * 64, "must be a tensor", TypeError),
]


@pytest.mark.parametrize("make,frag,exc", BAD_TENSORS, ids=["dtype", "length", "2d", "strided", "misaligned", "device", "list"])
def test_sequence_rejects_bad_tensors(make, frag, exc):
    with pytest.raises(exc, match=f"DecodeSequence: x {frag}" if exc is ValueError else "x must be a tensor"):
        DecodeSequence(64, "cpu", x=make())
    seq = DecodeSequence(64, "cpu")
    with pytest.raises(exc, match=f"DecodeSequence: tensor {frag}" if exc is ValueError else "tensor must be a tensor"):
        seq.new_input(64, tensor=make())
