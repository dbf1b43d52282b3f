"""runtime.SequenceDecoder on the GPU: whole quantized LLaMA-family models decoded one CUDA graph per token, against an fp64 twin.

Models are made as in test_model_gpu.py (random init from a config, eager attention, oracle.make_layer layers scaled to entries of about
1 / sqrt(in_features), loaded through checkpoint.load_quantized, then .cuda()); the fp64 twin is the same HF class in float64 holding the
dense fp64 weights W.T.  Kinds: A4 / A3 (Llama, hidden 1024, 8 heads, 2 KV heads, at 4 / 3 bits), C (Qwen2 with q/k/v bias and a
quantized lm_head), M (Mistral with its window >= max_len), H64 (Llama with head_dim 64), B (one 7B-shaped Llama layer), G7 (Qwen2
with the attention of Qwen2.5-0.5B: 14 heads of 64 on 2 KV heads, 7 query heads per KV head, and a quantized lm_head, at 4 bits) and
MQA (Llama with 16 heads of 128 on one KV head: each group over two clusters of the attention kernels, at 3 bits).  Each in fp16 and
bf16, after a prompt of 1 and of 17 tokens:
  * teacher-forced decode for 40 steps: at every step the decoder's logits are at most twice as far (max norm) from the twin's as the
    logits of a dense model of the same dtype (the twin's weights rounded) decoding the same tokens with HF's cache;
  * greedy generate matches the twin's greedy tokens up to the first step where the twin's top-2 margin is below twice the error
    measured above;
  * reset() and the same prompt give the same greedy tokens (up to that step) and the same logits to within the error measured
    above, not bitwise: the sequence kernel adds its partial sums in arrival order.
Besides: the cache filled to exactly max_len works and one step more raises; model(ids) gives the same logits after the decoder is
built as before (the decoder applies the sibling stacking only, and the model here is stacked already)."""
import copy

import numpy as np
import pytest
import torch

from backward_ref import dense_w_f64
from util import orc

pytestmark = pytest.mark.gpu

transformers = pytest.importorskip("transformers")

MAX_LEN = 64
STEPS = 40
SPEC = {  # kind: (config class, config kwargs, bits, lm_head quantized)
    "A4": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
                               vocab_size=512), 4, False),
    "A3": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
                               vocab_size=512), 3, False),
    "C": ("Qwen2Config", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
                              vocab_size=512), 4, True),
    "M": ("MistralConfig", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
                                vocab_size=512, sliding_window=MAX_LEN), 4, False),
    "H64": ("LlamaConfig", dict(hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=4,
                                vocab_size=512), 4, False),
    "B": ("LlamaConfig", dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=32,
                              vocab_size=256), 4, False),
    "G7": ("Qwen2Config", dict(hidden_size=896, intermediate_size=2432, num_hidden_layers=2, num_attention_heads=14, num_key_value_heads=2,
                               vocab_size=512), 4, True),
    "MQA": ("LlamaConfig", dict(hidden_size=2048, intermediate_size=5504, num_hidden_layers=2, num_attention_heads=16, num_key_value_heads=1,
                                vocab_size=512), 3, False),
}
MODEL_OF = {"LlamaConfig": "LlamaForCausalLM", "Qwen2Config": "Qwen2ForCausalLM", "MistralConfig": "MistralForCausalLM"}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _config(kind):
    cls, kw, _, _ = SPEC[kind]
    return getattr(transformers, cls)(max_position_embeddings=256, attn_implementation="eager", **kw)


def _new_model(kind):
    return getattr(transformers, MODEL_OF[SPEC[kind][0]])(_config(kind))


class Bank:
    """The scaled oracle layers of one kind and their dense fp64 weights W [K, N] on the GPU, made once per test module."""

    def __init__(self, kind):
        from squeezellm_b200 import checkpoint as ck
        _, _, bits, quant_head = SPEC[kind]
        torch.manual_seed(0)
        model = _new_model(kind)
        self.kind, self.bits, self.L, self.W = kind, bits, {}, {}
        for i, (name, lin) in enumerate(sorted(ck.find_linear_layers(model).items())):
            if name == "lm_head" and not quant_head:
                continue
            K, N = lin.in_features, lin.out_features
            L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=1000 + 17 * i, nonzero_full_rows=True, bias=lin.bias is not None)
            s = 1.0 / np.sqrt(K)
            L["lookup_table"] = (L["lookup_table"] * (s / 0.02)).astype(np.float32)
            L["vals"] = (L["vals"] * (s / 0.1)).astype(np.float32)
            L["full_rows"] = (L["full_rows"] * (s / 0.05)).astype(np.float32)
            self.L[name] = L
            self.W[name] = torch.from_numpy(dense_w_f64(L)).cuda()


_banks = {}


@pytest.fixture(scope="module")
def banks():
    yield _banks
    _banks.clear()
    torch.cuda.empty_cache()


def bank(kind):
    if kind not in _banks:
        _banks[kind] = Bank(kind)
    return _banks[kind]


def build(bk, dtype):
    """The quantized model of bk in dtype on the GPU, siblings stacked."""
    from squeezellm_b200 import checkpoint as ck, fusion
    torch.manual_seed(0)
    model = _new_model(bk.kind).to(dtype).eval()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    for name, L in bk.L.items():
        del state[name + ".weight"]
        for k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices", "bias"):
            if L.get(k) is not None:
                state[f"{name}.{k}"] = torch.from_numpy(L[k])
        state["sparse_threshold." + name] = len(L["vals"])
    res = ck.load_quantized(model, state, bk.bits, include_sparse=True, topX=10, skip=() if SPEC[bk.kind][3] else ("lm_head",))
    assert not res.missing_keys and not res.unexpected_keys, res
    model = model.cuda()
    fusion.fuse_siblings(model)
    return model


def twin_of(bk, model):
    twin = _new_model(bk.kind).to(torch.float64).eval()
    src = model.state_dict()
    sd = {}
    for k in twin.state_dict():
        layer, leaf = k.rsplit(".", 1)
        if layer in bk.L:
            sd[k] = bk.W[layer].t().contiguous() if leaf == "weight" else torch.from_numpy(bk.L[layer]["bias"]).double()
        else:
            sd[k] = src[k].double()
    twin.load_state_dict(sd)
    return twin.cuda()


def hf_decode(model, ids, T):
    """Logits [len(ids) - T + 1, vocab] (fp64) of the positions T-1 .. len-1: the prompt ids[:T], then one token at a time with HF's cache."""
    with torch.no_grad():
        o = model(input_ids=ids[None, :T], use_cache=True)
        out = [o.logits[0, -1].double()]
        for t in range(T, len(ids)):
            o = model(input_ids=ids[None, t:t + 1], past_key_values=o.past_key_values, use_cache=True)
            out.append(o.logits[0, -1].double())
    return torch.stack(out)


def decoder_logits(dec, ids, T):
    out = [dec.prefill(ids[:T]).double()]
    for t in range(T, len(ids)):
        out.append(dec.step(int(ids[t])).double())
    return torch.stack(out)


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", list(SPEC))
def test_decoder_against_the_fp64_twin(banks, record, kind, dtype):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    vocab = model.config.vocab_size
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, vocab, (17 + STEPS,), generator=gen).cuda()
    with torch.no_grad():
        before = model(input_ids=ids[None, :9]).logits.clone()
    dec = SequenceDecoder(model, MAX_LEN)
    with torch.no_grad():
        after = model(input_ids=ids[None, :9]).logits
    assert torch.equal(before, after), "the model's outputs changed when the decoder was built"
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    worst = 0.0
    for T in (1, 17):
        seq = ids[:T + STEPS]
        with torch.no_grad():
            lt = twin(input_ids=seq[None]).logits[0, T - 1:].double()
        ld = hf_decode(dense, seq, T)
        lq = decoder_logits(dec, seq, T)
        err_q = (lq - lt).abs().amax(dim=1)
        err_d = (ld - lt).abs().amax(dim=1)
        assert torch.isfinite(lq).all()
        ratio = float((err_q / err_d).max())
        worst = max(worst, ratio)
        assert (err_q <= 2 * err_d).all(), (T, err_q.tolist(), err_d.tolist())
        # reset, the same prompt and tokens: the logits agree within the error measured above (the sequence kernel and the one-row
        # prompt route add their partial sums in arrival order, so their last bits vary run to run)
        dec.reset()
        again = decoder_logits(dec, seq, T)
        rerun = float((again - lq).abs().max())
        assert rerun <= float(err_q.max()), (rerun, float(err_q.max()))
        record(f"rerun_diff_T{T}", rerun)
        # greedy against the twin's greedy tokens, up to the first step where the twin's top-2 margin is within the error; twice
        n_new = 20
        runs = []
        for _ in range(2):
            dec.reset()
            runs.append(dec.generate(seq[None, :T], n_new)[0, T:].tolist())
        tol = 2 * float(err_q.max())
        cur = seq[:T].clone()
        with torch.no_grad():
            for j in range(n_new):
                logit = twin(input_ids=cur[None]).logits[0, -1]
                top2 = torch.topk(logit, 2).values
                if float(top2[0] - top2[1]) < tol:
                    break
                want = int(logit.argmax())
                assert runs[0][j] == want and runs[1][j] == want, (T, j, runs, want)
                cur = torch.cat([cur, torch.tensor([want], device=cur.device)])
        record(f"greedy_agree_T{T}", j)
    for s in dec.sequences:
        s.check()
    record("worst_err_ratio", worst)


def test_cache_limits(banks):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank("A4")
    model = build(bk, torch.float16)
    dec = SequenceDecoder(model, 20)
    ids = torch.arange(17).cuda()
    dec.prefill(ids)
    for t in range(3):
        logits = dec.step(t)
    assert dec.position == 20 and torch.isfinite(logits).all()
    with pytest.raises(RuntimeError, match="the cache is full"):
        dec.step(0)
    with pytest.raises(ValueError, match="need 21 cache positions, max_len is 20"):
        dec.generate(ids[None], 5)
    out = dec.generate(ids[None], 4)  # 17 + 3 steps: exactly max_len
    assert out.shape == (1, 21) and dec.position == 20
    dec.reset()
    assert dec.position == 0
    with pytest.raises(ValueError, match="21 prompt tokens"):
        dec.prefill(torch.arange(21).cuda())


def test_generate_stops_at_eos(banks):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank("A4")
    model = build(bk, torch.float16)
    dec = SequenceDecoder(model, MAX_LEN)
    ids = torch.arange(5).cuda()[None]
    full = dec.generate(ids, 30)[0, 5:].tolist()
    eos = full[11]
    first = full.index(eos)
    out = dec.generate(ids, 30, eos_token_id=eos)[0, 5:].tolist()
    assert out == full[:first + 1]
