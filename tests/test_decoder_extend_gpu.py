"""SequenceDecoder.extend and BatchDecoder.extend on the GPU: prompts and appended turns run on the decoders' own kernels
(quant_cuda.attn_extend between the projections), against the fp64 twin of test_decoder_gpu.py.

Models, banks and the criterion are those of test_decoder_gpu.py: kinds A4 / A3 (Llama at 4 / 3 bits), C (Qwen2 with q/k/v bias and a
quantized lm_head), M (Mistral), H64 (head_dim 64), B (one 7B-shaped layer), G7 (Qwen2, 7 query heads per KV head) and MQA (16 heads
on one KV head), each in fp16 and bf16.  Every logit row the decoder
returns is at most twice as far (max norm) from the twin's as the logits of the dense model of the same dtype (the twin's weights
rounded) run by HF on the same schedule (HF takes several tokens at once with a cache).  Schedules:
  * extend(17) after reset(), then 40 teacher-forced steps;
  * prefill(9) (HF), 8 steps, extend(8), 20 steps: a second turn appended to a live sequence;
  * EXTEND_CHUNK = 5: a 17-token extend over four chunks, then 5 steps;
  * extend(64) and extend(65) (the projections' tensor-core route starts at 64 fp16 rows), then 5 steps (not on Mistral, whose
    window of 64 bounds its cache);
  * a 2048-token extend on the 7B-shaped layer (B, fp16 and bf16), then 4 steps.
BatchDecoder: extending slot 1 mid-generation leaves slot 0's next logits bitwise equal to a run without that extend, and slot 1's
logits meet the twin criterion.  Besides: rejected extends (empty, 2-D, too long, bad slot) raise ValueError and leave the positions and
the caches unchanged; the model's own outputs are unchanged by building and using the decoders."""
import copy

import pytest
import torch

from test_decoder_gpu import DTYPES, SPEC, bank, banks, build, twin_of  # noqa: F401  (banks: the module-scoped fixture)

pytestmark = pytest.mark.gpu

MAX_LEN = 128


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


def hf_schedule(model, ids, plan):
    """Logits (fp64) at the end of every segment of plan [(op, n)]: HF's forward of each segment's n tokens with the cache so far."""
    out, past, t = [], None, 0
    with torch.no_grad():
        for _, n in plan:
            o = model(input_ids=ids[None, t:t + n], past_key_values=past, use_cache=True)
            past, t = o.past_key_values, t + n
            out.append(o.logits[0, -1].double())
    return torch.stack(out)


def twin_rows(twin, ids, plan):
    ends = torch.tensor([sum(n for _, n in plan[:i + 1]) - 1 for i in range(len(plan))], device=ids.device)
    with torch.no_grad():
        return twin(input_ids=ids[None, :int(ends[-1]) + 1]).logits[0, ends].double()


def dec_schedule(dec, ids, plan, slot=None):
    """The decoder's logits (fp64) at the end of every segment: prefill (HF), extend or one step per segment."""
    out, t = [], 0
    for op, n in plan:
        seg = ids[t:t + n]
        args = () if slot is None else (slot,)
        if op == "prefill":
            logits = dec.prefill(*args, seg)
        elif op == "extend":
            logits = dec.extend(*args, seg)
        elif slot is None:
            logits = dec.step(int(seg[0]))
        else:
            toks = torch.zeros(dec.batch, dtype=torch.int64)
            toks[slot] = seg[0]
            logits = dec.step(toks)[slot]
        out.append(logits.double().clone())
        t += n
    return torch.stack(out)


def check_against_twin(lq, ld, lt, what):
    assert torch.isfinite(lq).all(), what
    err_q = (lq - lt).abs().amax(dim=1)
    err_d = (ld - lt).abs().amax(dim=1)
    assert (err_q <= 2 * err_d).all(), (what, err_q.tolist(), err_d.tolist())
    return float((err_q / err_d).max())


def steps(n):
    return [("step", 1)] * n


SCHEDULES = {
    "extend17": [("extend", 17)] + steps(40),
    "multi_turn": [("prefill", 9)] + steps(8) + [("extend", 8)] + steps(20),
    "extend64": [("extend", 64)] + steps(5),
    "extend65": [("extend", 65)] + steps(5),
}


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", list(SPEC))
def test_extend_against_the_fp64_twin(banks, record, monkeypatch, kind, dtype):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    vocab = model.config.vocab_size
    ids = torch.randint(0, vocab, (MAX_LEN,), generator=torch.Generator().manual_seed(13)).cuda()
    with torch.no_grad():
        before = model(input_ids=ids[None, :9]).logits.clone()
    max_len = min(MAX_LEN, getattr(model.config, "sliding_window", None) or MAX_LEN)  # Mistral: the window bounds the cache
    dec = SequenceDecoder(model, max_len)
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    worst = 0.0
    for name, plan in SCHEDULES.items():
        if sum(n for _, n in plan) > max_len:
            continue
        dec.reset()
        lq = dec_schedule(dec, ids, plan)
        assert dec.position == sum(n for _, n in plan) and int(dec.pos) == dec.position
        worst = max(worst, check_against_twin(lq, hf_schedule(dense, ids, plan), twin_rows(twin, ids, plan), name))
    plan = [("extend", 17)] + steps(5)   # four chunks of at most 5 tokens
    monkeypatch.setattr(SequenceDecoder, "EXTEND_CHUNK", 5)
    dec.reset()
    lq = dec_schedule(dec, ids, plan)
    worst = max(worst, check_against_twin(lq, hf_schedule(dense, ids, plan), twin_rows(twin, ids, plan), "chunks of 5"))
    for s in dec.sequences:
        s.check()
    with torch.no_grad():
        after = model(input_ids=ids[None, :9]).logits
    assert torch.equal(before, after), "the model's outputs changed"
    record("worst_err_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_long_prompt_on_the_7b_layer(banks, record, dtype):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank("B")
    dt = DTYPES[dtype]
    model = build(bk, dt)
    ids = torch.randint(0, model.config.vocab_size, (2052,), generator=torch.Generator().manual_seed(5)).cuda()
    dec = SequenceDecoder(model, 2056)
    plan = [("extend", 2048)] + steps(4)
    lq = dec_schedule(dec, ids, plan)
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    record("worst_err_ratio", check_against_twin(lq, hf_schedule(dense, ids, plan), twin_rows(twin, ids, plan), "2048 tokens"))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", ["A4", "C"])
def test_batch_extend_mid_generation(banks, record, kind, dtype):
    """Slot 1 gets a second turn between steps: slot 0's logits are bitwise those of the same run without it; slot 1 meets the twin."""
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    vocab = model.config.vocab_size
    gen = torch.Generator().manual_seed(17)
    a, b = (torch.randint(0, vocab, (MAX_LEN,), generator=gen).cuda() for _ in range(2))
    dec = BatchDecoder(model, MAX_LEN, 3)
    plan_b = [("extend", 9)] + steps(5) + [("extend", 8)] + steps(6)

    def run(with_turn):
        dec.reset()
        dec.extend(0, a[:6])
        dec.extend(1, b[:9])
        got = []
        for t in range(5):
            got.append(dec.step(torch.tensor([int(a[6 + t]), int(b[9 + t]), 0])).clone())
        if with_turn:
            dec.extend(1, b[14:22])
        for t in range(6):
            nb = int(b[22 + t]) if with_turn else int(b[14 + t])
            got.append(dec.step(torch.tensor([int(a[11 + t]), nb, 0])).clone())
        return torch.stack(got)

    plain, turned = run(False), run(True)
    assert torch.equal(plain[:, 0].view(torch.int16), turned[:, 0].view(torch.int16)), "slot 0 changed when slot 1 was extended"
    assert dec.positions == [17, 28, -1]
    dec.reset()
    lq = dec_schedule(dec, b, plan_b, slot=1)
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    record("worst_err_ratio", check_against_twin(lq, hf_schedule(dense, b, plan_b), twin_rows(twin, b, plan_b), "slot 1"))


def test_rejected_extends_change_nothing(banks):
    from squeezellm_b200.runtime import BatchDecoder, SequenceDecoder
    model = build(bank("A4"), torch.float16)
    ids = torch.arange(24).cuda()
    dec = SequenceDecoder(model, 24)
    dec.extend(ids[:10])
    k, v = dec.k_cache.clone(), dec.v_cache.clone()
    for bad, msg in [(ids[:0], "non-empty 1-D"), (ids[None, :3], "non-empty 1-D"), (ids[:15], "need 25 cache positions, max_len is 24"),
                     (ids[:4].float(), "integer token ids")]:
        with pytest.raises(ValueError, match=msg):
            dec.extend(bad)
        assert dec.position == 10 and int(dec.pos) == 10
    assert torch.equal(dec.k_cache, k) and torch.equal(dec.v_cache, v)
    dec.extend(ids[:14])  # exactly max_len
    assert dec.position == 24 and int(dec.pos) == 24
    with pytest.raises(ValueError, match="need 25 cache positions"):
        dec.extend(ids[:1])

    bdec = BatchDecoder(model, 24, 2)
    bdec.extend(0, ids[:10])
    k, v = bdec.k_cache.clone(), bdec.v_cache.clone()
    for slot, bad, msg in [(2, ids[:3], "slot must be an int in 0..1"), (-1, ids[:3], "slot must be an int"), ("0", ids[:3], "slot must be"),
                           (0, ids[:0], "non-empty 1-D"), (1, ids[None, :3], "non-empty 1-D"), (0, ids[:15], "need 25 cache positions")]:
        with pytest.raises(ValueError, match=msg):
            bdec.extend(slot, bad)
        assert bdec.positions == [10, -1] and bdec.pos.tolist() == [10, -1]
    assert torch.equal(bdec.k_cache, k) and torch.equal(bdec.v_cache, v)
    bdec.extend(1, ids[:24])  # an idle slot starts at 0, exactly max_len
    assert bdec.positions == [10, 24]
