"""Sampling in SequenceDecoder.generate and BatchDecoder.generate on the GPU, on the models of test_decoder_gpu.py (kinds A4: Llama with
a dense lm_head, C: Qwen2 with a quantized lm_head), fp16 and bf16.

  * Teacher-forced, both decoders: after every step, quant_cuda.sample on dec.logits at dec.pos passes the draw-by-draw check of
    test_sample_gpu.py against sample_ref on the same logits and positions, and with top_k = 1 gives the argmax of those logits (or a
    token tied with it).
  * BatchDecoder.generate: a rerun with the same seeds is bitwise equal (prompts of 2 or more tokens: section 3.18); a prompt's tokens
    are bitwise the same in slot 0 of a batch of 2 and of 5 with other prompts beside it; different seeds diverge; top_k = 1 is greedy
    generate bitwise up to a tie at the maximum (below); a greedy row among sampled rows keeps its greedy tokens; EOS cuts and
    releases a sampled row while the others run on, and a prompt admitted into a released slot mid-run (continuous batching) draws
    the tokens it draws alone.
  * SequenceDecoder.generate reruns are not bitwise (its sequence kernel adds in arrival order, section 3.17), so its draws are checked
    through the teacher-forced test; generate gives valid ids, keeps the prompt, and different seeds diverge.
  * model(ids) gives the same logits before and after sampling.
top_k = 1 keeps every token tied at the maximum, as HF's TopKLogitsWarper does, so it equals greedy except where the logits tie at
their maximum (common in bf16); the tests check that every difference starts at such a tie."""
import numpy as np
import pytest
import torch

import sample_ref as ref
from test_decoder_gpu import DTYPES, bank, banks, build  # noqa: F401  (banks: the module-scoped fixture)
from test_sample_gpu import check_row

pytestmark = pytest.mark.gpu

MAX_LEN = 64
STEPS = 24
LENS = [9, 17, 5, 12, 3]
CASES = [(k, dt) for k in ("A4", "C") for dt in DTYPES]
PARAMS = [(0.7, 50, 0.9), (1.0, 0, 1.0), (1.3, 5, 1.0), (0.5, 0, 0.8), (0.9, 1, 1.0)]


def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def set_params(dec, params, seeds):
    n = len(params)
    dec.temperature[:n].copy_(torch.tensor([p[0] for p in params]))
    dec.top_k[:n].copy_(torch.tensor([p[1] for p in params], dtype=torch.int32))
    dec.top_p[:n].copy_(torch.tensor([p[2] for p in params]))
    dec.seed[:n].copy_(torch.tensor(seeds, dtype=torch.int64))


def check_draws(logits, pos, params, seeds, toks):
    """Each active row's token against sample_ref on the same logits and position."""
    x = logits.float().cpu().numpy()
    for b, (t, k, p) in enumerate(params):
        if pos[b] < 0:
            continue
        if ref.greedy(x[b], t):
            assert toks[b] == int(np.argmax(x[b]))
        else:
            check_row(x[b], t, k, p, int(pos[b]), seeds[b], int(toks[b]))


@pytest.mark.parametrize("kind,dtype", CASES, ids=[f"{k}-{d}" for k, d in CASES])
def test_teacher_forced_draws(banks, kind, dtype):
    from squeezellm_b200.runtime import BatchDecoder, SequenceDecoder
    model = build(bank(kind), DTYPES[dtype])
    vocab = model.config.vocab_size
    gen = torch.Generator().manual_seed(3)
    seqs = [torch.randint(0, vocab, (T + STEPS,), generator=gen).cuda() for T in LENS]

    dec = SequenceDecoder(model, MAX_LEN)
    set_params(dec, [PARAMS[0]], [77])
    k1 = torch.zeros(1, dtype=torch.int32, device="cuda") + 1
    tok1 = torch.zeros(1, dtype=torch.int64, device="cuda")
    dec.prefill(seqs[0][:LENS[0]])
    for t in range(STEPS):
        logits = dec.step(seqs[0][LENS[0] + t]).view(1, -1)
        qc().sample(logits, dec.pos, dec.temperature, dec.top_k, dec.top_p, dec.seed, dec.tok)
        qc().sample(logits, dec.pos, dec.temperature, k1, dec.top_p, dec.seed, tok1)
        check_draws(logits, dec.pos.cpu().tolist(), [PARAMS[0]], [77], dec.tok.cpu().tolist())
        assert_argmax_or_tied(logits[0], tok1.item())
    del dec

    B = len(LENS)
    dec = BatchDecoder(model, MAX_LEN, B)
    seeds = [5, 6, 7, 2 ** 62 + 1, 123456789]
    set_params(dec, PARAMS, seeds)
    for b, T in enumerate(LENS):
        dec.prefill(b, seqs[b][:T])
    for t in range(STEPS):
        logits = dec.step(torch.stack([s[T + t] for s, T in zip(seqs, LENS)]))
        qc().sample(logits, dec.pos, dec.temperature, dec.top_k, dec.top_p, dec.seed, dec.tok)
        check_draws(logits, dec.pos.cpu().tolist(), PARAMS, seeds, dec.tok.cpu().tolist())


def assert_argmax_or_tied(logits, tok):
    """top_k = 1 keeps every token tied at the maximum (HF's rule), so it draws argmax(logits) unless the maximum is tied, and then one
    of the tied tokens."""
    ties = (logits == logits.max()).nonzero().flatten().tolist()
    assert tok in ties and (len(ties) > 1 or tok == logits.argmax().item()), (tok, ties)


def assert_greedy_or_tied(dec, ps, greedy, other):
    """other (top_k = 1) equals greedy row by row, except from a step whose logits tie at their maximum: the row is replayed alone up to
    its first difference (a row's logits do not depend on the other rows) and that step's logits must hold both tokens as tied maxima."""
    for i, p in enumerate(ps):
        if torch.equal(greedy[i], other[i]):
            continue
        j = int((greedy[i] != other[i]).nonzero()[0])
        dec.reset()
        lg = dec.prefill(i, p)
        for t in range(len(p), j):
            toks = torch.zeros(dec.batch, dtype=torch.int64)
            toks[i] = greedy[i][t]
            lg = dec.step(toks)[i]
        ties = (lg == lg.max()).nonzero().flatten().tolist()
        assert len(ties) > 1 and int(greedy[i][j]) in ties and int(other[i][j]) in ties, (i, j, ties)


def prompts(vocab, n, seed=4):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (T,), generator=gen) for T in LENS[:n]]


@pytest.mark.parametrize("kind,dtype", CASES, ids=[f"{k}-{d}" for k, d in CASES])
def test_batch_generate_sampling(banks, kind, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank(kind), DTYPES[dtype])
    vocab = model.config.vocab_size
    ids = torch.randint(0, vocab, (1, 11), generator=torch.Generator().manual_seed(8)).cuda()
    with torch.no_grad():
        before = model(input_ids=ids).logits.clone()
    ps = prompts(vocab, 5)
    kw = dict(temperature=0.8, top_p=0.95, seed=11)
    dec5 = BatchDecoder(model, MAX_LEN, 5)
    a = dec5.generate(ps, 20, **kw)
    b = dec5.generate(ps, 20, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)  # every prompt here has >= 2 tokens
    other = prompts(vocab, 5, seed=99)
    c = dec5.generate([ps[0]] + other[1:], 20, **kw)
    dec2 = BatchDecoder(model, MAX_LEN, 2)
    d = dec2.generate([ps[0], other[3]], 20, **kw)
    assert torch.equal(a[0], c[0]) and torch.equal(a[0], d[0])
    e = dec5.generate(ps, 20, temperature=0.8, top_p=0.95, seed=12)
    assert any(not torch.equal(x, y) for x, y in zip(a, e))
    assert sum(not torch.equal(x, y) for x, y in zip(a, e)) >= 3
    greedy = dec5.generate(ps, 20)
    k1 = dec5.generate(ps, 20, temperature=0.7, top_k=1, seed=3)
    mixed = dec5.generate(ps[:3], 20, temperature=[0.0, 0.9, 1.2], top_k=[0, 40, 0], seed=[1, 2, 3])
    assert torch.equal(mixed[0], greedy[0])
    assert not torch.equal(mixed[1], greedy[1]) or not torch.equal(mixed[2], greedy[2])
    # EOS: a token row 1 draws mid-run ends row 1 there; the other rows run on unchanged up to their own first EOS
    eos = int(a[1][len(ps[1]) + 6])
    f = dec5.generate(ps, 20, eos_token_id=eos, **kw)
    for x, y, p in zip(a, f, ps):
        new = x[len(p):].tolist()
        cut = new.index(eos) + 1 if eos in new else len(new)
        assert torch.equal(y, x[:len(p) + cut])
    assert len(f[1]) <= len(ps[1]) + 7
    assert_greedy_or_tied(dec5, ps, greedy, k1)
    with torch.no_grad():
        assert torch.equal(model(input_ids=ids).logits, before)


@pytest.mark.parametrize("kind,dtype", CASES[:2], ids=[f"{k}-{d}" for k, d in CASES[:2]])
def test_continuous_batching_while_sampling(banks, kind, dtype):
    """A prompt prefilled into a released slot mid-run, sampled after each step, draws what it draws in slot 0 of a fresh run."""
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank(kind), DTYPES[dtype])
    ps = prompts(model.config.vocab_size, 3)
    dec = BatchDecoder(model, MAX_LEN, 3)

    def run(admit_at):
        dec.reset()
        set_params(dec, [(0.9, 0, 0.95)] * 3, [41, 42, 43])
        first = [dec.prefill(i, p) for i, p in enumerate(ps[:2])]
        qc().sample(torch.stack(first), dec.pos[:2], dec.temperature[:2], dec.top_k[:2], dec.top_p[:2], dec.seed[:2], dec.tok[:2])
        got = []
        for t in range(12):
            if t == admit_at:
                dec.release(1)
                lg = dec.prefill(1, ps[2]).view(1, -1)
                qc().sample(lg, dec.pos[1:2], dec.temperature[1:2], dec.top_k[1:2], dec.top_p[1:2], dec.seed[1:2], dec.tok[1:2])
                got = [dec.tok[1].item()]
            logits = dec.step(dec.tok.clone())
            qc().sample(logits, dec.pos, dec.temperature, dec.top_k, dec.top_p, dec.seed, dec.tok)
            if t >= admit_at:
                got.append(dec.tok[1].item())
        return got

    mid = run(5)
    dec.reset()
    set_params(dec, [(0.9, 0, 0.95)] * 3, [42, 0, 0])
    lg = dec.prefill(0, ps[2]).view(1, -1)
    qc().sample(lg, dec.pos[:1], dec.temperature[:1], dec.top_k[:1], dec.top_p[:1], dec.seed[:1], dec.tok[:1])
    alone = [dec.tok[0].item()]
    for _ in range(6):
        logits = dec.step(dec.tok.clone())
        qc().sample(logits, dec.pos, dec.temperature, dec.top_k, dec.top_p, dec.seed, dec.tok)
        alone.append(dec.tok[0].item())
    assert mid[:7] == alone[:7]


@pytest.mark.parametrize("kind,dtype", CASES, ids=[f"{k}-{d}" for k, d in CASES])
def test_sequence_generate_sampling(banks, kind, dtype):
    from squeezellm_b200.runtime import SequenceDecoder
    model = build(bank(kind), DTYPES[dtype])
    vocab = model.config.vocab_size
    p = prompts(vocab, 1)[0]
    dec = SequenceDecoder(model, MAX_LEN)
    out = dec.generate(p, 20, temperature=0.8, top_p=0.9, seed=5)
    assert out.shape == (1, len(p) + 20) and ((out >= 0) & (out < vocab)).all()
    assert torch.equal(out[0, :len(p)].cpu(), p)
    again = dec.generate(p, 20, temperature=0.8, top_p=0.9, seed=5)
    assert torch.equal(again[0, :len(p) + 1], out[0, :len(p) + 1])  # the first token comes from HF's prefill: bitwise
    other = dec.generate(p, 20, temperature=1.5, seed=6)
    assert not torch.equal(out, other)
