"""Speculative decoding in SequenceDecoder (speculate=K) on the GPU, on the models of test_decoder_gpu.py (A4, A3, C with q/k/v bias and a
quantized lm_head, M, H64, the 7B-shaped B, G7 with 7 query heads per KV head and MQA with one KV head) in fp16 and bf16, K in
{3, 15} on every kind and {1, 7} besides on A4, prompts of 1 and 17 tokens, against the fp64 twin:
  * teacher-forced verify() chunks of K + 1 tokens: every logits row at most twice as far (max norm) from the twin's as the logits of
    the dense model of the same dtype decoding the same tokens with HF's cache (the criterion of test_decoder_gpu.py);
  * after each verify, quant_cuda.sample of every row at dec.vpos (= p + t + 1) passes the draw check of test_decoder_sample_gpu.py;
  * verify, rewind, verify again: bitwise equal logits;
  * greedy generate equals the twin's greedy tokens up to its first near-tie (top-2 margin below twice the error measured above) for
    four drafters: an oracle (the twin's tokens: every verify before that horizon accepts all it proposed), an always-wrong one
    (nothing accepted), the built-in prompt lookup on a repeating prompt, and one that proposes fewer than K ids or none;
  * sampled generate equals plain sampled generate for the same seed up to the first fp64 near-tie of the Gumbel-perturbed scores;
  * dec.position after generate equals plain generate's, and 10 further steps meet the twin criterion;
  * the model's outputs are unchanged by building the decoder.
Besides, on A4: EOS inside an accepted run, generating up to exactly max_len (the last iterations fall back to steps), a drafter's bad
output."""
import copy

import numpy as np
import pytest
import torch

import sample_ref as ref
from test_decoder_gpu import SPEC, DTYPES, bank, banks, build, hf_decode, twin_of  # noqa: F401  (banks: the module-scoped fixture)
from test_decoder_sample_gpu import check_draws

pytestmark = pytest.mark.gpu

MAX_LEN = 64
N_NEW = 20
KS = {kind: (1, 3, 7, 15) if kind == "A4" else (3, 15) for kind in SPEC}
SAMPLED = dict(temperature=0.8, top_k=0, top_p=1.0, seed=5)


def qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def twin_greedy(twin, prompt, n, tol):
    """The twin's greedy tokens after prompt, up to (not including) the first step whose top-2 margin is below tol."""
    cur, want = prompt.clone(), []
    with torch.no_grad():
        for _ in range(n):
            logit = twin(input_ids=cur[None]).logits[0, -1]
            top2 = torch.topk(logit, 2).values
            if float(top2[0] - top2[1]) < tol:
                break
            want.append(int(logit.argmax()))
            cur = torch.cat([cur, torch.tensor(want[-1:], device=cur.device)])
    return want


class Recorder:
    """A drafter fn(n, K) -> proposal (n: the new tokens so far, the pending one included) that records each call's history length."""

    def __init__(self, T0, K, fn):
        self.T0, self.K, self.fn, self.calls = T0, K, fn, []

    def __call__(self, toks):
        n = len(toks) - self.T0
        prop = self.fn(n, self.K)
        self.calls.append((n, len(prop)))
        return prop

    def emitted(self, total):
        """(n, proposed, emitted) of every call whose emitted count is known (all but the last; total: the new tokens at the end)."""
        ns = [c[0] for c in self.calls] + [total]
        return [(n, m, ns[i + 1] - n) for i, (n, m) in enumerate(self.calls)][:-1]


def teacher_forced(dec, twin, dense, seq, T0, K):
    """Prefill seq[:T0], then verify chunks of K + 1: (decoder logits, twin logits, dense logits) [rows, vocab] of positions T0-1 ..."""
    T = K + 1
    n = (min(len(seq), MAX_LEN) - T0) // T
    seq = seq[:T0 + n * T]
    rows = [dec.prefill(seq[:T0]).double()[None]]
    for c in range(n):
        rows.append(dec.verify(seq[T0 + c * T:T0 + (c + 1) * T]).double())
    assert dec.position == len(seq)
    with torch.no_grad():
        lt = twin(input_ids=seq[None]).logits[0, T0 - 1:].double()
    return torch.cat(rows), lt, hf_decode(dense, seq, T0), seq


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", list(SPEC))
def test_speculate_against_the_fp64_twin(banks, record, kind, dtype):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    vocab = model.config.vocab_size
    ids = torch.randint(0, vocab, (MAX_LEN,), generator=torch.Generator().manual_seed(11)).cuda()
    with torch.no_grad():
        before = model(input_ids=ids[None, :9]).logits.clone()
    plain = SequenceDecoder(model, MAX_LEN)
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    pattern = torch.randint(0, vocab, (5,), generator=torch.Generator().manual_seed(12)).cuda()
    repeating = pattern.repeat(4)[:17]
    for K in KS[kind]:
        dec = SequenceDecoder(model, MAX_LEN, speculate=K)
        with torch.no_grad():
            assert torch.equal(model(input_ids=ids[None, :9]).logits, before), "the model's outputs changed when the decoder was built"
        err = 0.0
        for T0 in (1, 17):
            # teacher-forced verify chunks against the twin
            lq, lt, ld, seq = teacher_forced(dec, twin, dense, ids, T0, K)
            err_q, err_d = (lq - lt).abs().amax(dim=1), (ld - lt).abs().amax(dim=1)
            assert torch.isfinite(lq).all()
            assert (err_q <= 2 * err_d).all(), (K, T0, err_q.tolist(), err_d.tolist())
            err = max(err, float(err_q.max()))
            record(f"K{K}_T{T0}_err_ratio", float((err_q / err_d).max()))
            # verify, rewind, verify: bitwise; then the draws of every row at vpos
            p = T0 + (K + 1)
            dec.rewind(p)
            first = dec.verify(seq[p:p + K + 1]).clone()
            dec.rewind(p)
            again = dec.verify(seq[p:p + K + 1])
            assert torch.equal(first, again)
            assert dec.vpos.tolist() == list(range(p + 1, p + K + 2))
            for buf, v in zip(dec._vsampling, (0.8, 40, 0.9, 77)):
                buf.fill_(v)
            qc().sample(dec.vlogits, dec.vpos, *dec._vsampling, dec.vdraw)
            check_draws(dec.vlogits, dec.vpos.tolist(), [(0.8, 40, 0.9)] * (K + 1), [77] * (K + 1), dec.vdraw.tolist())
        tol = 2 * err
        for T0, prompt in ((1, ids[:1]), (17, ids[:17]), (17, repeating)):
            want = twin_greedy(twin, prompt, N_NEW, tol)
            h = len(want)
            drafters = {"lookup": None}
            if prompt is not repeating:
                drafters = {
                    "oracle": Recorder(T0, K, lambda n, k: want[n:n + k]),
                    "wrong": Recorder(T0, K, lambda n, k: [(w + 1) % vocab for w in want[n:n + k]]),
                    "fewer": Recorder(T0, K, lambda n, k: [] if n % 3 == 0 else want[n:n + max(1, k // 2)]),
                }
            for name, dr in drafters.items():
                out = dec.generate(prompt[None], N_NEW, draft=dr)[0, T0:].tolist()
                assert out[:h] == want, (K, T0, name, out, want)
                assert dec.position == T0 + N_NEW - 1
                st = dec.spec_stats
                if name == "oracle":
                    for n, m, e in dr.emitted(len(out)):
                        if m and n + m <= h:
                            assert e == m + 1, (K, T0, dr.calls)
                    if h == N_NEW:
                        assert st["accepted"] == st["drafted"] > 0, st
                if name == "wrong":
                    for n, m, e in dr.emitted(len(out)):
                        if m and n + m <= h:
                            assert e == 1, (K, T0, dr.calls)
                if name == "lookup":
                    assert st["verifies"] > 0, st
                record(f"K{K}_T{T0}_{name}_stats", str(st))
                record(f"K{K}_T{T0}_{name}_horizon", h)
            # sampled: the tokens of plain sampled generate for the same seed, up to the first near-tie of the perturbed scores
            oracle_s = plain.generate(prompt[None], N_NEW, **SAMPLED)[0, T0:].tolist()
            got = dec.generate(prompt[None], N_NEW, draft=lambda toks: oracle_s[len(toks) - T0:len(toks) - T0 + K], **SAMPLED)
            got = got[0, T0:].tolist()
            assert dec.position == plain.position == T0 + N_NEW - 1
            if got != oracle_s:
                j = next(i for i, (a, b) in enumerate(zip(got, oracle_s)) if a != b)
                with torch.no_grad():
                    x = twin(input_ids=torch.cat([prompt, torch.tensor(got[:j], device=prompt.device)])[None]).logits[0, -1]
                s = x.double().cpu().numpy() / SAMPLED["temperature"] + ref.gumbel(vocab, T0 + j, SAMPLED["seed"])
                top2 = np.sort(s)[-2:]
                assert top2[1] - top2[0] < 2 * tol / SAMPLED["temperature"], (K, T0, j, got, oracle_s)
                record(f"K{K}_T{T0}_sampled_agree", j)
        # after generate: 10 further steps meet the twin criterion
        prompt = ids[:17]
        out = dec.generate(prompt[None], N_NEW, draft=lambda toks: [int(t) for t in ids[len(toks):len(toks) + K]])[0]
        L = len(out)
        assert dec.position == L - 1
        full = torch.cat([out, ids[:10]])
        steps = torch.stack([dec.step(int(full[L - 1 + i])).double() for i in range(10)])
        with torch.no_grad():
            lt = twin(input_ids=full[None, :L + 9]).logits[0, L - 1:].double()
        ld = hf_decode(dense, full[:L + 9], L)
        assert ((steps - lt).abs().amax(dim=1) <= 2 * (ld - lt).abs().amax(dim=1)).all()
        for s in dec.sequences:
            s.check()
        del dec


def test_eos_max_len_and_bad_drafts(banks):
    from squeezellm_b200.runtime import SequenceDecoder
    bk = bank("A4")
    model = build(bk, torch.float16)
    K = 3
    dec = SequenceDecoder(model, MAX_LEN, speculate=K)
    prompt = torch.arange(17).cuda()
    full = dec.generate(prompt[None], N_NEW)[0, 17:].tolist()
    oracle = lambda toks: full[len(toks) - 17:len(toks) - 17 + K]  # noqa: E731  (the decoder's own greedy tokens: all accepted)
    # EOS inside an accepted run: the first verify emits new tokens 1 .. K + 1; cut it at new token j, the first of 2, 3, 1 not seen before
    j = next(i for i in (2, 3, 1) if full[i] not in full[:i])
    out = dec.generate(prompt[None], N_NEW, eos_token_id=full[j], draft=oracle)[0, 17:].tolist()
    assert out == full[:j + 1] and dec.position == 17 + j
    assert dec.spec_stats["verifies"] == 1
    # up to exactly max_len: the prompt and max_new - 1 tokens fill the cache; the last iterations run ordinary steps
    n = MAX_LEN - 17 + 1
    long_plain = dec.generate(prompt[None], n, draft=lambda toks: [])[0, 17:].tolist()
    assert dec.spec_stats["verifies"] == 0
    got = dec.generate(prompt[None], n, draft=lambda toks: long_plain[len(toks) - 17:len(toks) - 17 + K])[0, 17:].tolist()
    assert len(got) == n and dec.position == MAX_LEN
    k = next((i for i, (a, b) in enumerate(zip(got, long_plain)) if a != b), None)
    if k is not None:  # both are greedy from the same prompt: a difference starts where the step path's logits nearly tie
        lg = dec.prefill(prompt)
        for t in long_plain[:k]:
            lg = dec.step(t)
        top2 = torch.topk(lg.float(), 2).values
        assert float(top2[0] - top2[1]) < 0.25, (k, got, long_plain)
    dec.rewind(61)
    with pytest.raises(ValueError, match="SequenceDecoder.verify: 4 tokens at position 61 need 65 cache positions"):
        dec.verify([1, 2, 3, 4])
    with pytest.raises(ValueError, match="SequenceDecoder.verify: 3 token ids"):
        dec.verify([1, 2, 3])
    with pytest.raises(ValueError, match="SequenceDecoder.rewind: position must be an int in 0..61"):
        dec.rewind(62)
    assert dec.position == 61
    # a drafter's bad output raises
    for bad in (lambda toks: [model.config.vocab_size], lambda toks: [1.5], lambda toks: None):
        with pytest.raises(ValueError, match="SequenceDecoder.generate: draft"):
            dec.generate(prompt[None], 8, draft=bad)
