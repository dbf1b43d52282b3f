"""GPU tests of BatchDecoder(pages=P): every row's logits are bitwise those of the contiguous BatchDecoder, through prefill, extend,
steps that cross page boundaries, churn in a pool smaller than batch x width, an empty pool, and fork."""
import pytest
import torch

from test_decoder_gpu import DTYPES, bank, banks, build  # noqa: F401  (banks: the module-scoped fixture)

pytestmark = pytest.mark.gpu

MAX_LEN = 256         # 4 pages per slot
STEPS = 40
PROMPTS = [2, 63, 64, 65, 130]
KINDS = ["A4", "C", "H64", "B", "G7", "MQA"]
CASES = [(k, d) for k in KINDS for d in DTYPES]


def _prompts(vocab, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (n + STEPS,), generator=g).cuda() for n in PROMPTS]


def forced(dec, seqs, use_extend):
    """Logits per row [STEPS + 1, vocab]: the prompt seqs[b][:n_b] by prefill or extend, then STEPS steps feeding the rest."""
    B = len(seqs)
    out = []
    for b, s in enumerate(seqs):
        n = len(s) - STEPS
        out.append([(dec.extend(b, s[:n]) if use_extend else dec.prefill(b, s[:n])).clone()])
    for t in range(STEPS):
        toks = torch.zeros(dec.batch, dtype=torch.int64)
        for b, s in enumerate(seqs):
            toks[b] = s[len(s) - STEPS + t]
        logits = dec.step(toks)
        for b in range(B):
            out[b].append(logits[b].clone())
    return [torch.stack(o) for o in out]


@pytest.mark.parametrize("kind,dtype", CASES, ids=[f"{k}-{d}" for k, d in CASES])
def test_paged_logits_equal_contiguous(banks, kind, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank(kind), DTYPES[dtype])
    seqs = _prompts(model.config.vocab_size)
    B = len(seqs)
    contiguous = BatchDecoder(model, MAX_LEN, B)
    want = {}
    for e in (False, True):
        contiguous.reset()
        want[e] = forced(contiguous, seqs, e)
    gen_want = contiguous.generate([s[:n] for s, n in zip(seqs, PROMPTS)], 30)
    del contiguous
    P = B * 4
    dec = BatchDecoder(model, MAX_LEN, B, pages=P)
    for e in (False, True):
        dec.reset()
        got = forced(dec, seqs, e)
        for b in range(B):
            # extend's own logits come from lm_head on one row: the one-row route, which is not bitwise reproducible
            first = 1 if e else 0
            assert torch.equal(got[b][first:], want[e][b][first:]), f"row {b} (prompt {PROMPTS[b]}, extend={e}) differs"
            torch.testing.assert_close(got[b][0], want[e][b][0], rtol=1e-2, atol=1e-2)
    gen = dec.generate([s[:n] for s, n in zip(seqs, PROMPTS)], 30)
    for a, w in zip(gen, gen_want):
        assert torch.equal(a, w)
    dec.reset()
    assert dec.free_pages == P
    ids = seqs[0][None, :8]
    with torch.no_grad():
        assert torch.equal(model(ids).logits, model(ids).logits)


def _alone(model, prompt, n_steps, feed):
    """Logits of `prompt` then n_steps fed tokens in a fresh contiguous decoder."""
    from squeezellm_b200.runtime import BatchDecoder
    dec = BatchDecoder(model, MAX_LEN, 3)   # the batch of the paged decoder: the attention's split rule depends on it
    out = [dec.prefill(0, prompt).clone()]
    for t in range(n_steps):
        out.append(dec.step(torch.tensor([int(feed[t]), 0, 0]))[0].clone())
    return torch.stack(out)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_small_pool_under_churn(banks, dtype):
    """A pool of 7 pages for 3 slots of 4: slots are released and refilled, so pages come back in a different order; each prompt's
    logits equal a fresh contiguous run of it."""
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), DTYPES[dtype])
    g = torch.Generator().manual_seed(1)
    seqs = [torch.randint(0, 512, (n,), generator=g).cuda() for n in (70, 130, 65, 100, 63)]
    dec = BatchDecoder(model, MAX_LEN, 3, pages=7)
    plan = [(0, 0), (1, 1)]   # (slot, prompt)
    rows = {}

    def start(slot, i):
        rows[slot] = (i, [dec.prefill(slot, seqs[i][:40]).clone()], 40)

    for slot, i in plan:
        start(slot, i)
    queue = [2, 3, 4]
    for _ in range(400):
        toks = torch.zeros(3, dtype=torch.int64)
        for slot, (i, logs, p) in rows.items():
            toks[slot] = seqs[i][p]
        logits = dec.step(toks)
        for slot in list(rows):
            i, logs, p = rows[slot]
            logs.append(logits[slot].clone())
            rows[slot] = (i, logs, p + 1)
            if p + 1 == len(seqs[i]):
                want = _alone(model, seqs[i][:40], len(seqs[i]) - 40, seqs[i][40:])
                assert torch.equal(torch.stack(logs), want), f"prompt {i} differs"
                dec.release(slot)
                del rows[slot]
                if queue:
                    start(slot, queue.pop(0))
        if not rows:
            break
    assert not rows and not queue
    assert dec.free_pages == 7


def test_empty_pool_raises_before_the_replay(banks):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), torch.float16)
    g = torch.Generator().manual_seed(2)
    a, b = torch.randint(0, 512, (64,), generator=g).cuda(), torch.randint(0, 512, (60,), generator=g).cuda()
    dec = BatchDecoder(model, MAX_LEN, 2, pages=2)
    ref = BatchDecoder(model, MAX_LEN, 2)
    dec.prefill(0, a)        # one full page: the next step needs a second
    dec.prefill(1, b)        # the last free page
    ref.prefill(0, a)
    ref.prefill(1, b)
    assert dec.free_pages == 0
    pos, table = dec.positions, dec.block_table.clone()
    with pytest.raises(RuntimeError, match=r"slot\(s\) \[0\]"):
        dec.step(torch.tensor([5, 6]))
    assert dec.positions == pos and torch.equal(dec.block_table, table) and dec.free_pages == 0
    dec.release(1)
    ref.release(1)
    for t in range(3):
        got = dec.step(torch.tensor([5 + t, 0]))[0].clone()
        assert torch.equal(got, ref.step(torch.tensor([5 + t, 0]))[0])


@pytest.mark.parametrize("n", [70, 64])
def test_fork(banks, n):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("C"), torch.float16)
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, 512, (n,), generator=g).cuda()
    dec = BatchDecoder(model, MAX_LEN, 3, pages=8)
    dec.prefill(0, prompt)
    free = dec.free_pages
    dec.fork(0, 2)
    assert dec.positions == [n, -1, n]
    assert dec.free_pages == free - (1 if n % 64 else 0)
    logits = dec.step(torch.tensor([7, 0, 7]))
    assert torch.equal(logits[0], logits[2])
    src = [logits[0].clone()]
    for t in range(10):   # diverge: different tokens in src and dst
        logits = dec.step(torch.tensor([11 + t, 0, 100 + t]))
        src.append(logits[0].clone())
    ref = BatchDecoder(model, MAX_LEN, 3)
    ref.prefill(0, prompt)
    want = [ref.step(torch.tensor([7, 0, 0]))[0].clone()]
    for t in range(10):
        want.append(ref.step(torch.tensor([11 + t, 0, 0]))[0].clone())
    assert torch.equal(torch.stack(src), torch.stack(want))
    with pytest.raises(ValueError):
        dec.fork(1, 0)   # src idle
    with pytest.raises(ValueError):
        dec.fork(0, 2)   # dst active
    dec.reset()
    assert dec.free_pages == 8
