"""BatchDecoder.extend_many on the GPU: several slots' prompts or new turns in one run through the model (quant_cuda.attn_extend_batch
between the projections), against the fp64 twin of test_decoder_gpu.py with the criterion of test_decoder_extend_gpu.py (every logit row
at most twice as far from the twin's as the dense model's of the same dtype run by HF on the same schedule).
  * fresh prompts of 17, 5, 40 and 1 tokens into slots 2, 0, 3 and 1 in one call, then steps: each slot meets the twin on its own
    schedule, in the contiguous and the paged layout, and the paged decoder's logits and gathered caches equal the contiguous one's
    bitwise (kinds A4, C, M, H64, G7 and MQA in fp16 and bf16);
  * second turns: two of three live slots, at different positions, get new turns in one call; the third slot's later step logits are
    bitwise those of a run without the call, and the turned slots meet the twin;
  * EXTEND_CHUNK = 5: prompts of 17 and 9 tokens split across passes;
  * forked slots take different turns in one call: the shared pages stay bitwise untouched and both slots meet the twin;
  * the 7B-shaped kind B: 8 prompts of 256 tokens (2048 rows in one pass);
  * every rejection leaves the positions, the caches, block_table and free_pages unchanged."""
import copy

import pytest
import torch

from test_decoder_extend_gpu import check_against_twin, hf_schedule, steps, twin_rows
from test_decoder_gpu import DTYPES, bank, banks, build, twin_of  # noqa: F401  (banks: the module-scoped fixture)

pytestmark = pytest.mark.gpu

MAX_LEN = 128
KINDS = ["A4", "C", "M", "H64", "G7", "MQA"]
CASES = [(k, d) for k in KINDS for d in DTYPES]
FRESH = {2: 17, 0: 5, 3: 40, 1: 1}   # slot: prompt tokens, in the order of the call
STEPS = 6


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


def _ids(vocab, n, count, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, vocab, (n,), generator=g).cuda() for _ in range(count)]


def _max_len(model):
    return min(MAX_LEN, getattr(model.config, "sliding_window", None) or MAX_LEN)  # Mistral: the window bounds the cache


def _fresh_run(dec, seqs):
    """extend_many of FRESH into their slots, then STEPS steps feeding each slot's sequence: {slot: logits [1 + STEPS, vocab]}."""
    dec.reset()
    slots = list(FRESH)
    got = dec.extend_many(slots, [seqs[s][:FRESH[s]] for s in slots])
    assert got.shape[0] == len(slots)
    rows = {s: [got[i].clone()] for i, s in enumerate(slots)}
    for t in range(STEPS):
        toks = torch.zeros(dec.batch, dtype=torch.int64)
        for s in slots:
            toks[s] = seqs[s][FRESH[s] + t]
        lg = dec.step(toks)
        for s in slots:
            rows[s].append(lg[s].clone())
    assert dec.positions == [FRESH[s] + STEPS for s in range(4)]
    return {s: torch.stack(r) for s, r in rows.items()}


def _gather(dec, slot):
    """Slot's k / v [n_layers, n_kv, pos, d] from either layout."""
    p = dec.positions[slot]
    if dec._pages is None:
        return dec.k_cache[:, slot, :, :p], dec.v_cache[:, slot, :, :p]
    pages = dec.block_table[slot, :-(-p // 64)].long()
    k = dec.k_cache[:, pages].permute(0, 2, 1, 3, 4).reshape(dec.n_layers, dec.n_kv, -1, dec.head_dim)[:, :, :p]
    v = dec.v_cache[:, pages].permute(0, 2, 1, 3, 4).reshape(dec.n_layers, dec.n_kv, -1, dec.head_dim)[:, :, :p]
    return k, v


@pytest.mark.parametrize("kind,dtype", CASES, ids=[f"{k}-{d}" for k, d in CASES])
def test_fresh_prompts_and_second_turns(banks, record, kind, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    max_len = _max_len(model)
    seqs = _ids(model.config.vocab_size, max_len, 4, seed=21)
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    worst = 0.0

    contiguous = BatchDecoder(model, max_len, 4)
    paged = BatchDecoder(model, max_len, 4, pages=4 * -(-max_len // 64))
    want = _fresh_run(contiguous, seqs)
    got = _fresh_run(paged, seqs)
    for s, n in FRESH.items():
        plan = [("extend", n)] + steps(STEPS)
        worst = max(worst, check_against_twin(want[s].double(), hf_schedule(dense, seqs[s], plan), twin_rows(twin, seqs[s], plan),
                                              f"slot {s}"))
        assert torch.equal(got[s], want[s]), f"slot {s}: the paged logits differ from the contiguous ones"
        for a, b in zip(_gather(paged, s), _gather(contiguous, s)):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"slot {s}: the paged cache differs"
    del paged

    # second turns: slots 0, 1, 2 live at 9, 5 and 12 (+3 steps); slots 2 and 0 get turns of 7 and 4 tokens in one call
    a, b, c = seqs[:3]
    dec = contiguous

    def run(with_turns):
        dec.reset()
        out = {0: [], 1: [], 2: []}
        lg = dec.extend_many([0, 1, 2], [a[:9], b[:5], c[:12]])
        for i in range(3):
            out[i].append(lg[i].clone())
        fed = {0: 9, 1: 5, 2: 12}
        for _ in range(3):
            lg = dec.step(torch.tensor([int(a[fed[0]]), int(b[fed[1]]), int(c[fed[2]]), 0]))
            for i in range(3):
                out[i].append(lg[i].clone())
                fed[i] += 1
        if with_turns:
            lg = dec.extend_many([2, 0], [c[15:22], a[12:16]])
            out[2].append(lg[0].clone())
            out[0].append(lg[1].clone())
            fed[2] += 7
            fed[0] += 4
        for _ in range(4):
            lg = dec.step(torch.tensor([int(a[fed[0]]), int(b[fed[1]]), int(c[fed[2]]), 0]))
            for i in range(3):
                out[i].append(lg[i].clone())
                fed[i] += 1
        return {i: torch.stack(o) for i, o in out.items()}

    plain, turned = run(False), run(True)
    assert torch.equal(plain[1].view(torch.int16), turned[1].view(torch.int16)), "slot 1 changed when slots 0 and 2 got turns"
    assert dec.positions == [9 + 3 + 4 + 4, 5 + 3 + 4, 12 + 3 + 7 + 4, -1]
    for i, (seq, first, turn) in {0: (a, 9, 4), 2: (c, 12, 7)}.items():
        plan = [("extend", first)] + steps(3) + [("extend", turn)] + steps(4)
        worst = max(worst, check_against_twin(turned[i].double(), hf_schedule(dense, seq, plan), twin_rows(twin, seq, plan),
                                              f"turned slot {i}"))
    record("worst_err_ratio", worst)


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_prompts_split_across_passes(banks, record, monkeypatch, paged, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank("A4")
    dt = DTYPES[dtype]
    model = build(bk, dt)
    a, b = _ids(model.config.vocab_size, MAX_LEN, 2, seed=5)
    monkeypatch.setattr(BatchDecoder, "EXTEND_CHUNK", 5)   # passes: a 0-4 | a 5-9 | a 10-14 | a 15-16 b 0-2 | b 3-7 | b 8
    dec = BatchDecoder(model, MAX_LEN, 3, pages=6 if paged else None)
    lg = dec.extend_many([1, 0], [a[:17], b[:9]])
    rows = {1: [lg[0].clone()], 0: [lg[1].clone()]}
    for t in range(4):
        out = dec.step(torch.tensor([int(b[9 + t]), int(a[17 + t]), 0]))
        rows[1].append(out[1].clone())
        rows[0].append(out[0].clone())
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    worst = 0.0
    for slot, seq, n in ((1, a, 17), (0, b, 9)):
        plan = [("extend", n)] + steps(4)
        worst = max(worst, check_against_twin(torch.stack(rows[slot]).double(), hf_schedule(dense, seq, plan), twin_rows(twin, seq, plan),
                                              f"slot {slot}"))
    record("worst_err_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_forked_slots_take_different_turns(banks, record, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank("C")
    dt = DTYPES[dtype]
    model = build(bk, dt)
    p, ta, tb = _ids(model.config.vocab_size, MAX_LEN, 3, seed=9)
    dec = BatchDecoder(model, MAX_LEN, 3, pages=6)
    first = dec.extend(0, p[:70]).clone()   # one full page and a partial one
    dec.fork(0, 2)
    shared = int(dec.block_table[0, 0])
    assert int(dec.block_table[2, 0]) == shared
    k0, v0 = dec.k_cache[:, shared].clone(), dec.v_cache[:, shared].clone()
    lg = dec.extend_many([0, 2], [ta[:6], tb[:11]])
    assert torch.equal(dec.k_cache[:, shared].view(torch.int16), k0.view(torch.int16))
    assert torch.equal(dec.v_cache[:, shared].view(torch.int16), v0.view(torch.int16))
    rows = {0: [first, lg[0].clone()], 2: [first, lg[1].clone()]}
    for t in range(3):
        out = dec.step(torch.tensor([int(ta[6 + t]), 0, int(tb[11 + t])]))
        rows[0].append(out[0].clone())
        rows[2].append(out[2].clone())
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    worst = 0.0
    for slot, turn, n in ((0, ta, 6), (2, tb, 11)):
        seq = torch.cat([p[:70], turn])
        plan = [("extend", 70), ("extend", n)] + steps(3)
        worst = max(worst, check_against_twin(torch.stack(rows[slot]).double(), hf_schedule(dense, seq, plan), twin_rows(twin, seq, plan),
                                              f"slot {slot}"))
    record("worst_err_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_eight_prompts_on_the_7b_layer(banks, record, dtype):
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank("B")
    dt = DTYPES[dtype]
    model = build(bk, dt)
    seqs = _ids(model.config.vocab_size, 258, 8, seed=4)
    dec = BatchDecoder(model, 264, 8)
    lg = dec.extend_many(list(range(8)), [s[:256] for s in seqs])
    rows = [[lg[i].clone()] for i in range(8)]
    for t in range(2):
        out = dec.step(torch.stack([s[256 + t] for s in seqs]).cpu())
        for i in range(8):
            rows[i].append(out[i].clone())
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    plan = [("extend", 256)] + steps(2)
    worst = 0.0
    for i, s in enumerate(seqs):
        worst = max(worst, check_against_twin(torch.stack(rows[i]).double(), hf_schedule(dense, s, plan), twin_rows(twin, s, plan),
                                              f"prompt {i}"))
    record("worst_err_ratio", worst)


@pytest.mark.parametrize("paged", [False, True])
def test_rejections_change_nothing(banks, paged):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), torch.float16)
    ids = torch.arange(40).cuda()
    dec = BatchDecoder(model, 24, 3, pages=2 if paged else None)   # paged: one page per slot, one left after slot 0's
    dec.extend(0, ids[:10])

    def state():
        s = [dec.positions, dec.pos.tolist(), dec.k_cache.clone(), dec.v_cache.clone(), dec.free_pages]
        return s + ([dec.block_table.clone()] if paged else [])

    before = state()
    bad = [
        ([0, 1], [ids[:3]], ValueError, "2 slots and 1 prompts; want one length in 1..3"),
        ([], [], ValueError, "0 slots and 0 prompts"),
        ([0, 1, 2, 0], [ids[:1]] * 4, ValueError, "4 slots and 4 prompts"),
        ([1, 3], [ids[:3], ids[:3]], ValueError, "slot must be an int in 0..2"),
        ([1, 1], [ids[:3], ids[:3]], ValueError, "the slots must be distinct"),
        ([1, 2], [ids[:3], ids[:0]], ValueError, "prompt 1: input_ids must be a non-empty 1-D"),
        ([1, 2], [ids[None, :3], ids[:3]], ValueError, "prompt 0: input_ids must be a non-empty 1-D"),
        ([1, 2], [ids[:3], ids[:3].float()], ValueError, "prompt 1: input_ids must hold integer token ids"),
        ([2, 0], [ids[:3], ids[:15]], ValueError, "prompt 1: 15 tokens at position 10 need 25 cache positions, max_len is 24"),
    ]
    if paged:  # slots 1 and 2 need a page each, one is free
        bad.append(([2, 0, 1], [ids[:3], ids[:2], ids[:3]], RuntimeError, r"slot\(s\) \[0, 1, 2\]"))
    for slots, prompts, exc, msg in bad:
        with pytest.raises(exc, match=msg):
            dec.extend_many(slots, prompts)
        after = state()
        assert after[0] == before[0] and after[1] == before[1] and after[4] == before[4], msg
        for x, y in zip(after[2:], before[2:]):
            if isinstance(x, torch.Tensor):
                assert torch.equal(x, y), msg
    lg = dec.extend_many([2, 0], [ids[:14], ids[:14]])   # exactly max_len for slot 0
    assert lg.shape == (2, model.config.vocab_size)
    assert dec.positions == [24, -1, 14]
