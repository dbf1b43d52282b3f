"""runtime.BatchDecoder on the GPU: several sequences decoded at once, one CUDA graph per step, against the fp64 twin of
test_decoder_gpu.py (same models, same banks of oracle layers, same criteria, applied per row).

Kinds A4 (Llama, 8 heads / 2 KV heads), C (Qwen2 with q/k/v bias and a quantized lm_head) and H64 (head_dim 64), in fp16 and bf16 at
batch 2 and 5, the 7B-shaped layer B and G7 (7 query heads per KV head) at batch 5, and MQA (16 heads on one KV head) at batch 2;
the rows hold prompts of different lengths (1, 9, 17, 5, 12 tokens):
  * teacher-forced decode for 40 steps: every row's logits at most twice as far (max norm) from the twin's as a dense model of the same
    dtype decoding the same tokens with HF's cache;
  * greedy generate matches the twin's greedy tokens, row by row, up to the twin's first near-tie;
  * a row's logits are bitwise unchanged when the other rows hold different prompts or are idle (every op of a step is row-wise);
  * a rerun after reset() gives bitwise-equal tokens for the prompts of 2 or more tokens (a 1-token prompt's prefill runs the one-row
    route, which adds in arrival order: its tokens are checked against the twin only);
  * model(ids) gives the same logits after the decoder is built as before.
Besides: EOS on one row cuts and releases that row while the others run on; release() and prefill() of a new prompt mid-run gives it
the tokens it gets alone in a fresh decoder; a slot filled to exactly max_len works and one step more raises."""
import copy

import pytest
import torch

from test_decoder_gpu import DTYPES, bank, banks, build, hf_decode, twin_of  # noqa: F401  (banks: the module-scoped fixture)

pytestmark = pytest.mark.gpu

MAX_LEN = 64
STEPS = 40
LENS = [1, 9, 17, 5, 12]
CASES = ([(k, dt, B) for k in ("A4", "C", "H64") for dt in DTYPES for B in (2, 5)] + [("B", dt, 5) for dt in DTYPES]
         + [(k, dt, B) for k, B in (("G7", 5), ("MQA", 2)) for dt in DTYPES])


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


def teacher_forced(dec, seqs, lens):
    """Logits [rows, STEPS + 1, vocab] (fp64): each row's prefill, then STEPS steps feeding seqs[b][T_b + t]; rows past len(seqs) idle."""
    out = [[dec.prefill(b, s[:T]).double()] for b, (s, T) in enumerate(zip(seqs, lens))]
    for t in range(STEPS):
        toks = torch.zeros(dec.batch, dtype=torch.int64)
        for b, (s, T) in enumerate(zip(seqs, lens)):
            toks[b] = s[T + t]
        logits = dec.step(toks)
        for b in range(len(seqs)):
            out[b].append(logits[b].double().clone())
    return [torch.stack(o) for o in out]


@pytest.mark.parametrize("kind,dtype,B", CASES, ids=[f"{k}-{d}-B{b}" for k, d, b in CASES])
def test_batch_decoder_against_the_fp64_twin(banks, record, kind, dtype, B):
    from squeezellm_b200.runtime import BatchDecoder
    bk = bank(kind)
    dt = DTYPES[dtype]
    model = build(bk, dt)
    vocab = model.config.vocab_size
    gen = torch.Generator().manual_seed(11)
    lens = LENS[:B]
    seqs = [torch.randint(0, vocab, (T + STEPS,), generator=gen).cuda() for T in lens]
    with torch.no_grad():
        before = model(input_ids=seqs[1][None, :9]).logits.clone()
    dec = BatchDecoder(model, MAX_LEN, B)
    with torch.no_grad():
        after = model(input_ids=seqs[1][None, :9]).logits
    assert torch.equal(before, after), "the model's outputs changed when the decoder was built"
    assert dec.positions == [-1] * B
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)

    lq = teacher_forced(dec, seqs, lens)
    assert dec.positions == [T + STEPS for T in lens]
    worst, err_rows = 0.0, []
    for b, (s, T) in enumerate(zip(seqs, lens)):
        with torch.no_grad():
            lt = twin(input_ids=s[None]).logits[0, T - 1:].double()
        ld = hf_decode(dense, s, T)
        err_q = (lq[b] - lt).abs().amax(dim=1)
        err_d = (ld - lt).abs().amax(dim=1)
        assert torch.isfinite(lq[b]).all()
        assert (err_q <= 2 * err_d).all(), (b, T, err_q.tolist(), err_d.tolist())
        worst = max(worst, float((err_q / err_d).max()))
        err_rows.append(float(err_q.max()))
    record("worst_err_ratio", worst)

    # row independence: row 1 (9 tokens: its prefill runs the multi-row route, bit-reproducible) with the other rows holding other
    # prompts, then idle; its step logits bitwise equal to the first run's
    other = [torch.randint(0, vocab, (T + STEPS,), generator=gen).cuda() for T in lens]
    for variant in ("other", "idle"):
        dec.reset()
        if variant == "other":
            rows = [seqs[1] if b == 1 else other[b] for b in range(B)]
            again = teacher_forced(dec, rows, lens)[1]
        else:
            dec.prefill(1, seqs[1][:9])
            again = [dec.step(torch.cat([seqs[1][9 + t:10 + t]] * B))[1].double().clone() for t in range(STEPS)]
            again = torch.stack([lq[1][0]] + again)
            assert dec.positions == [-1 if b != 1 else 9 + STEPS for b in range(B)]
        assert torch.equal(again[1:], lq[1][1:]), f"row 1's logits changed when the other rows were {variant}"

    # greedy, twice: every row against the twin's greedy tokens up to its first near-tie; the rerun bitwise equal (prompts >= 2 tokens)
    n_new = 20
    prompts = [s[:T] for s, T in zip(seqs, lens)]
    runs = []
    for _ in range(2):
        dec.reset()
        runs.append([o[T:].tolist() for o, T in zip(dec.generate(prompts, n_new), lens)])
    for b, T in enumerate(lens):
        if T >= 2:
            assert runs[0][b] == runs[1][b], (b, runs[0][b], runs[1][b])
        tol = 2 * err_rows[b]
        cur = prompts[b].clone()
        with torch.no_grad():
            for j in range(n_new):
                logit = twin(input_ids=cur[None]).logits[0, -1]
                top2 = torch.topk(logit, 2).values
                if float(top2[0] - top2[1]) < tol:
                    break
                want = int(logit.argmax())
                assert runs[0][b][j] == want and runs[1][b][j] == want, (b, T, j, runs, want)
                cur = torch.cat([cur, torch.tensor([want], device=cur.device)])
        record(f"greedy_agree_row{b}", j)


def test_eos_cuts_and_releases_one_row(banks):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), torch.float16)
    dec = BatchDecoder(model, MAX_LEN, 3)
    prompts = [torch.arange(5).cuda(), torch.arange(10, 19).cuda(), torch.arange(30, 33).cuda()]
    full = [o[len(p):].tolist() for o, p in zip(dec.generate(prompts, 30), prompts)]
    eos = full[1][11]
    cut = [f[:f.index(eos) + 1] if eos in f else f for f in full]
    assert len(cut[1]) <= 12
    outs = dec.generate(prompts, 30, eos_token_id=eos)
    got = [o[len(p):].tolist() for o, p in zip(outs, prompts)]
    assert got == cut
    assert dec.positions[1] == -1, "the row that produced EOS was not released"
    for b in range(3):
        if len(cut[b]) == 30:  # a row without EOS ran to the end
            assert dec.positions[b] == len(prompts[b]) + 29


def test_continuous_batching(banks):
    """Slot 1 is released mid-run and refilled with a new prompt while slot 0 keeps going: the new prompt gets the tokens it gets alone
    in a fresh decoder, and slot 0 the tokens it gets without the swap."""
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), torch.float16)
    B, n_new = 3, 12
    p0, p1, p2 = torch.arange(3, 10).cuda(), torch.arange(40, 45).cuda(), torch.arange(70, 81).cuda()
    alone = BatchDecoder(model, MAX_LEN, B)
    want0 = alone.generate([p0], 5 + n_new)[0][len(p0):].tolist()
    want2 = alone.generate([p2], n_new)[0][len(p2):].tolist()
    del alone

    dec = BatchDecoder(model, MAX_LEN, B)
    toks = torch.zeros(B, dtype=torch.int64, device="cuda")
    toks[0] = dec.prefill(0, p0).argmax()
    toks[1] = dec.prefill(1, p1).argmax()
    got0 = [int(toks[0])]
    for _ in range(5):
        toks = dec.step(toks).argmax(dim=-1)
        got0.append(int(toks[0]))
    dec.release(1)
    assert dec.positions == [len(p0) + 5, -1, -1]
    toks[1] = dec.prefill(1, p2).argmax()
    got2 = [int(toks[1])]
    for _ in range(n_new - 1):
        toks = dec.step(toks).argmax(dim=-1)
        got0.append(int(toks[0]))
        got2.append(int(toks[1]))
    assert got2 == want2
    assert got0 == want0[:len(got0)]


def test_cache_limits(banks):
    from squeezellm_b200.runtime import BatchDecoder
    model = build(bank("A4"), torch.float16)
    dec = BatchDecoder(model, 20, 2)
    dec.prefill(0, torch.arange(17).cuda())
    dec.prefill(1, torch.arange(5).cuda())
    for t in range(3):
        logits = dec.step([t, t])
    assert dec.positions == [20, 8] and torch.isfinite(logits).all()
    with pytest.raises(RuntimeError, match=r"the cache of slot\(s\) \[0\] is full \(max_len=20\)"):
        dec.step([0, 0])
    dec.release(0)
    dec.step([0, 0])
    assert dec.positions == [-1, 9]
    with pytest.raises(ValueError, match="need 21 cache positions, max_len is 20"):
        dec.generate([torch.arange(17)], 5)
    out = dec.generate([torch.arange(17), torch.arange(4)], 4)  # 17 + 3 steps: exactly max_len
    assert [o.shape[0] for o in out] == [21, 8] and dec.positions == [20, 7]
    dec.reset()
    assert dec.positions == [-1, -1]
    with pytest.raises(ValueError, match="21 prompt tokens"):
        dec.prefill(0, torch.arange(21).cuda())
