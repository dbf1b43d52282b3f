#!/usr/bin/env python3
"""Speculative decoding's cost: runtime.SequenceDecoder(speculate=K) on the synthetic LLaMA-7B w4-s45 of decoder_timing.make_model
(32 layers, fp16, dense fp16 lm_head), with the KV cache holding random values.

  (1) attention  one layer's attention for T in {2, 4, 8, 16} new tokens at context ctx in {128, 1024, 4096}, for the 7B MHA layer
                 (32, 32, 128) and a GQA layer (32, 8, 128): quant_cuda.attn_verify, quant_cuda.attn_extend at the same start and T,
                 and one quant_cuda.attn_decode; us per call and the K / V bytes read over the time as a share of the data sheet's
                 3.35 TB/s
  (2) verify     the verify graph (T = K + 1 rows) against one step of the ordinary graph, ms, at the same contexts; the break-even
                 accepted drafts per verify, verify / step - 1 (a verify of n accepted drafts emits n + 1 tokens)
  (3) generate   tokens/s of generate() after a 128-token prompt: plain, and K in {3, 7} with an oracle drafter cut to accept 0, K/2
                 and K drafts per verify (the rest replaced by wrong ids); and a drafter that never proposes (every iteration an ordinary
                 step: the speculative loop's host overhead).  The oracle's tokens are the speculative decoder's own: generate with
                 the oracle is rerun on its own output until the two agree (the verify rows round differently from the step graph, so
                 plain generate's tokens are not what a verify draws).  The accepted drafts per verify reached are printed with each arm.
Arms of (1) and (2) run blocks of calls timed with CUDA events, alternating block by block, median of 7 blocks.  (3) times whole
generate() calls with a host clock after a device synchronise, the prefill taken out (a 1-token generate of the same prompt), median
of 3.  The first line names the card, its power limit and max SM clock (nvidia-smi, read-only query).

    python tests/perf/speculative_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import HBM, make_model, time_blocks  # noqa: E402

CONTEXTS = (128, 1024, 4096)
TOKENS = (2, 4, 8, 16)
BLOCK = 16


def emit(row):
    print(json.dumps(row), flush=True)


def rule(nh, nkv, T):
    """sqllm_attn_verify_splits: the split count before the launch lowers it until every cluster is resident."""
    clusters = nkv * -(-T * (nh // nkv) // 8)
    return max(1, min(8, torch.cuda.get_device_properties(0).multi_processor_count // clusters))


def attention(qc, contexts):
    d, cap = 128, max(contexts) + 64
    g = torch.Generator(device="cuda").manual_seed(3)
    for nh, nkv in ((32, 32), (32, 8)):
        kc = torch.randn(nkv, cap, d, generator=g, device="cuda").half()
        vc = torch.randn(nkv, cap, d, generator=g, device="cuda").half()
        inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, device="cuda").double() / d))
        ang = torch.arange(cap, device="cuda").double()[:, None] * inv[None]
        cos, sin = ang.cos().float().contiguous(), ang.sin().float().contiguous()
        for ctx in contexts:
            pos = torch.tensor([ctx], dtype=torch.int32, device="cuda")
            for T in TOKENS:
                qkv = torch.randn(T, (nh + 2 * nkv) * d, generator=g, device="cuda").half()
                out = torch.empty(T, nh * d, dtype=torch.float16, device="cuda")
                q1 = qkv[0].contiguous()
                o1 = out[0]
                arms = {
                    "verify": (lambda: None, lambda: qc.attn_verify(qkv, pos, cos, sin, kc, vc, out, nh, nkv, d ** -0.5), 200),
                    "extend": (lambda: None, lambda: qc.attn_extend(qkv, ctx, cos, sin, kc, vc, out, nh, nkv, d ** -0.5), 200),
                    "decode": (lambda: None, lambda: qc.attn_decode(q1, pos, cos, sin, kc, vc, o1, nh, nkv, d ** -0.5), 200),
                }
                t = time_blocks(arms)
                row = {"kind": "attention", "heads": [nh, nkv, d], "ctx": ctx, "T": T,
                       "splits_verify": qc.attn_verify_splits(nh, nkv, T, d, torch.float16), "splits_rule": rule(nh, nkv, T),
                       "verify_beats_extend": t["verify"] < t["extend"]}
                for a, n_pos in (("verify", ctx + T), ("extend", ctx + T), ("decode", ctx + 1)):
                    row[f"{a}_us"] = round(1e3 * t[a], 2)
                    row[f"{a}_share_of_3.35TBps"] = round(2 * nkv * n_pos * d * 2 / (t[a] * 1e-3) / HBM, 3)
                emit(row)
        del kc, vc
        torch.cuda.empty_cache()


def fill_random(t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for i in range(t.shape[0]):
        t[i].copy_(torch.randn(t[i].shape, generator=g, device="cuda").half())


def at(dec, ctx):
    dec.pos.fill_(ctx)
    dec._pos = [ctx]
    dec.tok.fill_(1)


def verify_steps(model, contexts, Ks):
    from squeezellm_b200.runtime import SequenceDecoder
    max_len = max(contexts) + 2 * BLOCK + 16
    decs = {}
    for K in Ks:
        decs[K] = SequenceDecoder(model, max_len, speculate=K)
        fill_random(decs[K].k_cache, 5)
        fill_random(decs[K].v_cache, 6)
    base = decs[Ks[0]]
    for ctx in contexts:
        arms = {"step": (lambda: at(base, ctx), base.graph.replay, BLOCK)}
        for K, dec in decs.items():
            arms[f"verify_T{K + 1}"] = ((lambda dec=dec: at(dec, ctx)), dec.vgraph.replay, BLOCK)
        t = time_blocks(arms)
        for K in Ks:
            v = t[f"verify_T{K + 1}"]
            emit({"kind": "verify_step", "ctx": ctx, "T": K + 1, "verify_ms": round(v, 3), "step_ms": round(t["step"], 3),
                  "verify_over_step": round(v / t["step"], 3), "break_even_accepted": round(v / t["step"] - 1, 2)})
    decs.clear()
    torch.cuda.empty_cache()


def timed(fn, reps=3):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return statistics.median(out)


def generate_rates(model, n_new, Ks):
    from squeezellm_b200.runtime import SequenceDecoder
    vocab = model.config.vocab_size
    prompt = torch.randint(0, vocab, (1, 128), generator=torch.Generator().manual_seed(1)).cuda()
    plain = SequenceDecoder(model, 128 + n_new + 16)
    ref = plain.generate(prompt, n_new)[0, 128:].tolist()
    prefill = timed(lambda: plain.generate(prompt, 1))
    t = timed(lambda: plain.generate(prompt, n_new)) - prefill
    emit({"kind": "generate", "arm": "plain", "new_tokens": n_new, "tokens_per_s": round((n_new - 1) / t, 1)})
    del plain
    for K in Ks:
        dec = SequenceDecoder(model, 128 + n_new + 16, speculate=K)
        own, rounds = ref, 0
        while rounds < 8:  # the fixed point: the oracle proposes exactly what the decoder draws, so every draft is accepted
            rounds += 1
            nxt = dec.generate(prompt, n_new, draft=lambda toks, own=own: own[len(toks) - 128:len(toks) - 128 + K])[0, 128:].tolist()
            if nxt == own:
                break
            own = nxt
        emit({"kind": "oracle_fixed_point", "K": K, "rounds": rounds, "reached": nxt == own})
        for a in sorted({0, K // 2, K}):
            def oracle(toks, a=a, K=K):
                n = len(toks) - 128
                right = own[n:n + a]
                return right + [(w + 1) % vocab for w in own[n + a:n + K]]
            pre = timed(lambda: dec.generate(prompt, 1, draft=oracle))
            t = timed(lambda: dec.generate(prompt, n_new, draft=oracle)) - pre
            out = dec.generate(prompt, n_new, draft=oracle)[0, 128:].tolist()
            st = dec.spec_stats
            emit({"kind": "generate", "arm": f"oracle_accept_{a}_of_{K}", "K": K, "new_tokens": n_new, "tokens_per_s": round((n_new - 1) / t, 1),
                  "stats": st, "accepted_per_verify": round(st["accepted"] / max(1, st["verifies"]), 2),
                  "same_tokens_as_oracle": out == own, "same_tokens_as_plain": out == ref})
        pre = timed(lambda: dec.generate(prompt, 1, draft=lambda toks: []))
        t = timed(lambda: dec.generate(prompt, n_new, draft=lambda toks: [])) - pre
        emit({"kind": "generate", "arm": "no_drafts", "K": K, "new_tokens": n_new, "tokens_per_s": round((n_new - 1) / t, 1)})
        t = timed(lambda: dec.generate(prompt, n_new)) - pre
        emit({"kind": "generate", "arm": "prompt_lookup", "K": K, "new_tokens": n_new, "tokens_per_s": round((n_new - 1) / t, 1),
              "stats": dec.spec_stats})
        del dec
        torch.cuda.empty_cache()


def main():
    quick = "--quick" in sys.argv
    from squeezellm_b200.quant import quant_cuda as qc
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    emit({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]})
    contexts = (128, 1024) if quick else CONTEXTS
    attention(qc, contexts)
    model = make_model(2 if quick else 32)
    verify_steps(model, contexts, (1, 3, 7, 15))
    generate_rates(model, 32 if quick else 128, (3, 7))


if __name__ == "__main__":
    main()
