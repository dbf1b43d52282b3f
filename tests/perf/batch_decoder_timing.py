#!/usr/bin/env python3
"""Several sequences decoded at once: runtime.BatchDecoder on the synthetic LLaMA-7B w4-s45 of decoder_timing.make_model (32 layers,
fp16, dense fp16 lm_head), with every row's KV cache holding random values and every row at the same context.

Sweep: batch B in {2, 4, 8, 16, 32} and runtime.SequenceDecoder as B = 1, at contexts 128, 1024 and 4096.  A configuration whose
caches would exceed MAX_CACHE_GB is skipped and reported as such.  Per configuration:
  (a) step       the decoder's graph: ms per step, aggregate tokens/s (B / step) and per-sequence tokens/s (1 / step)
  (b) attention  one layer's attention alone at position ctx for every row: quant_cuda.attn_decode_batch against B single-row
                 quant_cuda.attn_decode calls on the rows' slices and against scaled_dot_product_attention on the same caches, with the
                 K / V bytes read per call over the time, as a share of the data sheet's 3.35 TB/s
Every arm runs blocks of steps (calls) timed with CUDA events; the arms of one configuration alternate block by block, the positions
are set back to the context before each block, and the median of 7 blocks is kept.  The first line names the card, its power limit
and max SM clock (nvidia-smi, read-only query).

--profile (a run of its own): a torch.profiler trace of STEPS_PROFILED steps of B = 8 at context 1024, kernel time split into the
projections (the LUT-GEMV kernels), the attention and everything else (norms, SiLU, residual adds, embedding, lm_head, argmax).

    python tests/perf/batch_decoder_timing.py [--quick] [--profile]
"""
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import HBM, make_model, time_blocks  # noqa: E402

CONTEXTS = (128, 1024, 4096)
BATCHES = (1, 2, 4, 8, 16, 32)
BLOCK = 16          # steps per timed block
MAX_CACHE_GB = 40   # k + v caches of all layers and rows
STEPS_PROFILED = 8


def cache_gb(n_layers, B, max_len, nkv=32, d=128):
    return 2 * n_layers * B * nkv * max_len * d * 2 / 1e9


def fill_random(t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for i in range(t.shape[0]):  # one layer at a time: no full-size fp32 temporary
        t[i].copy_(torch.randn(t[i].shape, generator=g, device="cuda").half())


def decoder_for(model, B, max_len):
    from squeezellm_b200.runtime import BatchDecoder, SequenceDecoder
    dec = SequenceDecoder(model, max_len) if B == 1 else BatchDecoder(model, max_len, B)
    fill_random(dec.k_cache, 5)
    fill_random(dec.v_cache, 6)
    return dec


def set_positions(dec, B, ctx):
    dec.pos.fill_(ctx)
    dec._pos = [ctx] * B
    dec.tok.fill_(1)


def attention_arms(dec, B, ctx, qc, g):
    """(b): the three ways to run one layer's attention for B rows at position ctx."""
    nh, nkv, d = dec.n_heads, dec.n_kv, dec.head_dim
    kc, vc = dec.k_cache[0], dec.v_cache[0]
    if B == 1:
        kc, vc = kc[None], vc[None]
    qkv = torch.randn(B, (nh + 2 * nkv) * d, generator=g, device="cuda").half()
    out = torch.empty(B, nh * d, dtype=torch.float16, device="cuda")
    pos = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
    pos1 = pos[:1]
    qh = qkv[:, :nh * d].view(B, nh, 1, d)

    def batch():
        qc.attn_decode_batch(qkv, pos, dec.rope_cos, dec.rope_sin, kc, vc, out, nh, nkv, dec.scale)

    def singles():
        for b in range(B):
            qc.attn_decode(qkv[b], pos1, dec.rope_cos, dec.rope_sin, kc[b], vc[b], out[b], nh, nkv, dec.scale)

    def sdpa():
        F.scaled_dot_product_attention(qh, kc[:, :, :ctx + 1], vc[:, :, :ctx + 1], scale=dec.scale)
    return {"batch": batch, "singles": singles, "sdpa": sdpa}


def main():
    quick = "--quick" in sys.argv
    from squeezellm_b200.quant import quant_cuda as qc
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    n_layers = 2 if quick else 32
    contexts = (128, 1024) if quick else CONTEXTS
    batches = (1, 2, 8) if quick else BATCHES
    model = make_model(n_layers)
    g = torch.Generator(device="cuda").manual_seed(7)
    if "--profile" in sys.argv:
        return profile(model, 8, 1024, n_layers)
    for B in batches:
        fits = [c for c in contexts if cache_gb(n_layers, B, c + 2 * BLOCK) <= MAX_CACHE_GB]
        for c in contexts:
            if c not in fits:
                print(json.dumps({"kind": "skipped", "B": B, "ctx": c, "cache_GB": round(cache_gb(n_layers, B, c + 2 * BLOCK), 1)}), flush=True)
        if not fits:
            continue
        max_len = max(fits) + 2 * BLOCK
        dec = decoder_for(model, B, max_len)
        for ctx in fits:
            att = attention_arms(dec, B, ctx, qc, g)
            n_att = max(10, 200 // B)
            t = time_blocks({"step": (lambda: set_positions(dec, B, ctx), dec.graph.replay, BLOCK),
                             "attn_batch": (lambda: None, att["batch"], n_att), "attn_singles": (lambda: None, att["singles"], n_att),
                             "attn_sdpa": (lambda: None, att["sdpa"], n_att)})
            kv_bytes = B * 2 * dec.n_kv * (ctx + 1) * dec.head_dim * 2
            row = {"kind": "config", "B": B, "ctx": ctx, "decoder": "SequenceDecoder" if B == 1 else "BatchDecoder",
                   "ms_per_step": round(t["step"], 3), "tokens_per_s": round(B * 1e3 / t["step"], 1),
                   "tokens_per_s_per_seq": round(1e3 / t["step"], 1),
                   "splits_batch": qc.attn_decode_batch_splits(dec.n_heads, dec.n_kv, B), "splits_single": qc.attn_decode_splits(dec.n_heads, dec.n_kv)}
            for a in ("batch", "singles", "sdpa"):
                ms = t["attn_" + a]
                row[f"attn_{a}_us"] = round(1e3 * ms, 2)
                row[f"attn_{a}_share_of_3.35TBps"] = round(kv_bytes / (ms * 1e-3) / HBM, 3)
            print(json.dumps(row), flush=True)
        del dec
        torch.cuda.empty_cache()


def profile(model, B, ctx, n_layers):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof
    dec = decoder_for(model, B, ctx + STEPS_PROFILED + 2 * BLOCK)
    set_positions(dec, B, ctx)
    for _ in range(3):
        dec.graph.replay()
    set_positions(dec, B, ctx)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as p:
        for _ in range(STEPS_PROFILED):
            dec.graph.replay()
        torch.cuda.synchronize()
    split, names = {"projections": 0.0, "attention": 0.0, "glue": 0.0}, {}
    for e in p.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if not us or e.key.startswith(("ProfilerStep", "cudaGraph")) or e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = e.key
        part = "projections" if "lutgemv" in k or "rows::" in k else "attention" if "attn" in k else "glue"
        split[part] += us / STEPS_PROFILED
        names[k[:90]] = round(us / STEPS_PROFILED, 1)
    total = sum(split.values())
    print(json.dumps({"kind": "profile", "B": B, "ctx": ctx, "layers": n_layers, "us_per_step": {k: round(v, 1) for k, v in split.items()},
                      "share": {k: round(v / total, 3) for k, v in split.items()} if total else None}), flush=True)
    print(json.dumps({"kind": "profile_kernels", "us_per_step": dict(sorted(names.items(), key=lambda kv: -kv[1])[:25])}), flush=True)


if __name__ == "__main__":
    main()
