#!/usr/bin/env python3
"""Admitting several prompts at once: BatchDecoder.extend_many against one BatchDecoder.extend per prompt, on the synthetic LLaMA-7B
w4-s45 of decoder_timing.py (32 layers, fp16, random QuantLinearLUT projections, dense fp16 lm_head, 32 heads of 128), batch 16.

  (a) admission: K in {2, 4, 8, 16} prompts of L in {16, 128, 512} tokens into idle slots 0 .. K-1, K sequential extend calls against
      one extend_many, for the contiguous and the paged layout;
  (b) one layer's attention alone: quant_cuda.attn_extend_batch on K segments against the K attn_extend launches it replaces, at
      K in {2, 4, 8, 16} segments of 16 and of 128 fresh tokens, and a mix of 4 fresh 16-token prompts with 4 turns of 16 tokens on
      4096-token histories (the splits differ: two attention launches).
Every arm runs blocks timed with CUDA events and a device synchronise; the arms alternate block by block (a reset of the slots between
blocks, outside the timed window), and the median of 5 blocks is kept.  The first line names the card, its power limit and max SM
clock (nvidia-smi, read-only query).

    python tests/perf/batch_extend_timing.py
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import make_model, time_blocks  # noqa: E402

BATCH = 16
KS = (2, 4, 8, 16)
LS = (16, 128, 512)
HISTORY = 4096


def admission(dec, ids, layout):
    for L in LS:
        for K in KS:
            prompts = [ids[k, :L] for k in range(K)]

            def sequential():
                for k in range(K):
                    dec.extend(k, prompts[k])

            def many():
                dec.extend_many(list(range(K)), prompts)
            t = time_blocks({"sequential": (dec.reset, sequential, 1), "extend_many": (dec.reset, many, 1)}, blocks=5)
            print(json.dumps({"kind": "admission", "layout": layout, "K": K, "L": L, "sequential_ms": round(t["sequential"], 2),
                              "extend_many_ms": round(t["extend_many"], 2), "speedup": round(t["sequential"] / t["extend_many"], 2)}),
                  flush=True)


def attention(nh, nkv, d, scale):
    from squeezellm_b200.quant import quant_cuda
    cap = HISTORY + 128
    g = torch.Generator(device="cuda").manual_seed(3)
    k = torch.randn(BATCH, nkv, cap, d, generator=g, device="cuda").half()
    v = torch.randn(BATCH, nkv, cap, d, generator=g, device="cuda").half()
    inv = 1.0 / (10000.0 ** (np.arange(0, d, 2, dtype=np.float64) / d))
    ang = np.arange(cap, dtype=np.float64)[:, None] * inv[None, :]
    cos, sin = torch.from_numpy(np.cos(ang)).float().cuda(), torch.from_numpy(np.sin(ang)).float().cuda()
    mixes = [(f"{K}x(0,{T})", [(0, T)] * K) for T in (16, 128) for K in KS]
    mixes.append(("4x(0,16)+4x(4096,16)", [(0, 16)] * 4 + [(HISTORY, 16)] * 4))
    nothing = lambda: None  # noqa: E731
    for name, mix in mixes:
        rows = sum(T for _, T in mix)
        qkv = torch.randn(rows, (nh + 2 * nkv) * d, generator=g, device="cuda").half()
        out = torch.empty(rows, nh * d, dtype=torch.float16, device="cuda")
        slots, starts, ts = list(range(len(mix))), [s for s, _ in mix], [T for _, T in mix]
        r0 = np.cumsum([0] + ts).tolist()

        def batch():
            quant_cuda.attn_extend_batch(qkv, slots, starts, ts, cos, sin, k, v, out, nh, nkv, scale)

        def single():
            for i in range(len(mix)):
                quant_cuda.attn_extend(qkv[r0[i]:r0[i + 1]], starts[i], cos, sin, k[i], v[i], out[r0[i]:r0[i + 1]], nh, nkv, scale)
        t = time_blocks({"batch": (nothing, batch, 50), "single": (nothing, single, 50)}, blocks=5)
        splits = sorted({quant_cuda.attn_extend_splits(nh, nkv, T, s) for s, T in mix})
        print(json.dumps({"kind": "attention", "mix": name, "splits": splits, "batch_us": round(1e3 * t["batch"], 2),
                          "single_launches_us": round(1e3 * t["single"], 2), "speedup": round(t["single"] / t["batch"], 2)}), flush=True)


def main():
    from squeezellm_b200.runtime import BatchDecoder
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    model = make_model(32)
    g = torch.Generator(device="cuda").manual_seed(7)
    ids = torch.randint(0, model.config.vocab_size, (BATCH, max(LS)), generator=g, device="cuda")
    max_len = max(LS)
    for layout, pages in (("contiguous", None), ("paged", BATCH * -(-max_len // 64))):
        dec = BatchDecoder(model, max_len, BATCH, pages=pages)
        admission(dec, ids, layout)
        nh, nkv, d, scale = dec.n_heads, dec.n_kv, dec.head_dim, dec.scale
        del dec
        torch.cuda.empty_cache()
    attention(nh, nkv, d, scale)


if __name__ == "__main__":
    main()
