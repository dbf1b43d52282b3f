#!/usr/bin/env python3
"""Prompts on the decoder's own kernels: SequenceDecoder.extend against SequenceDecoder.prefill (the model's own HF forward and a copy
of its cache) on the synthetic LLaMA-7B w4-s45 of decoder_timing.py (32 layers, fp16, random QuantLinearLUT projections, dense fp16
lm_head, 32 heads, head_dim 128).

  (a) time to first token: prefill against extend from position 0, at 16 / 128 / 512 / 2048 prompt tokens;
  (b) multi-turn append: 64 tokens appended to a 4096-token history by extend, against a prefill of all 4160 tokens (what a user
      without extend runs);
  (c) one layer's attention alone: quant_cuda.attn_extend (its append and attention launches) against scaled_dot_product_attention
      on the same q, K, V with a bottom-right causal mask, at (start 0, T 2048) and (start 4096, T 64): achieved TFLOP/s counting the
      algorithmic causal FLOPs (4 d per query-key pair at or below the diagonal, per head) and their share of the data sheet's 989
      dense fp16 TFLOP/s; for the short chunk also the K / V bytes over the time as a share of 3.35 TB/s.
Every arm runs blocks of calls timed with CUDA events; the arms alternate block by block, and the median of the blocks is kept.  The
first line names the card, its power limit and max SM clock (nvidia-smi, read-only query).

    python tests/perf/extend_timing.py            # (a) - (c)
    python tests/perf/extend_timing.py --profile  # a torch.profiler table of one 2048-token extend, in a run of its own
"""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import make_model, time_blocks  # noqa: E402

HBM = 3.35e12
PEAK = 989e12
PROMPTS = (16, 128, 512, 2048)
HISTORY, TURN = 4096, 64


def causal_flops(nh, d, start, T):
    return 4 * d * nh * sum(start + t + 1 for t in range(T))


def main():
    from squeezellm_b200.quant import quant_cuda
    from squeezellm_b200.runtime import SequenceDecoder
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    model = make_model(32)
    dec = SequenceDecoder(model, HISTORY + TURN + 64)
    nh, nkv, d = dec.n_heads, dec.n_kv, dec.head_dim
    g = torch.Generator(device="cuda").manual_seed(7)
    ids = torch.randint(0, model.config.vocab_size, (HISTORY + TURN,), generator=g, device="cuda")

    if "--profile" in sys.argv:
        from torch.profiler import ProfilerActivity, profile
        dec.reset()
        dec.extend(ids[:2048])
        torch.cuda.synchronize()
        dec.reset()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            dec.extend(ids[:2048])
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=20), flush=True)
        return

    # (a) time to first token
    for T in PROMPTS:
        def prefill(T=T):
            dec.prefill(ids[:T])

        def extend(T=T):
            dec.reset()
            dec.extend(ids[:T])
        dec.reset()
        lp = dec.prefill(ids[:T]).float()
        dec.reset()
        le = dec.extend(ids[:T]).float()
        agree = float((lp - le).abs().max() / lp.abs().max())
        t = time_blocks({"prefill": (dec.reset, prefill, 1), "extend": (dec.reset, extend, 1)}, blocks=5)
        print(json.dumps({"kind": "ttft", "tokens": T, "prefill_ms": round(t["prefill"], 2), "extend_ms": round(t["extend"], 2),
                          "speedup": round(t["prefill"] / t["extend"], 2), "logits_rel_diff": agree}), flush=True)

    # (b) multi-turn: 64 tokens on a 4096-token history
    dec.reset()
    dec.extend(ids[:HISTORY])

    def back_to_history():
        dec.pos.fill_(HISTORY)
        dec._pos = [HISTORY]

    def append():
        dec.extend(ids[HISTORY:])

    def prefill_all():
        dec.prefill(ids)
    t = time_blocks({"extend": (back_to_history, append, 1), "prefill": (back_to_history, prefill_all, 1)}, blocks=5)
    print(json.dumps({"kind": "multi_turn", "history": HISTORY, "appended": TURN, "extend_ms": round(t["extend"], 2),
                      "prefill_all_ms": round(t["prefill"], 2), "speedup": round(t["prefill"] / t["extend"], 2)}), flush=True)

    # (c) one layer's attention
    kc, vc = dec.k_cache[0], dec.v_cache[0]
    kc.copy_(torch.randn(kc.shape, generator=g, device="cuda").half())
    vc.copy_(torch.randn(vc.shape, generator=g, device="cuda").half())
    for start, T in ((0, 2048), (HISTORY, TURN)):
        qkv = torch.randn(T, (nh + 2 * nkv) * d, generator=g, device="cuda").half()
        out = torch.empty(T, nh * d, dtype=torch.float16, device="cuda")
        qh = qkv[:, :nh * d].view(T, nh, d).transpose(0, 1)[None].contiguous()
        L = start + T
        mask = (torch.arange(L, device="cuda")[None, :] <= start + torch.arange(T, device="cuda")[:, None])[None, None]

        def kernel(start=start, qkv=qkv, out=out):
            quant_cuda.attn_extend(qkv, start, dec.rope_cos, dec.rope_sin, kc, vc, out, nh, nkv, dec.scale)

        def sdpa(qh=qh, L=L, mask=mask):
            F.scaled_dot_product_attention(qh, kc[None, :, :L], vc[None, :, :L], attn_mask=mask, scale=dec.scale, enable_gqa=nh != nkv)
        nothing = lambda: None  # noqa: E731
        n = 20 if T > 64 else 200
        t = time_blocks({"kernel": (nothing, kernel, n), "sdpa": (nothing, sdpa, n)})
        fl = causal_flops(nh, d, start, T)
        kv_bytes = 2 * nkv * L * d * 2
        row = {"kind": "attention", "start": start, "T": T, "splits": quant_cuda.attn_extend_splits(nh, nkv, T, start),
               "kernel_us": round(1e3 * t["kernel"], 2), "sdpa_us": round(1e3 * t["sdpa"], 2),
               "kernel_TFLOPs": round(fl / (t["kernel"] * 1e-3) / 1e12, 1), "sdpa_TFLOPs": round(fl / (t["sdpa"] * 1e-3) / 1e12, 1),
               "kernel_share_of_989": round(fl / (t["kernel"] * 1e-3) / PEAK, 3), "sdpa_share_of_989": round(fl / (t["sdpa"] * 1e-3) / PEAK, 3)}
        if T <= 64:
            row.update({"kernel_share_of_3.35TBps": round(kv_bytes / (t["kernel"] * 1e-3) / HBM, 3),
                        "sdpa_share_of_3.35TBps": round(kv_bytes / (t["sdpa"] * 1e-3) / HBM, 3)})
        print(json.dumps(row), flush=True)
    for s in dec.sequences:
        s.check()


if __name__ == "__main__":
    main()
