#!/usr/bin/env python3
"""Whole-model greedy decode on one GPU: runtime.SequenceDecoder on a synthetic LLaMA-7B w4-s45 (32 layers, fp16, random
QuantLinearLUT projections as sequence_bf16_timing.synth_module makes them, dense fp16 lm_head), with the KV cache holding random
values at contexts 128, 1024 and 4096.

Arms, at each context:
  (a) decoder    SequenceDecoder's graph: ms per token and tokens/s
  (b) sdpa_graph the same token graph with torch's RoPE, cache writes (index_copy_) and scaled_dot_product_attention over the
                 cache up to the block's last position (masked past pos) in place of the attention kernel
  (c) hf         HF's per-token forward of the same (sibling-stacked) quantized model with a DynamicCache: what a user runs today
  (d) kernel / sdpa  one layer's attention alone: quant_cuda.attn_decode against scaled_dot_product_attention on K, V [0..ctx],
                 with the K / V bytes read per call over the kernel time, as a share of the data sheet's 3.35 TB/s
Every arm runs blocks of tokens (calls) timed with CUDA events; the arms alternate block by block, the position is set back to the
context before each block, and the median of 7 blocks is kept.  The first line names the card, its power limit and max SM clock
(nvidia-smi, read-only query).

    python tests/perf/decoder_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sequence_bf16_timing import synth_module  # noqa: E402

HBM = 3.35e12
CONTEXTS = (128, 1024, 4096)
BLOCK = 16  # tokens per timed block of the graph arms


def make_model(n_layers):
    import transformers
    from squeezellm_b200.quant import QuantLinearLUT  # noqa: F401
    cfg = transformers.LlamaConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=n_layers, num_attention_heads=32,
                                   num_key_value_heads=32, vocab_size=32000, max_position_embeddings=8192, attn_implementation="sdpa")
    torch.set_default_dtype(torch.float16)
    try:
        with torch.device("cuda"):
            model = transformers.LlamaForCausalLM(cfg).eval()
    finally:
        torch.set_default_dtype(torch.float32)
    seed = 2000
    for layer in model.model.layers:
        for block, names in (("self_attn", ("q_proj", "k_proj", "v_proj", "o_proj")), ("mlp", ("gate_proj", "up_proj", "down_proj"))):
            mod = getattr(layer, block)
            for n in names:
                lin = getattr(mod, n)
                setattr(mod, n, synth_module(4, lin.in_features, lin.out_features, seed))
                seed += 1
    torch.cuda.empty_cache()
    return model


class TorchAttention:
    """quant_cuda with attn_decode replaced by torch ops over the cache's first `length` positions (positions past pos masked)."""

    def __init__(self, qc, length):
        self.qc, self.length = qc, length

    def attn_decode(self, qkv, pos, cos, sin, kc, vc, out, nh, nkv, scale):
        d = kc.shape[-1]
        p = pos.long()
        c, s = cos.index_select(0, p), sin.index_select(0, p)  # [1, d/2]

        def rope(x):
            a, b = x[..., :d // 2].float(), x[..., d // 2:].float()
            return torch.cat([a * c - b * s, b * c + a * s], dim=-1).to(x.dtype)
        q = rope(qkv[:nh * d].view(nh, d))
        k = rope(qkv[nh * d:(nh + nkv) * d].view(nkv, d))
        v = qkv[(nh + nkv) * d:].view(nkv, d)
        kc.index_copy_(1, p, k.view(nkv, 1, d))
        vc.index_copy_(1, p, v.view(nkv, 1, d))
        mask = torch.arange(self.length, device=qkv.device) <= p
        o = F.scaled_dot_product_attention(q.view(1, nh, 1, d), kc[None, :, :self.length], vc[None, :, :self.length],
                                           attn_mask=mask.view(1, 1, 1, -1), scale=scale, enable_gqa=nh != nkv)
        out.copy_(o.view(-1))


def capture(dec, qc):
    real = dec._qc
    dec._qc = qc
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.no_grad():
            with torch.cuda.stream(side):
                dec._step()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                logits = dec._step()
        torch.cuda.synchronize()
    finally:
        dec._qc = real
    return g, logits


def time_blocks(arms, blocks=7):
    """arms: {name: (reset, step, n)}: reset() outside the timed window, then n step() calls between two events; the arms alternate
    block by block.  -> median ms per step."""
    ms = {a: [] for a in arms}
    for a, (reset, step, n) in arms.items():  # warm-up
        reset()
        step()
    torch.cuda.synchronize()
    for _ in range(blocks):
        for a, (reset, step, n) in arms.items():
            reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                step()
            e1.record()
            e1.synchronize()
            ms[a].append(e0.elapsed_time(e1) / n)
    return {a: statistics.median(v) for a, v in ms.items()}


def main():
    quick = "--quick" in sys.argv
    from transformers import DynamicCache

    from squeezellm_b200.quant import quant_cuda
    from squeezellm_b200.runtime import SequenceDecoder
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    n_layers = 2 if quick else 32
    contexts = (128, 1024) if quick else CONTEXTS
    model = make_model(n_layers)
    max_len = max(contexts) + 2 * BLOCK
    dec = SequenceDecoder(model, max_len)
    nh, nkv, d = dec.n_heads, dec.n_kv, dec.head_dim
    g = torch.Generator(device="cuda").manual_seed(5)
    dec.k_cache.copy_(torch.randn(dec.k_cache.shape, generator=g, device="cuda").half())
    dec.v_cache.copy_(torch.randn(dec.v_cache.shape, generator=g, device="cuda").half())
    print(json.dumps({"kind": "setup", "layers": n_layers, "max_len": max_len, "splits": quant_cuda.attn_decode_splits(nh, nkv),
                      "sm": quant_cuda.sm_count()}), flush=True)
    for ctx in contexts:
        def set_pos(ctx=ctx):
            dec.pos.fill_(ctx)
            dec._pos = [ctx]
            dec.tok.fill_(1)
        g_sdpa, logits_sdpa = capture(dec, TorchAttention(quant_cuda, ctx + BLOCK + 1))
        # one token of each graph from the same state: the logits agree to the attention's rounding
        set_pos()
        dec.graph.replay()
        la = dec.logits.float().clone()
        set_pos()
        g_sdpa.replay()
        lb = logits_sdpa.float().clone()
        agree = float((la - lb).abs().max() / lb.abs().max())

        cache = DynamicCache()
        for i in range(n_layers):
            cache.update(dec.k_cache[i, :, :ctx][None].clone(), dec.v_cache[i, :, :ctx][None].clone(), i)
        hf_tok = torch.ones(1, 1, dtype=torch.long, device="cuda")

        def hf_reset():
            cache.crop(ctx)

        def hf_step():
            with torch.no_grad():
                model(input_ids=hf_tok, past_key_values=cache, use_cache=True)

        # (d): one layer's attention alone, at position ctx
        qkv = torch.randn((nh + 2 * nkv) * d, generator=g, device="cuda").half()
        out = torch.empty(nh * d, dtype=torch.float16, device="cuda")
        pos1 = torch.tensor([ctx], dtype=torch.int32, device="cuda")
        kc, vc = dec.k_cache[0], dec.v_cache[0]
        qh = qkv[:nh * d].view(1, nh, 1, d)

        def kernel():
            quant_cuda.attn_decode(qkv, pos1, dec.rope_cos, dec.rope_sin, kc, vc, out, nh, nkv, dec.scale)

        def sdpa():
            F.scaled_dot_product_attention(qh, kc[None, :, :ctx + 1], vc[None, :, :ctx + 1], scale=dec.scale)

        nothing = lambda: None  # noqa: E731
        t = time_blocks({"decoder": (set_pos, dec.graph.replay, BLOCK), "sdpa_graph": (set_pos, g_sdpa.replay, BLOCK),
                         "hf": (hf_reset, hf_step, 4), "kernel": (nothing, kernel, 200), "sdpa": (nothing, sdpa, 200)})
        kv_bytes = 2 * nkv * (ctx + 1) * d * 2
        print(json.dumps({
            "kind": "context", "ctx": ctx,
            "decoder_ms_per_token": round(t["decoder"], 3), "decoder_tokens_per_s": round(1e3 / t["decoder"], 1),
            "sdpa_graph_ms_per_token": round(t["sdpa_graph"], 3), "hf_ms_per_token": round(t["hf"], 3),
            "kernel_us": round(1e3 * t["kernel"], 2), "sdpa_us": round(1e3 * t["sdpa"], 2),
            "kernel_kv_TBps": round(kv_bytes / (t["kernel"] * 1e-3) / 1e12, 3), "sdpa_kv_TBps": round(kv_bytes / (t["sdpa"] * 1e-3) / 1e12, 3),
            "kernel_share_of_3.35TBps": round(kv_bytes / (t["kernel"] * 1e-3) / HBM, 3),
            "sdpa_share_of_3.35TBps": round(kv_bytes / (t["sdpa"] * 1e-3) / HBM, 3),
            "logits_rel_diff_decoder_vs_sdpa_graph": agree}), flush=True)
        del g_sdpa, logits_sdpa, cache
        torch.cuda.empty_cache()
    for s in dec.sequences:
        s.check()


if __name__ == "__main__":
    main()
