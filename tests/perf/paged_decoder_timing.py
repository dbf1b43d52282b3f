#!/usr/bin/env python3
"""The paged KV cache against the contiguous one, on the synthetic LLaMA-7B w4-s45 of decoder_timing.make_model (32 heads of 128,
fp16).  The first line names the card, its power limit and max SM clock (nvidia-smi, read-only query).  Every arm runs blocks of
calls (steps) timed with CUDA events; the arms of one configuration alternate block by block and the median of 7 blocks is kept.

  (a) attention  one layer: quant_cuda.attn_decode_paged on randomly permuted pages against attn_decode_batch, at B in {8, 16, 32} and
                 context in {1024, 4096}, with the K / V bytes over the time as a share of the data sheet's 3.35 TB/s; and
                 attn_extend_paged against attn_extend at (start, T) = (0, 2048) and (4096, 64)
  (b) step       BatchDecoder(pages=P) against BatchDecoder at B in {8, 16} and context in {128, 1024, 4096}; at B = 16 and 4096
                 the two decoders' caches (2 x 34 GB) do not fit on an 80 GB card together, so there the arms run one after the
                 other, each alone on the card, instead of alternating
  (c) mixed      B = 32 with 16 rows at 4096 tokens of context and 16 at 256: only the paged decoder (the contiguous caches would need
                 32 x 4096 positions); its step time and aggregate tokens/s

    python tests/perf/paged_decoder_timing.py [--quick]
"""
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import HBM, make_model, time_blocks  # noqa: E402

PAGE = 64
BLOCK = 16
NH = NKV = 32
D = 128


def emit(**row):
    print(json.dumps(row), flush=True)


def rand(shape, g):
    return torch.randn(shape, generator=g, device="cuda").half()


def paged_layer(B, ctx, g):
    """One layer's pools for B rows at position ctx on randomly permuted pages, and the same content contiguous."""
    width = -(-(ctx + 1) // PAGE)
    n = B * width
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(B * ctx)).to(torch.int32)
    table = perm.view(B, width).cuda()
    kp, vp = rand((n, NKV, PAGE, D), g), rand((n, NKV, PAGE, D), g)
    kc = kp[table.long()].permute(0, 2, 1, 3, 4).reshape(B, NKV, width * PAGE, D).contiguous()
    vc = vp[table.long()].permute(0, 2, 1, 3, 4).reshape(B, NKV, width * PAGE, D).contiguous()
    return kp, vp, table, kc, vc, width * PAGE


def attention(qc, quick):
    from test_attn_decode_gpu import rope_tables
    g = torch.Generator(device="cuda").manual_seed(1)
    scale = D ** -0.5
    for B in ((8,) if quick else (8, 16, 32)):
        for ctx in ((1024,) if quick else (1024, 4096)):
            kp, vp, table, kc, vc, cap = paged_layer(B, ctx, g)
            cos, sin = rope_tables(cap, D)
            qkv = rand((B, (NH + 2 * NKV) * D), g)
            out = torch.empty(B, NH * D, dtype=torch.float16, device="cuda")
            pos = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
            t = time_blocks({
                "paged": (lambda: None, lambda: qc.attn_decode_paged(qkv, pos, cos, sin, kp, vp, table, out, NH, NKV, scale), 50),
                "contiguous": (lambda: None, lambda: qc.attn_decode_batch(qkv, pos, cos, sin, kc, vc, out, NH, NKV, scale), 50)})
            kv = B * 2 * NKV * (ctx + 1) * D * 2
            emit(kind="attn_decode", B=B, ctx=ctx, **{f"us_{a}": round(ms * 1e3, 1) for a, ms in t.items()},
                 **{f"hbm_share_{a}": round(kv / (ms * 1e-3) / HBM, 3) for a, ms in t.items()}, paged_over_contiguous=round(t["paged"] / t["contiguous"], 3))
            del kp, vp, kc, vc
    for start, T in ((0, 2048), (4096, 64)):
        kp, vp, table, kc, vc, cap = paged_layer(1, start + T - 1, g)
        cos, sin = rope_tables(cap, D)
        qkv = rand((T, (NH + 2 * NKV) * D), g)
        out = torch.empty(T, NH * D, dtype=torch.float16, device="cuda")
        t = time_blocks({
            "paged": (lambda: None, lambda: qc.attn_extend_paged(qkv, start, cos, sin, kp, vp, table[0], out, NH, NKV, scale), 20),
            "contiguous": (lambda: None, lambda: qc.attn_extend(qkv, start, cos, sin, kc[0], vc[0], out, NH, NKV, scale), 20)})
        emit(kind="attn_extend", start=start, T=T, **{f"us_{a}": round(ms * 1e3, 1) for a, ms in t.items()},
             paged_over_contiguous=round(t["paged"] / t["contiguous"], 3))


def fill_random(t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for i in range(t.shape[0]):
        t[i].copy_(torch.randn(t[i].shape, generator=g, device="cuda").half())


def place(dec, ctxs):
    """Every row b at position ctxs[b] (pages assigned up to ctxs[b] + BLOCK on a paged decoder), token 1."""
    if dec._pages is not None and not any(dec._pages.held(b) for b in range(dec.batch)):
        dec._reserve({b: (c + BLOCK + 1, False) for b, c in enumerate(ctxs)})
    dec.pos.copy_(torch.tensor(ctxs, dtype=torch.int32))
    dec._pos = list(ctxs)
    dec.tok.fill_(1)


def steps(model, quick):
    from squeezellm_b200.runtime import BatchDecoder
    for B in ((8,) if quick else (8, 16)):
        for ctx in ((128, 1024) if quick else (128, 1024, 4096)):
            max_len = ctx + 2 * BLOCK
            pages = B * -(-(ctx + BLOCK + 1) // PAGE)
            make = {"paged": lambda: BatchDecoder(model, max_len, B, pages=pages), "contiguous": lambda: BatchDecoder(model, max_len, B)}
            together = B * ctx <= 8 * 4096
            groups = [list(make)] if together else [[a] for a in make]
            t = {}
            for group in groups:
                decs = {a: make[a]() for a in group}
                for i, d in enumerate(decs.values()):
                    fill_random(d.k_cache, 5 + i)
                    fill_random(d.v_cache, 7 + i)
                t.update(time_blocks({a: (lambda d=d: place(d, [ctx] * B), d.graph.replay, BLOCK) for a, d in decs.items()}))
                del decs, d
                gc.collect()   # the decoders' graphs hold their memory until collected
                torch.cuda.empty_cache()
            emit(kind="step", B=B, ctx=ctx, **{f"ms_{a}": round(ms, 3) for a, ms in t.items()},
                 paged_over_contiguous=round(t["paged"] / t["contiguous"], 4), alternated=together)


def mixed(model, n_layers):
    from squeezellm_b200.runtime import BatchDecoder
    B, long_ctx, short_ctx = 32, 4096, 256
    max_len = long_ctx + 2 * BLOCK
    ctxs = [long_ctx] * 16 + [short_ctx] * 16
    pages = sum(-(-(c + BLOCK + 1) // PAGE) for c in ctxs)
    dec = BatchDecoder(model, max_len, B, pages=pages)
    fill_random(dec.k_cache, 5)
    fill_random(dec.v_cache, 6)
    t = time_blocks({"paged": (lambda: place(dec, ctxs), dec.graph.replay, BLOCK)})["paged"]
    per_page = 2 * n_layers * NKV * PAGE * D * 2
    emit(kind="mixed", B=B, contexts="16 x 4096 + 16 x 256", pages=pages, pool_GB=round(pages * per_page / 1e9, 1),
         contiguous_GB=round(2 * n_layers * B * NKV * max_len * D * 2 / 1e9, 1), ms_per_step=round(t, 3),
         tokens_per_s=round(B * 1e3 / t, 1))


def main():
    quick = "--quick" in sys.argv
    from squeezellm_b200.quant import quant_cuda as qc
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    emit(kind="card", nvidia_smi=q.stdout.strip().splitlines()[:1])
    attention(qc, quick)
    gc.collect()
    torch.cuda.empty_cache()
    n_layers = 2 if quick else 32
    model = make_model(n_layers)
    steps(model, quick)
    mixed(model, n_layers)


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    main()
