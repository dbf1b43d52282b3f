#!/usr/bin/env python3
"""What the sequence kernel's ops cost, on one GPU: a LLaMA-7B w4-s45 token's quantized part (32 decoder layers, gate/up and q/k/v
stacked: 128 items) with and without the ops between the matvecs.

Arms, on the same layers and inputs (fp16):
  seq_plain   the 128 matvecs as one DecodeSequence, each reading its predecessor's output directly (what bench.py's token does)
  seq_ops     the same 128 matvecs as one DecodeSequence with what a decoder layer puts between them, inside the launch:
              o = o_proj(a) + h, gu = gate_up(rmsnorm(o)), d = down(silu(g) u) + o, qkv = qkv(rmsnorm(d)); the next layer's a is
              qkv's v slice (attention is not part of this measurement), its h is d
  graph_ops   the same computation as QuantLinearLUT forwards with the RMSNorms, SiLU gating and residual adds as torch ops, all
              captured in one CUDA graph

Each arm is timed with CUDA events over a block of calls; the arms alternate block by block and the median of 7 blocks is kept.  The
last output of seq_ops and graph_ops is compared in the max norm (reported; the torch RMSNorm rounds x r to fp16 before multiplying by
the weight, the kernel does not).  The first line names the card, its power limit and max SM clock (nvidia-smi, read-only query).

    python tests/perf/sequence_ops_timing.py [--quick]
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sequence_bf16_timing import synth_module, timed  # noqa: E402
from squeezellm_b200.runtime import DecodeSequence, GraphedDecodeStep  # noqa: E402

H, I = 4096, 11008
LAYER = [("o", H, H), ("gate_up", H, 2 * I), ("down", I, H), ("qkv", H, 3 * H)]
EPS = 1e-5


def rmsnorm(x, w):
    xf = x.float()
    return w * (xf * torch.rsqrt(xf.pow(2).mean() + EPS)).to(x.dtype)


def build(mods, norms, ops):
    seq = DecodeSequence(H, "cuda", lut_mode="exact")
    hv, h_t = seq.new_input(H)
    a, h = seq.input, hv
    for layer in range(len(mods) // 4):
        mo, mgu, md, mq = mods[4 * layer:4 * layer + 4]
        w1, w2 = norms[layer]
        if ops:
            o = seq.matvec(mo, a, residual=h)
            gu = seq.matvec(mgu, o, norm=(w2, EPS))
            d = seq.matvec(md, gu[0:I], up=gu[I:2 * I], residual=o)
            q = seq.matvec(mq, d, norm=(w1, EPS))
        else:
            o = seq.matvec(mo, a)
            gu = seq.matvec(mgu, o)
            d = seq.matvec(md, gu[0:I])
            q = seq.matvec(mq, d)
        a, h = q[2 * H:3 * H], d
    seq.compile(outputs=[q])
    return seq, h_t


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    nlayers = 2 if quick else 32
    mods = [synth_module(4, K, N, seed=2000 + 4 * layer + j) for layer in range(nlayers) for j, (_, K, N) in enumerate(LAYER)]
    g = torch.Generator(device="cuda").manual_seed(3)
    norms = [tuple((1 + 0.1 * torch.randn(H, device="cuda", generator=g)).half() for _ in range(2)) for _ in range(nlayers)]
    x = torch.randn(H, device="cuda", generator=g).half()
    h0 = torch.randn(H, device="cuda", generator=g).half()

    plain, _ = build(mods, norms, False)
    withops, h_t = build(mods, norms, True)
    plain.x.copy_(x)
    withops.x.copy_(x)
    h_t.copy_(h0)

    def step(a):
        h = h0
        for layer in range(nlayers):
            mo, mgu, md, mq = mods[4 * layer:4 * layer + 4]
            w1, w2 = norms[layer]
            o = mo(a) + h
            gu = mgu(rmsnorm(o, w2))
            d = md(torch.nn.functional.silu(gu[:I]) * gu[I:]) + o
            qkv = mq(rmsnorm(d, w1))
            a, h = qkv[2 * H:3 * H], d
        return qkv

    graph = GraphedDecodeStep(step, x, warmup=2)
    graph.x_dev.copy_(x)
    ys = withops.replay()[0].clone()
    yg = graph.replay().clone()
    torch.cuda.synchronize()
    assert not withops.error() and torch.isfinite(ys).all()
    rel = float((ys.double() - yg.double()).abs().max() / yg.double().abs().max())
    n = 5 if quick else 20
    t = timed({"seq_plain": plain.replay, "seq_ops": withops.replay, "graph_ops": graph.replay}, n, 5 if quick else 7)
    assert not plain.error() and not withops.error()
    print(json.dumps(dict(kind="7B-token-quantized-part", layers=nlayers, items=len(mods), **{k + "_ms": v for k, v in t.items()},
                          ops_vs_plain=round(t["seq_ops"] / t["seq_plain"], 4), seq_ops_speedup_vs_graph_ops=round(t["graph_ops"] / t["seq_ops"], 3),
                          last_output_max_norm_seq_ops_vs_graph_ops=float(f"{rel:.3e}"))), flush=True)


if __name__ == "__main__":
    main()
