#!/usr/bin/env python3
"""Token sampling on the GPU: quant_cuda.sample against torch.argmax and against HF's warpers followed by softmax and
torch.multinomial, and its cost inside the decoders' generate loop.

(a) kernel  R rows in {1, 8, 32, 79} x V in {32000, 128256, 151936} of fp16 logits (normal, scale 3) x {greedy, temperature 0.7,
            top-k 50, top-p 0.9, top-k 50 + top-p 0.9}: us per call of quant_cuda.sample; of torch.argmax (greedy); and of the torch
            composite HF's generate runs (TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper, softmax, multinomial; argmax for
            greedy).  Every arm is CALLS calls captured in one CUDA graph, so launch overhead is the graph's for all three; the arms
            alternate block by block and the median of 7 blocks is kept.
(b) decode  tokens/s of the decode loop of SequenceDecoder and BatchDecoder (B = 8) generate on the synthetic 7B w4-s45 of
            decoder_timing.make_model (32 layers, fp16, vocab 32000) at 128 tokens of context: the step graph alone (greedy) against
            the step graph followed by the sample launch (temperature 0.7, top-p 0.9), alternated block by block.
The first line names the card, its power limit and max SM clock (nvidia-smi, read-only query).

    python tests/perf/sample_timing.py [--quick]
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from decoder_timing import make_model, time_blocks  # noqa: E402

ROWS = (1, 8, 32, 79)
VOCABS = (32000, 128256, 151936)
MODES = {"greedy": (0.0, 0, 1.0), "temp0.7": (0.7, 0, 1.0), "topk50": (0.7, 50, 1.0), "topp0.9": (0.7, 0, 0.9),
         "topk50+topp0.9": (0.7, 50, 0.9)}
CALLS = 20
CTX = 128
BLOCK = 16


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(CALLS):
            fn()
    torch.cuda.synchronize()
    return g


def kernel_sweep(quick):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

    from squeezellm_b200.quant import quant_cuda
    for V in VOCABS[:1] if quick else VOCABS:
        for R in ROWS[:2] if quick else ROWS:
            x = (torch.randn(R, V, device="cuda") * 3).half()
            out = torch.zeros(R, dtype=torch.int64, device="cuda")
            ids = torch.zeros(R, 1, dtype=torch.int64, device="cuda")
            for mode, (t, k, p) in MODES.items():
                par = [torch.zeros(R, dtype=torch.int32, device="cuda"), torch.full((R,), t, device="cuda"),
                       torch.full((R,), k, dtype=torch.int32, device="cuda"), torch.full((R,), p, device="cuda"),
                       torch.arange(R, dtype=torch.int64, device="cuda")]

                def ours():
                    quant_cuda.sample(x, par[0], par[1], par[2], par[3], par[4], out)

                def composite():
                    if t == 0:
                        out.copy_(x.argmax(dim=-1))
                        return
                    s = TemperatureLogitsWarper(t)(ids, x.float())
                    if k:
                        s = TopKLogitsWarper(k)(ids, s)
                    if p < 1:
                        s = TopPLogitsWarper(p)(ids, s)
                    out.copy_(torch.multinomial(torch.softmax(s, dim=-1), 1).view(-1))

                arms = {"sample": graphed(ours), "torch": graphed(composite)}
                if t == 0:
                    arms["argmax"] = graphed(lambda: out.copy_(x.argmax(dim=-1)))
                ms = time_blocks({a: (lambda: None, g.replay, 3) for a, g in arms.items()})
                print(json.dumps({"kind": "kernel", "V": V, "R": R, "mode": mode,
                                  **{f"{a}_us": round(v * 1e3 / CALLS, 2) for a, v in ms.items()}}), flush=True)


def decode_loop(quick):
    from squeezellm_b200.runtime import BatchDecoder, SequenceDecoder
    model = make_model(2 if quick else 32)
    for B in (1, 8):
        dec = SequenceDecoder(model, CTX + 4 * BLOCK) if B == 1 else BatchDecoder(model, CTX + 4 * BLOCK, B)
        dec.temperature.fill_(0.7)
        dec.top_p.fill_(0.9)
        dec.seed.copy_(torch.arange(B))
        logits = dec.logits.view(B, -1)

        def reset():
            dec.pos.fill_(CTX)

        def greedy():
            dec.graph.replay()

        def sampled():
            dec.graph.replay()
            dec._sample(logits)

        ms = time_blocks({"greedy": (reset, greedy, BLOCK), "sampled": (reset, sampled, BLOCK)})
        print(json.dumps({"kind": "decode", "decoder": type(dec).__name__, "B": B, "ctx": CTX,
                          **{f"{a}_ms_per_step": round(v, 4) for a, v in ms.items()},
                          **{f"{a}_tokens_per_s": round(B * 1e3 / v, 1) for a, v in ms.items()},
                          "sample_share": round(ms["sampled"] / ms["greedy"] - 1, 4)}), flush=True)
        del dec
        torch.cuda.empty_cache()


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    with torch.no_grad():
        kernel_sweep(quick)
        decode_loop(quick)


if __name__ == "__main__":
    main()
