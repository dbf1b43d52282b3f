#!/usr/bin/env python3
"""Fisher information timing on one GPU.

Per layer: quant_cuda.fisher_accumulate on the LLaMA-7B shapes [out, in] = 4096x4096, 11008x4096 and 4096x11008, and on a whole
decoder layer (q, k, v, o: 4096x4096; gate, up: 11008x4096; down: 4096x11008: seven calls), 8192 rows per call split into
(samples S, seq_len T) = (64, 128), (16, 512), (4, 2048), in fp16 and bf16.  Arms, alternated:
  kernel   quant_cuda.fisher_accumulate: one launch per layer, F read and written once
  cublas   per sample g = torch.mm(dy_s^T, x_s, out_dtype=torch.float32) (cuBLAS, fp32 output from 16-bit operands), then
           F.addcmul_(g, g): about 16 bytes per weight per sample on top of the GEMM
  fp32mm   per sample g = dy_s^T.float() @ x_s.float() with TF32 off, then F.addcmul_(g, g)
CUDA events around several calls, median of 5 alternating repetitions.  Per line: ms of each arm, the kernel's TFLOP/s from
2 rows N K per layer, that rate over the 989 TFLOP/s H100 SXM data-sheet dense fp16/bf16 figure (a data-sheet figure, not a
reached one), and the largest relative difference between the kernel's and the cublas arm's F (1 % floor).

End to end: a randomly initialised LLaMA-7B-shaped LlamaForCausalLM with 4 decoder layers in fp16 (no download).  Tokens/s of
quantize.fisher_information against per-sequence autograd (one backward per sequence with the linear weights requiring grad,
each fp16 weight.grad squared into fp32 sums), and the largest relative difference of the two results (1 % floor).

The first line names the card, its power limit and its maximum SM clock (nvidia-smi, read-only query).

    python tests/perf/fisher_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402
from squeezellm_b200 import quantize as qz  # noqa: E402
from squeezellm_b200.checkpoint import find_linear_layers  # noqa: E402

PEAK = 989e12
SHAPES = {"7B-4096x4096": [(4096, 4096)], "7B-11008x4096": [(11008, 4096)], "7B-4096x11008": [(4096, 11008)],
          "7B-decoder-layer": [(4096, 4096)] * 4 + [(11008, 4096)] * 2 + [(4096, 11008)]}
SPLITS = [(64, 128), (16, 512), (4, 2048)]
ROWS = 8192


def time_ms(fn, n):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n


def rel(a, b):
    a, b = a.double(), b.double()
    den = torch.maximum(b.abs(), 1e-2 * b.abs().max())
    return float(((a - b).abs() / den).max())


def cublas_arm(x, dy, f, T):
    for s in range(x.shape[0] // T):
        g = torch.mm(dy[s * T:(s + 1) * T].t(), x[s * T:(s + 1) * T], out_dtype=torch.float32)
        f.addcmul_(g, g)


def fp32_arm(x, dy, f, T):
    for s in range(x.shape[0] // T):
        g = dy[s * T:(s + 1) * T].t().float() @ x[s * T:(s + 1) * T].float()
        f.addcmul_(g, g)


def per_layer(quick):
    reps, n = (2, 1) if quick else (5, 2)
    torch.backends.cuda.matmul.allow_tf32 = False
    gen = torch.Generator(device="cuda").manual_seed(0)
    for dtype in (torch.float16, torch.bfloat16):
        data = {}
        for (N, K) in set(s for v in SHAPES.values() for s in v):
            data[(N, K)] = (torch.randn(ROWS, K, device="cuda", generator=gen).to(dtype),
                            torch.randn(ROWS, N, device="cuda", generator=gen).to(dtype))
        for name, layers in SHAPES.items():
            fs = [torch.zeros(N, K, device="cuda") for (N, K) in layers]
            for S, T in SPLITS[:1] if quick else SPLITS:
                def arm(fn):
                    return lambda: [fn(*data[s], f, T) for s, f in zip(layers, fs)]
                arms = {"kernel": arm(qc.fisher_accumulate), "cublas": arm(cublas_arm), "fp32mm": arm(fp32_arm)}
                a, b = torch.zeros_like(fs[-1]), torch.zeros_like(fs[-1])
                qc.fisher_accumulate(*data[layers[-1]], a, T)
                cublas_arm(*data[layers[-1]], b, T)
                diff = rel(a, b)
                del a, b
                ms = {k: [] for k in arms}
                for _ in range(reps):
                    for k, fn in arms.items():
                        time_ms(fn, 1)  # warm-up of this arm
                        ms[k].append(time_ms(fn, n))
                med = {k: statistics.median(v) for k, v in ms.items()}
                flop = sum(2.0 * ROWS * N * K for (N, K) in layers)
                tf = flop / (med["kernel"] * 1e-3)
                print(json.dumps({"shape": name, "dtype": str(dtype).replace("torch.", ""), "samples": S, "seq_len": T, "rows": ROWS,
                                  "kernel_ms": round(med["kernel"], 3), "cublas_ms": round(med["cublas"], 3),
                                  "fp32mm_ms": round(med["fp32mm"], 3), "kernel_TFLOPs": round(tf / 1e12, 1),
                                  "frac_of_989": round(tf / PEAK, 3), "speedup_vs_cublas": round(med["cublas"] / med["kernel"], 2),
                                  "speedup_vs_fp32mm": round(med["fp32mm"] / med["kernel"], 2),
                                  "max_rel_diff_vs_cublas": diff}), flush=True)
            del fs
        del data
        torch.cuda.empty_cache()


def autograd_fisher(model, batches, names):
    """Per-sequence autograd: one backward per sequence, each fp16 weight.grad squared into fp32 sums."""
    lin = find_linear_layers(model)
    for p in model.parameters():
        p.requires_grad_(False)
    for n in names:
        lin[n].weight.requires_grad_(True)
    F = {n: torch.zeros(lin[n].weight.shape, device="cuda") for n in names}
    for ids in batches:
        for b in range(ids.shape[0]):
            logits = model(ids[b:b + 1]).logits[0, :-1].float()
            torch.nn.functional.cross_entropy(logits, ids[b, 1:], reduction="sum").backward()
            for n in names:
                g = lin[n].weight.grad
                F[n].addcmul_(g.float(), g.float())
                lin[n].weight.grad = None
    for n in names:
        lin[n].weight.requires_grad_(False)
    return {f"{n}.weight": f for n, f in F.items()}


def end_to_end(quick):
    import transformers
    cfg = transformers.LlamaConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1 if quick else 4,
                                   num_attention_heads=32, num_key_value_heads=32, vocab_size=32000, max_position_embeddings=2048)
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = transformers.LlamaForCausalLM(cfg).half().eval()
    names = [n for n in find_linear_layers(model) if n != "lm_head"]
    gen = torch.Generator(device="cuda").manual_seed(1)
    for B, T, nb in ([(2, 128, 1)] if quick else [(8, 512, 2), (2, 2048, 2)]):
        batches = [torch.randint(0, 32000, (B, T), device="cuda", generator=gen) for _ in range(nb)]
        out = {}
        for arm, fn in (("fisher_information", lambda: qz.fisher_information(model, batches)),
                        ("per_sequence_autograd", lambda: autograd_fisher(model, batches, names))):
            fn()  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out[arm] = fn()
            torch.cuda.synchronize()
            out[arm + "_s"] = time.perf_counter() - t0
        a, b = out["fisher_information"], out["per_sequence_autograd"]
        diff = max(rel(a[k], b[k]) for k in a)
        tokens = B * T * nb
        print(json.dumps({"kind": "end_to_end", "layers": cfg.num_hidden_layers, "batch": B, "seq_len": T, "batches": nb,
                          "fisher_information_tokens_per_s": round(tokens / out["fisher_information_s"], 1),
                          "per_sequence_autograd_tokens_per_s": round(tokens / out["per_sequence_autograd_s"], 1),
                          "speedup": round(out["per_sequence_autograd_s"] / out["fisher_information_s"], 2),
                          "max_rel_diff": diff,
                          "nonfinite_autograd": sum(int(not torch.isfinite(v).all()) for v in b.values())}), flush=True)
        del out, a, b


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    per_layer(quick)
    end_to_end(quick)


if __name__ == "__main__":
    main()
