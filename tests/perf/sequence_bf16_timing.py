#!/usr/bin/env python3
"""bf16 in the sequence kernel and the exchange, on one GPU.

Arms, on the same layers and inputs:
  seq_fp16      a LLaMA-7B w4-s45 token (32 decoder layers, q/k/v and gate/up stacked: 128 items) as one fp16 DecodeSequence
  seq_bf16      the same token as one bf16 DecodeSequence (runtime.DecodeSequence(dtype=torch.bfloat16))
  graph_bf16    the same 128 matvecs as bf16 one-GEMV launches (QuantLinearLUT on one bf16 row) captured in one CUDA graph: the
                one-GPU bf16 route without the sequence kernel
  xchg_fp16 / xchg_bf16   the world-1 exchange (quant_cuda.lutgemv_fused_exchange / _bf16) per launch on the four 7B shapes

Each arm is timed with CUDA events over a block of calls; the arms alternate block by block and the median of 7 blocks is kept.
Outputs are checked against each other: every item of each sequence against a one-GEMV launch of its dtype on the input that item
consumed (at most one rounding step of the dtype apart, see steps_apart), and the bf16 graph's last output against the bf16
sequence's, in the max norm (reported).  Weights are generated on the device from a seed;
the codebook is scaled to N(0, 1/K) so the chain stays O(1).  The first line names the card and its power limit (nvidia-smi,
read-only query).

    python tests/perf/sequence_bf16_timing.py [--quick]
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from squeezellm_b200.quant import QuantLinearLUT  # noqa: E402
from squeezellm_b200.quant import quant_cuda as qc  # noqa: E402
from squeezellm_b200.runtime import DecodeSequence, GraphedDecodeStep  # noqa: E402

H, I = 4096, 11008
LAYER = [("qkv", H, 3 * H, 0), ("o", H, H, 2 * H), ("gate_up", H, 2 * I, 0), ("down", I, H, 0)]  # (name, K, N, x offset in the previous output)
SP, TOPX = 0.0045, 10


def synth_module(bits, K, N, seed):
    """A QuantLinearLUT with random packed indices, a sorted N(0, 1/K) codebook, 0.45 % CSR outliers and 10 dense rows, made on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = QuantLinearLUT(bits, K, N, False, include_sparse=True, numvals=0, topX=TOPX)
    qw = torch.randint(-2**31, 2**31 - 1, (K // 32 * bits, N), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    lut = torch.sort(torch.randn((N, 2**bits), device="cuda", generator=g) / K ** 0.5, dim=1).values.contiguous()
    nnz = int(round(SP * K * N))
    key = torch.unique(torch.randint(0, N, (nnz,), device="cuda", generator=g).to(torch.int64) * K
                       + torch.randint(0, K, (nnz,), device="cuda", generator=g))
    r, c = key // K, key % K
    rows = torch.zeros(N + 1, dtype=torch.int32, device="cuda")
    rows[1:] = torch.cumsum(torch.bincount(r, minlength=N), 0).to(torch.int32)
    m.qweight, m.lookup_table = qw, lut
    m.register_buffer("rows", rows)
    m.register_buffer("cols", c.to(torch.int32).contiguous())
    m.register_buffer("vals", torch.randn(key.numel(), device="cuda", generator=g) * 0.1 / K ** 0.5)
    m.register_buffer("full_rows", torch.randn((K, TOPX), device="cuda", generator=g) * 0.05 / K ** 0.5)
    m.register_buffer("full_row_indices", torch.randperm(N, device="cuda", generator=g)[:TOPX].to(torch.int32))
    m.numvals = key.numel()
    return m


def time_block(fn, n):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n


def timed(arms, n, blocks):
    for fn in arms.values():  # warm-up
        fn()
    torch.cuda.synchronize()
    t = {a: [] for a in arms}
    for _ in range(blocks):
        for a, fn in arms.items():
            t[a].append(time_block(fn, n))
    return {a: round(statistics.median(v), 4) for a, v in t.items()}


def steps_apart(a, b, step):
    """max over elements of |a - b| in rounding steps of the output dtype (step = 2^-7 bf16, 2^-10 fp16) of the larger value, with a
    floor of 1e-4 of the vector's largest output: an output that cancels to near zero differs by the fp32 summation order, not by
    its rounding."""
    a, b = a.double(), b.double()
    return float(((a - b).abs() / (step * torch.maximum(a.abs(), b.abs()) + 1e-4 * b.abs().max())).max())


def build_seq(mods, dtype, all_outputs):
    seq = DecodeSequence(H, "cuda", lut_mode="exact", dtype=dtype)
    prev, vecs = seq.input, []
    for i, m in enumerate(mods):
        _, K, N, off = LAYER[i % 4]
        prev = seq.matvec(m, prev[off:off + K])
        vecs.append(prev)
    return seq.compile(outputs=vecs if all_outputs else vecs[-1:])


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)
    nlayers = 2 if quick else 32
    blocks = 5 if quick else 7
    mods = [synth_module(4, K, N, seed=1000 + 4 * layer + j) for layer in range(nlayers) for j, (_, K, N, _) in enumerate(LAYER)]
    x = torch.randn(H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    xb, x16 = x.bfloat16(), x.half()

    # ---- correctness: every item against a one-GEMV launch of its dtype on the input it consumed ----
    check = {}
    for dtype, xin, step in ((torch.float16, x16, 2.0 ** -10), (torch.bfloat16, xb, 2.0 ** -7)):
        seq = build_seq(mods, dtype, True)
        seq.x.copy_(xin)
        outs = [o.clone() for o in seq.replay()]
        torch.cuda.synchronize()
        assert not seq.error()
        worst = 0.0
        for i, m in enumerate(mods):
            _, K, N, off = LAYER[i % 4]
            inp = xin if i == 0 else outs[i - 1][off:off + K].clone()
            y = m(inp)
            worst = max(worst, steps_apart(outs[i], y, step))
        assert worst <= 1.0 + 1e-6, (dtype, worst)
        check[str(dtype)] = dict(items=len(mods), max_steps_vs_one_gemv=round(worst, 3), last_absmax=float(outs[-1].abs().max()))
        del seq
    print(json.dumps({"kind": "check", **check}), flush=True)

    # ---- timing: one token ----
    s16, sbf = build_seq(mods, torch.float16, False), build_seq(mods, torch.bfloat16, False)
    s16.x.copy_(x16)
    sbf.x.copy_(xb)

    def step(v):
        cur = v
        for i, m in enumerate(mods):
            _, K, N, off = LAYER[i % 4]
            cur = m(cur[off:off + K])
        return cur

    graph = GraphedDecodeStep(step, xb, warmup=2)
    graph.x_dev.copy_(xb)
    ys = sbf.replay()[0].clone()
    yg = graph.replay().clone()
    torch.cuda.synchronize()
    rel = float((ys.double() - yg.double()).abs().max() / yg.double().abs().max())
    n = 5 if quick else 20
    t = timed({"seq_fp16": s16.replay, "seq_bf16": sbf.replay, "graph_bf16": graph.replay}, n, blocks)
    assert not s16.error() and not sbf.error()
    rec = dict(kind="7B-token", layers=nlayers, items=len(mods), **{k + "_ms": v for k, v in t.items()},
               bf16_vs_fp16_seq=round(t["seq_bf16"] / t["seq_fp16"], 4), seq_bf16_speedup_vs_graph_bf16=round(t["graph_bf16"] / t["seq_bf16"], 3),
               last_output_max_norm_seq_vs_graph_bf16=float(f"{rel:.3e}"))
    print(json.dumps(rec), flush=True)
    del s16, sbf, graph

    # ---- the world-1 exchange per launch ----
    for j, (name, K, N, _) in enumerate(LAYER):
        m = mods[j]
        lay = (m.qweight, m.lookup_table, 4, None, m.rows, m.cols, m.vals, m.full_rows, m.full_row_indices)
        xk = torch.randn(K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(j))
        xk16, xkb = xk.half(), xk.bfloat16()
        xarena = torch.zeros(2 * 2 * N + 8192, dtype=torch.uint8, device="cuda")
        xbase = torch.tensor([xarena.data_ptr()], dtype=torch.int64, device="cuda")

        def f16():
            qc.lutgemv_fused_exchange(xk16, *lay, xbase.data_ptr(), 4096, 0, 64, 128, 1, 0, 1, N)

        def fbf():
            qc.lutgemv_fused_exchange_bf16(xkb, *lay, xbase.data_ptr(), 4096, 0, 64, 128, 1, 0, 1, N)

        fbf()
        torch.cuda.synchronize()
        got = xarena[4096:4096 + 2 * N].view(torch.bfloat16).clone()
        assert int(xarena[128:132].view(torch.int32).item()) == 0
        step1 = steps_apart(got, qc.lutgemv_fused(xkb, *lay), 2.0 ** -7)
        assert step1 <= 1.0 + 1e-6, (name, step1)
        t = timed({"xchg_fp16": f16, "xchg_bf16": fbf}, 50 if quick else 200, blocks)
        print(json.dumps(dict(kind="exchange-world1", shape=name, K=K, N=N, **{k + "_ms": v for k, v in t.items()},
                              bf16_vs_fp16=round(t["xchg_bf16"] / t["xchg_fp16"], 4), max_steps_vs_lutgemv_fused=round(step1, 3))), flush=True)


if __name__ == "__main__":
    main()
