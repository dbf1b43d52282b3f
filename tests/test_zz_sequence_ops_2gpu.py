"""The sequence kernel's ops across TWO real GPUs (skipped with fewer than two).  Every rank records the same chain over its own column
shards, stacked siblings as members (sharding.ShardedSiblingGroup), and passes sharding.PeerArena: the inputs, the up slices of the
SiLU gating and the residuals are polled at system scope out of the words the owners store into every rank's arena.  Each rank
exports every item's full-length vector, and each vector is checked per element against the fp64 oracle of the UNSHARDED layers
applied to the exported sources, with the bound of tests/test_sequence_ops_gpu.py:

    0  o    = o_proj(a) + h                          residual: an external vector
    1  gu   = [gate | up](rmsnorm(o))                two members
    2  d    = down(silu(gu[:I]) * gu[I:]) + o        SiLU gating within one item's vector; residual: item 0
    3  qkv  = [q | k | v](rmsnorm(d)) + r            three members; residual: an external vector of the three members' full length
    4  gu2  = [gate2 | up2](rmsnorm(d)) + gu         two members; residual: item 1 (member-wise full-length indices)

One replay has a late rank (the others wait inside the kernel, bounded, and nothing is lost)."""
import os
import sys
import time

import numpy as np
import pytest
import torch

from util import ROOT

pytestmark = pytest.mark.gpu

H, I = 512, 768


def _worker(rank, world, port, results):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        from test_sequence_ops_gpu import TDT, _check, _layer, _round, _vec, rmsnorm64, silu_mul64
        from squeezellm_b200.runtime import DecodeSequence
        from squeezellm_b200.sharding import PeerArena, ShardedSiblingGroup
        worst = 0.0
        for bits, mode in ((4, "exact"), (3, "bf16"), (4, "fp16")):
            dt = TDT[mode]
            names = {"o": (H, H), "gate": (H, I), "up": (H, I), "down": (I, H), "q": (H, H), "k": (H, H), "v": (H, H),
                     "gate2": (H, I), "up2": (H, I)}
            L, M = {}, {}
            for j, (nm, (K, N)) in enumerate(names.items()):
                L[nm], M[nm] = _layer(bits, K, N, "csr", seed=500 + 10 * j + bits)
            shard = lambda ms, nm: ShardedSiblingGroup([M[m] for m in ms], rank, world, nm).layer   # noqa: E731
            o_l, gu_l, d_l = shard(["o"], "o"), shard(["gate", "up"], "gu"), shard(["down"], "d")
            qkv_l, gu2_l = shard(["q", "k", "v"], "qkv"), shard(["gate2", "up2"], "gu2")
            rng = np.random.default_rng(bits)
            w1, w2 = (_round(1.0 + 0.1 * rng.standard_normal(H), dt) for _ in range(2))
            w1_t, w2_t = (torch.from_numpy(w).to(dev, dt) for w in (w1, w2))

            seq = DecodeSequence(H, dev, lut_mode="fp16" if mode == "fp16" else "exact", peer=PeerArena(rank, world, dev), dtype=dt)
            hv, h_t = seq.new_input(H)
            rv, r_t = seq.new_input(3 * H)
            o = seq.matvec(o_l, seq.input, residual=hv)
            gu = seq.matvec(gu_l, o, members=2, norm=(w2_t, 1e-5))
            d = seq.matvec(d_l, gu[0:I], up=gu[I:2 * I], residual=o)
            qkv = seq.matvec(qkv_l, d, members=3, norm=(w1_t, 1e-5), residual=rv)
            gu2 = seq.matvec(gu2_l, d, members=2, norm=(w2_t, 1e-5), residual=gu)
            seq.compile(outputs=[o, gu, d, qkv, gu2])

            for rep in range(3):
                a, h, r = _vec(H, 10 + rep, dt), _vec(H, 20 + rep, dt), _vec(3 * H, 30 + rep, dt)
                seq.x.copy_(torch.from_numpy(a).to(dev, dt))
                h_t.copy_(torch.from_numpy(h).to(dev, dt))
                r_t.copy_(torch.from_numpy(r).to(dev, dt))
                if rep == 1 and rank == 1:
                    torch.cuda.synchronize()
                    time.sleep(0.3)
                outs = [x.clone() for x in seq.replay()]
                torch.cuda.synchronize()
                assert not seq.error(), "a bounded in-kernel wait gave up"
                go, ggu, gd, gqkv, ggu2 = (x.double().cpu().numpy() for x in outs)
                n_o = rmsnorm64(go, w2, 1e-5)
                n_d1, n_d2 = rmsnorm64(gd, w1, 1e-5), rmsnorm64(gd, w2, 1e-5)
                checks = [(go, "o", a, h, None), (ggu[:I], "gate", n_o, None, "rms"), (ggu[I:], "up", n_o, None, "rms"),
                          (gd, "down", silu_mul64(ggu[:I], ggu[I:]), go, "silu")]
                checks += [(gqkv[m * H:(m + 1) * H], nm, n_d1, r[m * H:(m + 1) * H], "rms") for m, nm in enumerate("qkv")]
                checks += [(ggu2[m * I:(m + 1) * I], nm, n_d2, ggu[m * I:(m + 1) * I], "rms") for m, nm in enumerate(("gate2", "up2"))]
                for got, nm, xp, res, tr in checks:
                    worst = max(worst, _check(got, L[nm], xp, mode, dt, res=res, what=f"rank {rank} w{bits} {mode} rep {rep} {nm}", transform=tr))
            dist.barrier()
            del seq
        results[rank] = worst
    except BaseException as e:  # noqa: BLE001 - reported by the parent
        results[rank] = f"{type(e).__name__}: {e}"
    finally:
        torch.cuda.synchronize()
        os._exit(0)


def test_sequence_ops_two_gpus_match_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    results = ctx.Manager().dict()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, results)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert not p.is_alive(), "worker hung"
    res = dict(results)
    assert len(res) == 2 and all(isinstance(v, float) and v <= 1.0 for v in res.values()), res
