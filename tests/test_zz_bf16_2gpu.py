"""bf16 decode across TWO real GPUs (skipped with fewer than two GPUs): a bf16 DecodeSequence over column shards with a PeerArena,
including a late rank, and a bf16 stacked layer through ShardedSiblingGroup + PeerExchange.  Every rank must end up with the full
vectors of the fp64 oracle of the UNSHARDED layers, with bf16 hand-overs, in bf16."""
import os
import sys
import time

import numpy as np
import pytest
import torch

from util import ROOT, orc

pytestmark = pytest.mark.gpu

CHAIN_TOL = 2 * 2.0 ** -7   # two bf16 steps of the largest output (tests/test_sequence_bf16_gpu.py)


def _bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).bfloat16().double().numpy()


def _worker(rank, world, port, results):
    import torch.distributed as dist
    import torch.nn as nn
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    from squeezellm_b200.quant import QuantLinearLUT
    from squeezellm_b200.runtime import DecodeSequence
    from squeezellm_b200.sharding import PeerArena, PeerExchange, ShardedSiblingGroup, shard_bounds, shard_state
    try:
        worst = 0.0
        # ---- a bf16 sequence over column shards ----
        for bits, dims in ((4, [(4096, 4096, 0), (2048, 11008, 1024), (11008, 4096, 0), (4096, 8192, 0)]),
                           (3, [(512, 1024, 0), (512, 768, 256), (768, 512, 0)])):
            Ls = []
            for i, (K, N, _) in enumerate(dims):
                L = orc.make_layer(bits, K, N, sparsity=0.0045 if K > 1000 else 0.02, topX=6, seed=300 + 7 * i + bits, nonzero_full_rows=True)
                L["lookup_table"] = (L["lookup_table"] * (50.0 / np.sqrt(K))).astype(np.float32)
                Ls.append(L)
            peer = PeerArena(rank, world, dev)
            seq = DecodeSequence(dims[0][0], dev, lut_mode="exact", peer=peer, dtype=torch.bfloat16)
            prev, vecs, keep = seq.input, [], []
            for L, (K, N, off) in zip(Ls, dims):
                c0, c1 = shard_bounds(N, world)[rank]
                st = shard_state({k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else None) for k, v in L.items()
                                  if k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices")}, c0, c1)
                m = QuantLinearLUT(bits, K, c1 - c0, False, include_sparse=True, numvals=int(st["vals"].numel()), topX=6)
                m.load_state_dict(st, strict=False)
                m = m.to(dev)
                keep.append(m)
                prev = seq.matvec(m, prev[off:off + K])
                vecs.append(prev)
            seq.compile(outputs=vecs)
            for rep in range(3):
                x = _bf16(orc.make_vec(dims[0][0], seed=10 + rep).reshape(-1))
                seq.x.copy_(torch.from_numpy(x).to(dev))
                if rep == 1 and rank == 1:
                    torch.cuda.synchronize()
                    time.sleep(0.3)      # a late rank: the others wait inside the kernel (bounded), nothing is lost
                outs = [o.clone() for o in seq.replay()]
                torch.cuda.synchronize()
                assert not seq.error()
                cur = None
                for o, L, (K, N, off) in zip(outs, Ls, dims):
                    xin = x if cur is None else cur[off:off + K]
                    cur = _bf16(orc.forward_f64(L, xin.astype(np.float32).reshape(1, K)).reshape(N))
                    assert o.dtype == torch.bfloat16
                    got = o.double().cpu().numpy()
                    worst = max(worst, float(np.abs(got - cur).max() / np.abs(cur).max()))
            dist.barrier()
        # ---- a bf16 stacked layer through PeerExchange ----
        pex = PeerExchange(rank, world, dev)
        bits, K, N = 4, 4096, 4096
        Ls = [orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=40 + i, nonzero_full_rows=True, bias=True) for i in range(3)]
        members = []
        for L in Ls:
            m = QuantLinearLUT(bits, K, N, True, include_sparse=True, numvals=len(L["vals"]), topX=10)
            m.load_state_dict({k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray) and k in m.state_dict()}, strict=False)
            members.append(m.to(dev))
        box = nn.Module()
        box.q_proj, box.k_proj, box.v_proj = members
        ShardedSiblingGroup(members, rank, world, "a", peer=pex)
        for it in range(3):
            xt = torch.from_numpy(orc.make_vec(K, seed=it + 1)).to(dev).reshape(-1).bfloat16()
            xb = xt.float().cpu().numpy().reshape(1, K)
            if it == 1 and rank == 1:
                time.sleep(0.3)
            ys = [m(xt) for m in members]
            torch.cuda.synchronize()
            for y, L in zip(ys, Ls):
                assert y.dtype == torch.bfloat16 and y.shape == (N,)
                w = orc.forward_f64(L, xb, mul_init=L["bias"][None, :]).reshape(-1)
                worst = max(worst, float(np.abs(y.double().cpu().numpy() - w).max() / np.abs(w).max()))
        assert not pex.error()
        dist.barrier()
        results[rank] = worst
    finally:
        torch.cuda.synchronize()
        os._exit(0 if results.get(rank) is not None else 1)   # symmetric-memory / NCCL teardown can hang: leave without it


def test_bf16_sequence_and_exchange_on_two_gpus():
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
    hung = [p for p in procs if p.is_alive()]
    for p in hung:
        p.kill()
    assert not hung, "worker hung"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert len(results) == 2 and max(results.values()) < CHAIN_TOL, dict(results)
