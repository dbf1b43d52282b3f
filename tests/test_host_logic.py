"""CPU tests of the host-side mirror of the reference interface (squeezellm/quant.py) and of the column-sharding
logic (world_size-2 gloo; the local compute is the CPU oracle - the CUDA module is covered by -m gpu)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.nn as nn

from util import layer_as_read, orc, quant_layer, rel_err, TIGHT_TOL


def test_quantlinearlut_buffers_match_reference_format():
    from squeezellm_b200.quant import QuantLinearLUT
    m = QuantLinearLUT(3, 256, 128, True, include_sparse=True, numvals=77, topX=10)
    sd = m.state_dict()
    assert {k: (tuple(v.shape), v.dtype) for k, v in sd.items()} == {
        "qweight": ((24, 128), torch.int32), "bias": ((128,), torch.float32), "lookup_table": ((128, 8), torch.float32),
        "rows": ((129,), torch.int32), "cols": ((77,), torch.int32), "vals": ((77,), torch.float32),
        "full_rows": ((256, 10), torch.float32), "full_row_indices": ((10,), torch.int32)}
    m4 = QuantLinearLUT(4, 256, 128, False)
    assert set(m4.state_dict()) == {"qweight", "lookup_table"} and m4.qweight.shape == (32, 128) and m4.bias is None
    with pytest.raises(NotImplementedError):
        QuantLinearLUT(2, 256, 128, False)
    with pytest.raises(NotImplementedError, match="balanced"):
        QuantLinearLUT(4, 256, 128, False, include_sparse=True, numvals=5, balanced=True)


@pytest.mark.parametrize("kind", ["dense", "csr", "csr+dense-rows", "biased"])
def test_from_buffers_equals_constructor_and_load_state_dict(kind):
    """QuantLinearLUT.from_buffers: the state_dict (keys, dtypes, values) and attributes of the constructor + load_state_dict,
    holding the given tensors themselves (no copy)."""
    from squeezellm_b200.quant import QuantLinearLUT
    sp, topx = {"dense": (0.0, 0), "csr": (0.02, 0), "csr+dense-rows": (0.02, 5), "biased": (0.02, 5)}[kind]
    L = orc.make_layer(3, 256, 128, sparsity=sp, topX=topx, seed=6, nonzero_full_rows=True, bias=kind == "biased")
    buffers = {k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)}
    want = QuantLinearLUT(3, 256, 128, L["bias"] is not None, include_sparse=sp > 0, numvals=len(L["vals"]) if sp else 0, topX=topx)
    want.load_state_dict(buffers)
    got = QuantLinearLUT.from_buffers(3, buffers)
    sd, sd_want = got.state_dict(), want.state_dict()
    assert list(sd) == list(sd_want)
    assert all(sd[k].dtype == sd_want[k].dtype and torch.equal(sd[k], sd_want[k]) for k in sd)
    attrs = ("infeatures", "outfeatures", "bits", "include_sparse", "include_bias", "numvals", "topX")
    assert [getattr(got, a) for a in attrs] == [getattr(want, a) for a in attrs]
    assert all(getattr(got, k) is t for k, t in buffers.items())
    for missing in ("qweight", "lookup_table", "rows", "vals", "full_row_indices"):  # incomplete sets fail here, not at a launch
        if missing in buffers:
            with pytest.raises((ValueError, KeyError)):
                QuantLinearLUT.from_buffers(3, {k: t for k, t in buffers.items() if k != missing})


def test_make_quant_lut_replaces_named_linears_like_the_reference():
    from squeezellm_b200.quant import QuantLinearLUT, make_quant_lut

    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.o_proj = nn.Linear(128, 128, bias=False), nn.Linear(128, 64, bias=True)

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.layers = nn.ModuleList([Block(), Block()])
            self.lm_head = nn.Linear(128, 32, bias=False)

    net = Net()
    names = {f"layers.{i}.{n}" for i in range(2) for n in ("q_proj", "o_proj")}   # lm_head stays fp16 (llama.py:172-174)
    numvals = {n: 11 for n in names}
    make_quant_lut(net, names, 4, include_sparse=True, numvals=numvals, topX=10)
    for i in range(2):
        q, o = net.layers[i].q_proj, net.layers[i].o_proj
        assert isinstance(q, QuantLinearLUT) and isinstance(o, QuantLinearLUT)
        assert (q.infeatures, q.outfeatures, q.bias) == (128, 128, None) and o.bias is not None and o.outfeatures == 64
        assert q.cols.numel() == 11 and q.topX == 10 and q.full_rows.shape == (128, 10)
    assert isinstance(net.lm_head, nn.Linear)
    # llama.py:181-182: load_state_dict(strict=False) with checkpoint keys == buffer names
    sd = {"layers.0.q_proj.qweight": torch.ones((16, 128), dtype=torch.int32)}
    missing = net.load_state_dict(sd, strict=False)
    assert int(net.layers[0].q_proj.qweight[0, 0]) == 1 and "layers.0.q_proj.lookup_table" in missing.missing_keys


def test_round_to_nearest_pole_sim():
    from squeezellm_b200.quant import round_to_nearest_pole_sim
    poles = np.array([-0.5, -0.1, 0.2, 0.7], dtype=np.float32)
    w = torch.tensor([0.0, 0.16, -0.4, 9.0])
    assert torch.allclose(round_to_nearest_pole_sim(w, poles), torch.tensor([-0.1, 0.2, -0.5, 0.7]))


def test_shard_bounds_and_state_reassemble():
    from squeezellm_b200.sharding import shard_bounds, shard_state
    assert shard_bounds(22016, 8) == [(i * 2752, (i + 1) * 2752) for i in range(8)]       # 65B gate/up: not 128-divisible
    b = shard_bounds(132, 8)
    assert b[0] == (0, 20) and b[-1][1] == 132 and all((c1 - c0) % 4 == 0 for c0, c1 in b)
    L = orc.make_layer(4, 256, 132, sparsity=0.02, topX=10, seed=4, nonzero_full_rows=True, bias=True)
    st = {k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)}
    x = orc.make_vec(256, seed=1)
    want = orc.forward_f64(L, x, mul_init=L["bias"][None])
    got = np.zeros_like(want)
    for c0, c1 in b:
        s = shard_state(st, c0, c1)
        Ls = dict(bits=4, infeatures=256, outfeatures=c1 - c0, **{k: v.numpy() for k, v in s.items()})
        got[:, c0:c1] = orc.forward_f64(Ls, x, mul_init=Ls["bias"][None])
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)


def _csr_in_first_half():
    """w4 128 -> 64 with CSR outliers in channels [0, 32) only and dense rows for channels 5, 40 and 50: the second half of a
    two-way split gets an empty CSR next to its dense rows."""
    L = orc.make_layer(4, 128, 64, sparsity=0.05, topX=3, seed=11, nonzero_full_rows=True)
    n = int(L["rows"][32])
    L["rows"] = np.concatenate([L["rows"][:33], np.full(32, n)]).astype(np.int32)
    L["cols"], L["vals"] = L["cols"][:n], L["vals"][:n]
    L["full_row_indices"] = np.array([5, 40, 50], dtype=np.int32)
    return L


def test_shard_without_csr_entries_keeps_its_dense_rows():
    """A shard whose channels have no CSR entry holds an empty CSR, so its forward still reads its dense rows: the shards of
    from_full and of a ShardedSiblingGroup reassemble the full layer.  from_full rejects arguments that contradict the state."""
    from squeezellm_b200.sharding import ShardedQuantLinearLUT, ShardedSiblingGroup
    L = _csr_in_first_half()
    st = {k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)}
    x = orc.make_vec(128, seed=1)
    want = orc.forward_f64(L, x)
    for rank, (c0, c1) in enumerate([(0, 32), (32, 64)]):
        shard = ShardedQuantLinearLUT.from_full(st, 4, 128, 64, rank, 2, True, 3, "cpu").local
        group = ShardedSiblingGroup([quant_layer(L)], rank, 2, "o_proj").layer
        for m in (shard, group):
            assert m._sparse_args()[3] is not None
            assert np.allclose(orc.forward_f64(layer_as_read(m), x), want[:, c0:c1], rtol=1e-12, atol=1e-12)
    for args in ((4, 96, 64, 0, 2, True, 3), (4, 128, 64, 0, 2, False, 3), (4, 128, 64, 0, 2, True, 0)):
        with pytest.raises(ValueError, match="from_full"):
            ShardedQuantLinearLUT.from_full(st, *args, "cpu")


def test_sharded_members_refuse_dequantize_and_dissolve():
    """A sharded member holds only its rank's columns: dequantize / to_linear and its group's dissolve raise and change nothing."""
    from squeezellm_b200.sharding import ShardedSiblingGroup
    ms = [quant_layer(orc.make_layer(4, 128, 64, sparsity=0.02, topX=3, seed=20 + i, nonzero_full_rows=True)) for i in range(3)]
    g = ShardedSiblingGroup(ms, 0, 2, "qkv")

    def snapshot():
        return [(m._sibling_group, m.outfeatures, {k: (v.data_ptr(), tuple(v.shape)) for k, v in m.state_dict().items()})
                for m in ms]
    before = snapshot()
    for m in ms:
        with pytest.raises(NotImplementedError, match="sharded"):
            m.dequantize()
        with pytest.raises(NotImplementedError, match="sharded"):
            m.to_linear()
    with pytest.raises(NotImplementedError, match="dissolve"):
        g.dissolve()
    assert snapshot() == before and all(m._sibling_group[0] is g for m in ms)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from squeezellm_b200.sharding import ShardedQuantLinearLUT, shard_bounds, shard_state
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        L = orc.make_layer(3, 256, 136, sparsity=0.02, topX=4, seed=9, nonzero_full_rows=True)
        st = {k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray)}
        c0, c1 = shard_bounds(136, world)[rank]
        s = shard_state(st, c0, c1)
        Ls = dict(bits=3, infeatures=256, outfeatures=c1 - c0, **{k: v.numpy() for k, v in s.items()})
        x = torch.from_numpy(orc.make_vec(256, seed=2))

        def local(xx):  # CPU stand-in for the CUDA shard kernel
            return torch.from_numpy(orc.forward_f64(Ls, xx.numpy()).astype(np.float32))

        m = ShardedQuantLinearLUT(None, 136, c0, c1, matvec_fn=local)
        y = m(x)
        q.put((rank, y.numpy(), orc.forward_f64(L, x.numpy())))
    finally:
        dist.destroy_process_group()


def test_column_sharded_allreduce_world2_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, y, want in res:
        assert y.shape == (1, 136)
        assert rel_err(y, want) < TIGHT_TOL, f"rank {rank}"


def _worker_stacked(rank, world, port, q):
    import torch.distributed as dist
    from squeezellm_b200.sharding import exchange_stacked
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        N, members = 24, 3
        w = N // world
        full = torch.arange(members * N, dtype=torch.float32).reshape(members, N) + 1.0   # member m's full output vector
        y_local = torch.cat([full[m, rank * w:(rank + 1) * w] for m in range(members)])     # what the stacked shard computes
        out = exchange_stacked(y_local, members, rank, world)
        buf = torch.full((members, N), 7.0)                                                  # reused buffer must be re-zeroed
        out2 = exchange_stacked(y_local, members, rank, world, out=buf)
        q.put((rank, torch.equal(out, full), torch.equal(out2, full) and out2.data_ptr() == buf.data_ptr()))
    finally:
        dist.destroy_process_group()


def test_stacked_shard_exchange_world2_gloo():
    """One all-reduce rebuilds the full outputs of all members of a stacked (q/k/v-style) column shard."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_stacked, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(a and b for _, a, b in res), res


def _layer_dict(m):
    """QuantLinearLUT (CPU buffers) -> the oracle's layer dict."""
    d = dict(bits=m.bits, infeatures=m.infeatures, outfeatures=m.outfeatures, qweight=m.qweight.contiguous().numpy(),
             lookup_table=m.lookup_table.contiguous().numpy(), bias=m.bias.numpy() if m.bias is not None else None)
    for k in ("rows", "cols", "vals", "full_rows", "full_row_indices"):
        d[k] = getattr(m, k).numpy() if hasattr(m, k) else None
    return d


def _worker_shard_model(rank, world, port, q):
    import torch.distributed as dist
    from squeezellm_b200.sharding import shard_model
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        class Attn(nn.Module):
            def __init__(self):
                super().__init__()
                self.full = {}
                for i, n in enumerate(("q_proj", "k_proj", "v_proj", "o_proj")):
                    L = orc.make_layer(4, 128, 64, sparsity=0.05, topX=3, seed=40 + i, nonzero_full_rows=True)
                    self.full[n] = L
                    setattr(self, n, quant_layer(L))

        attn = Attn()
        groups = shard_model(attn, rank, world)
        for g in groups:  # CPU stand-in for the CUDA launch of the stacked shard
            g.compute = lambda layer, xx: torch.from_numpy(orc.forward_f64(_layer_dict(layer), xx.numpy().reshape(1, -1)).astype(np.float32))
        x = torch.from_numpy(orc.make_vec(128, seed=5)).reshape(1, 128)
        outs = {n: getattr(attn, n)(x).numpy() for n in ("q_proj", "k_proj", "v_proj", "o_proj")}
        ok = all(rel_err(outs[n], orc.forward_f64(attn.full[n], x.numpy())) < TIGHT_TOL for n in outs)
        shapes = sorted((len(g.members), g.launches, g.w) for g in groups)
        q.put((rank, ok, shapes, attn.q_proj.qweight.shape[1]))
    finally:
        dist.destroy_process_group()


def test_shard_model_world2_gloo():
    """shard_model: q/k/v become one stacked shard + one exchange, o_proj a group of one; every rank gets full-width outputs."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_shard_model, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, shapes, width in res:
        assert ok, f"rank {rank}"
        assert shapes == [(1, 1, 32), (3, 1, 32)], shapes     # o_proj alone (1 launch), q/k/v together (1 launch), 32 columns per rank
        assert width == 32                                     # members now hold this rank's shard
