"""The exchange entry point with bf16 activations (sqllm_lutgemv_fused_exchange_dt / quant_cuda.lutgemv_fused_exchange_bf16) on ONE GPU:
world = 1, the "peer" arena is the local one, so the kernel path is the multi-GPU one (stores through the arena base table, system-scope
publish, wait on the local counter).  The arena vectors are bf16, each element rounded once with the bias inside the fp32 sum; they
are checked per element against the fp64 oracle on the bf16 input (bound_ratio <= 1) and against lutgemv_fused on the same input.
A ShardedSiblingGroup over a world-1 PeerExchange (a plain CUDA arena instead of symmetric memory) must give the unsharded bf16
module path's results with no dtype conversion."""
import numpy as np
import pytest
import torch

from util import OUT_ROUNDING, abs_sum, bound_ratio, orc, to_torch

pytestmark = pytest.mark.gpu

FLAG, STATE, ERROR, DATA = 0, 64, 128, 4096
R_BF16, ETA_BF16 = OUT_ROUNDING["bfloat16"]


def one_step_apart(a, b):
    """Two bf16 results of the same fp32-accumulated value summed in different orders: at most one bf16 rounding step apart."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return bool(np.all(np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + ETA_BF16))


@pytest.mark.parametrize("bits,K,w,members,sp,topx", [(4, 1024, 1024, 2, 0.01, 4), (3, 512, 256, 1, 0.0, 0), (4, 4096, 4096, 3, 0.0045, 10),
                                                      (4, 256, 32, 1, 0.02, 4),  # narrower than one strip: one ragged strip
                                                      (3, 1024, 512, 3, 0.01, 40)],  # more than 32 dense rows: the general dense-row branch
                         ids=["w4-2x1024", "w3-1x256", "w4-qkv", "w4-1x32", "w3-3x512-t40"])
def test_bf16_exchange_world1_matches_oracle_and_counts_arrivals(bits, K, w, members, sp, topx):
    from squeezellm_b200 import quant as Q
    qc = Q.quant_cuda
    N = members * w
    L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=K + N, nonzero_full_rows=True, bias=True)
    if topx and sp == 0:
        L["full_rows"] = L["full_row_indices"] = None
    T = to_torch(L)
    xt = torch.from_numpy(orc.make_vec(K, seed=6)).cuda().reshape(-1).bfloat16()
    xb = xt.float().cpu().numpy().reshape(1, K)
    arena = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    base = torch.tensor([arena.data_ptr()], dtype=torch.int64, device="cuda")
    want = orc.forward_f64(L, xb, mul_init=L["bias"][None, :]).reshape(-1)
    S = abs_sum(L, xb, L["bias"]).reshape(-1)

    def counter(off):
        return int(arena[off:off + 8].view(torch.int64).item())

    for call in (1, 2):  # counters only grow: the second call must wait for 2x the arrivals and still deliver
        arena[DATA:DATA + 2 * N].zero_()
        qc.lutgemv_fused_exchange_bf16(xt, T["qweight"], T["lookup_table"], bits, T["bias"], T.get("rows"), T.get("cols"), T.get("vals"),
                                       T.get("full_rows"), T.get("full_row_indices"), base.data_ptr(), DATA, FLAG, STATE, ERROR,
                                       1, 0, members, w)
        torch.cuda.synchronize()
        got = arena[DATA:DATA + 2 * N].view(torch.bfloat16).float().cpu().numpy().astype(np.float64)
        assert bound_ratio(got, want, S, want, R_BF16, eta=ETA_BF16) <= 1.0
        assert int(arena[ERROR:ERROR + 4].view(torch.int32).item()) == 0
        nown = counter(FLAG) // call
        assert 1 <= nown <= min(qc.sm_count(), (N + 63) // 64) and counter(FLAG) == call * nown and counter(STATE) == call * nown
    # the plain fused call on the same bf16 input
    y = qc.lutgemv_fused(xt, T["qweight"], T["lookup_table"], bits, T["bias"], T.get("rows"), T.get("cols"), T.get("vals"),
                         T.get("full_rows"), T.get("full_row_indices"))
    assert y.dtype == torch.bfloat16
    assert one_step_apart(got, y.float().cpu().numpy())


def test_bf16_exchange_rejects_other_dtypes():
    from squeezellm_b200 import quant as Q
    qc = Q.quant_cuda
    T = to_torch(orc.make_layer(4, 256, 128, seed=3))
    arena = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    base = torch.tensor([arena.data_ptr()], dtype=torch.int64, device="cuda")
    for dt in (torch.float16, torch.float32):
        x = torch.zeros(256, device="cuda", dtype=dt)
        with pytest.raises(RuntimeError, match="lutgemv_fused_exchange_bf16: x must be bf16"):
            qc.lutgemv_fused_exchange_bf16(x, T["qweight"], T["lookup_table"], 4, None, None, None, None, None, None, base.data_ptr(),
                                           DATA, FLAG, STATE, ERROR, 1, 0, 1, 128)


def _local_peer(device):
    from squeezellm_b200.sharding import PeerExchange

    class LocalPeerExchange(PeerExchange):
        """A world-1 PeerExchange on a plain CUDA arena: everything but the symmetric-memory rendezvous."""

        def __init__(self, device, arena_bytes=8 << 20):
            self.rank, self.world, self.device, self.group = 0, 1, device, None
            self.arena = torch.zeros(arena_bytes, dtype=torch.uint8, device=device)
            self._base = torch.tensor([self.arena.data_ptr()], dtype=torch.int64, device=device)
            self.peer_base = self._base.data_ptr()
            self.offsets, self.next = {}, self.DATA
            self.arena_bytes = arena_bytes
            self.calls, self.check_every = 0, 4096

    return LocalPeerExchange(device)


def _block(seed):
    """A tiny Llama-shaped decoder block of QuantLinearLUT layers (hidden 256, intermediate 704), q/k/v with a bias."""
    from squeezellm_b200.quant import QuantLinearLUT
    H, I = 256, 704
    shapes = {"q_proj": (H, H, True), "k_proj": (H, H, True), "v_proj": (H, H, True), "o_proj": (H, H, False),
              "gate_proj": (H, I, False), "up_proj": (H, I, False), "down_proj": (I, H, False)}
    block, layers = torch.nn.Module(), {}
    for i, (name, (K, N, bias)) in enumerate(shapes.items()):
        L = orc.make_layer(4, K, N, sparsity=0.01, topX=3, seed=seed + i, nonzero_full_rows=True, bias=bias)
        L["lookup_table"] = (L["lookup_table"] * (50.0 / np.sqrt(K))).astype(np.float32)
        m = QuantLinearLUT(4, K, N, bias, include_sparse=True, numvals=len(L["vals"]), topX=3)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray) and k in m.state_dict()}, strict=False)
        setattr(block, name, m.cuda())
        layers[name] = L
    return block, layers


def _run_block(block, x, feed=None):
    """The block's seven matvecs on x; `feed` (an earlier run's results) supplies the inputs after the first, so that two runs compare
    layer by layer on identical inputs."""
    q, k, v = block.q_proj(x), block.k_proj(x), block.v_proj(x)
    o = block.o_proj(v if feed is None else feed["v_proj"])
    gi = o if feed is None else feed["o_proj"]
    g, u = block.gate_proj(gi), block.up_proj(gi)
    d = block.down_proj((g * u).contiguous() if feed is None else feed["gate_up"])
    return {"q_proj": q, "k_proj": k, "v_proj": v, "o_proj": o, "gate_proj": g, "up_proj": u, "down_proj": d,
            "gate_up": (g * u).contiguous()}


def test_sharded_block_through_a_world1_peer_exchange_matches_the_module_path(monkeypatch):
    from squeezellm_b200.quant import quant_cuda as qc
    from squeezellm_b200.sharding import shard_model
    ref, layers = _block(seed=50)
    sharded, _ = _block(seed=50)
    peer = _local_peer(torch.device("cuda"))
    calls = []
    for n in ("lutgemv_fused_exchange", "lutgemv_fused_exchange_bf16"):
        real = getattr(qc, n)
        monkeypatch.setattr(qc, n, (lambda real, n: lambda *a, **kw: (calls.append((n, a[0].dtype)), real(*a, **kw))[1])(real, n))
    groups = shard_model(sharded, 0, 1, peer=peer)
    assert len(groups) == 4   # q/k/v and gate/up stacked, o and down groups of one
    for s in (1, 2):
        x = torch.from_numpy(orc.make_vec(256, seed=60 + s)).cuda().reshape(1, 1, 256).bfloat16()
        want = _run_block(ref, x)
        del calls[:]
        got = _run_block(sharded, x, feed=want)
        torch.cuda.synchronize()
        assert calls == [("lutgemv_fused_exchange_bf16", torch.bfloat16)] * 4, calls   # one launch per group, bf16 in, no conversion
        for name, y in got.items():
            if name == "gate_up":
                continue
            assert y.dtype == torch.bfloat16 and y.shape == want[name].shape, name
            assert one_step_apart(y.float().cpu().numpy(), want[name].float().cpu().numpy()), name
        # q against the fp64 oracle on the bf16 input, bias inside the sum
        xb = x.float().cpu().numpy().reshape(1, 256)
        L = layers["q_proj"]
        wq = orc.forward_f64(L, xb, mul_init=L["bias"][None, :])
        assert bound_ratio(got["q_proj"].float().cpu().numpy().reshape(1, -1), wq, abs_sum(L, xb, L["bias"]), wq, R_BF16, eta=ETA_BF16) <= 1.0
    assert not peer.error()
