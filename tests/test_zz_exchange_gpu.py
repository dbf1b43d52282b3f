"""The exchange entry point (sqllm_lutgemv_fused_exchange / quant_cuda.lutgemv_fused_exchange) on ONE GPU: world = 1, the
"peer" arena is the local one.  Same kernel path as the multi-GPU run (stores through the arena base table, system-scope
publish, wait on the local counter); the multi-rank behaviour itself is checked by bench.py's start-up self-check against
the NCCL path and, since round 2, against the fp64 oracle (bench.py parity_check)."""
import numpy as np
import pytest
import torch

from util import orc, rel_err, to_torch, REL_TOL

FLAG, STATE, ERROR, DATA = 0, 64, 128, 4096
EXCHANGE_LAYERS = [(4, 1024, 1024, 2, 0.01, 4), (3, 512, 256, 1, 0.0, 0), (4, 4096, 4096, 3, 0.0045, 10),
                   (4, 256, 32, 1, 0.02, 4),  # narrower than one strip: one ragged strip
                   (3, 1024, 512, 3, 0.01, 40)]  # more than 32 dense rows: the general dense-row branch
EXCHANGE_IDS = ["w4-2x1024", "w3-1x256", "w4-qkv", "w4-1x32", "w3-3x512-t40"]


def exchange_layer(bits, K, w, members, sp, topx):
    """The oracle layer of `members` stacked shards of width w (EXCHANGE_LAYERS), with a bias."""
    N = members * w
    L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=K + N, nonzero_full_rows=True, bias=True)
    if topx and sp == 0:
        L["full_rows"] = L["full_row_indices"] = None
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("bits,K,w,members,sp,topx", EXCHANGE_LAYERS, ids=EXCHANGE_IDS)
def test_exchange_world1_matches_oracle_and_counts_arrivals(bits, K, w, members, sp, topx):
    from squeezellm_b200 import quant as Q
    qc = Q.quant_cuda
    N = members * w
    L = exchange_layer(bits, K, w, members, sp, topx)
    T = to_torch(L)
    x = orc.make_vec(K, seed=6)
    xt = torch.from_numpy(x).cuda().reshape(-1).half()
    arena = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    base = torch.tensor([arena.data_ptr()], dtype=torch.int64, device="cuda")
    want = orc.forward_f64(L, x, mul_init=L["bias"][None, :]).reshape(members, w)

    def counter(off):
        return int(arena[off:off + 8].view(torch.int64).item())

    for call in (1, 2):  # counters only grow: the second call must wait for 2x the arrivals and still deliver
        arena[DATA:DATA + 2 * N].zero_()
        qc.lutgemv_fused_exchange(xt, T["qweight"], T["lookup_table"], bits, T["bias"], T.get("rows"), T.get("cols"), T.get("vals"),
                                  T.get("full_rows"), T.get("full_row_indices"), base.data_ptr(), DATA, FLAG, STATE, ERROR,
                                  1, 0, members, w)
        torch.cuda.synchronize()
        got = arena[DATA:DATA + 2 * N].view(torch.float16).view(members, w).float().cpu().numpy()
        assert rel_err(got, want) < REL_TOL
        assert int(arena[ERROR:ERROR + 4].view(torch.int32).item()) == 0
        # every CTA that owns a strip (at most one per SM, at most one per strip) announces itself once per call
        nown = counter(FLAG) // call
        assert 1 <= nown <= min(qc.sm_count(), (N + 63) // 64) and counter(FLAG) == call * nown and counter(STATE) == call * nown
    # same numbers as the plain fused call
    y = qc.lutgemv_fused(xt, T["qweight"], T["lookup_table"], bits, T["bias"], T.get("rows"), T.get("cols"), T.get("vals"),
                         T.get("full_rows"), T.get("full_row_indices"))
    assert rel_err(got.reshape(-1), y.float().cpu().numpy()) < REL_TOL


@pytest.mark.gpu
def test_exchange_rejects_bad_descriptors():
    from squeezellm_b200 import quant as Q
    qc = Q.quant_cuda
    L = orc.make_layer(4, 256, 128, seed=3)
    T = to_torch(L)
    xt = torch.zeros(256, device="cuda", dtype=torch.float16)
    arena = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    base = torch.tensor([arena.data_ptr()], dtype=torch.int64, device="cuda")
    args = (xt, T["qweight"], T["lookup_table"], 4, None, None, None, None, None, None, base.data_ptr())
    with pytest.raises(RuntimeError):   # rank outside the world
        qc.lutgemv_fused_exchange(*args, DATA, FLAG, STATE, ERROR, 1, 1, 1, 128)
    with pytest.raises(RuntimeError):   # members does not divide the stacked width
        qc.lutgemv_fused_exchange(*args, DATA, FLAG, STATE, ERROR, 1, 0, 3, 128)
    with pytest.raises(RuntimeError):   # misaligned destination
        qc.lutgemv_fused_exchange(*args, DATA + 2, FLAG, STATE, ERROR, 1, 0, 1, 128)
    with pytest.raises(RuntimeError):   # full width smaller than world * shard width
        qc.lutgemv_fused_exchange(*args, DATA, FLAG, STATE, ERROR, 1, 0, 1, 64)
