"""GPU parity of the sequence kernel (csrc/lutgemv_seq.cuh, runtime.DecodeSequence): a chain of dependent matvecs run as ONE
persistent launch must give what the same layers give when called one by one (squeezellm/llama.py:226-234 drives
QuantLinearLUT.forward layer by layer), and what the fp64 oracle gives for the same chain with fp16 hand-overs."""
import numpy as np
import pytest
import torch

from util import OUT_ROUNDING, REL_TOL, abs_sum, bound_ratio, late_owned_strips, orc, rel_err

pytestmark = pytest.mark.gpu

R_F16, ETA_F16 = OUT_ROUNDING["float16"]


def _module(L, bits, K, N, topX):
    from squeezellm_b200.quant import QuantLinearLUT
    has_csr = L.get("rows") is not None
    dense_only = not has_csr and L.get("full_rows") is not None

    class DenseRowsOnly(QuantLinearLUT):  # dense rows without CSR outliers (the C ABI takes them; a checkpoint never has them)
        def _sparse_args(self):
            return None, None, None, self.full_rows, self.full_row_indices

    m = (DenseRowsOnly if dense_only else QuantLinearLUT)(bits, K, N, False, include_sparse=has_csr or dense_only,
                                                           numvals=len(L["vals"]) if has_csr else 0, topX=topX if has_csr or dense_only else 0)
    sd = m.state_dict()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in L.items() if isinstance(v, np.ndarray) and k in sd}, strict=False)
    return m.cuda()


def _chain(bits, dims, sparsity, topX, seed):
    """dims: [(K, N, x_offset into the previous output)]; returns oracle layers + modules.  topX > 0 with sparsity 0: dense rows
    without CSR outliers."""
    from squeezellm_b200.quant import quant_cuda as qc
    layers, mods = [], []
    for i, (K, N, _) in enumerate(dims):
        L = orc.make_layer(bits, K, N, sparsity=sparsity, topX=topX, seed=seed + 17 * i, nonzero_full_rows=True)
        rng = np.random.default_rng(seed + 17 * i + 1)
        late = late_owned_strips(bits, K, N, qc.sm_count()) if topX > 32 else []
        if topX > 32 and len(late):  # CTAs that own more than 8 strips: rows in their 9th and later strips, duplicates, channel 0
            f = rng.choice(late, size=topX) * 64 + rng.integers(0, 64, size=topX)
            f[1], f[2], f[3] = f[0], 0, N - 1
            L["full_row_indices"] = f.astype(np.int32)
        elif topX > 32 and i % 2 == 1:  # every row in one strip, with duplicates
            L["full_row_indices"] = (N // 128 * 64 + rng.integers(0, 64, size=topX)).astype(np.int32)
        elif topX >= 3 and i % 2 == 0:  # dense rows that feed the same output channel (their parts travel combined), one of them channel 0
            L["full_row_indices"][1] = L["full_row_indices"][0]
            L["full_row_indices"][2] = 0
        # keep activations O(1) through the chain
        L["lookup_table"] = (L["lookup_table"] * (50.0 / np.sqrt(K))).astype(np.float32)  # centroids ~ N(0, 1/K): |y| ~ |x|
        layers.append(L)
        mods.append(_module(L, bits, K, N, topX))
    return layers, mods


def _oracle_chain(layers, dims, x, lut_fp16=False):
    outs, prev = [], None
    for L, (K, N, off) in zip(layers, dims):
        xin = x if prev is None else prev[off:off + K]
        LL = dict(L)
        if lut_fp16:
            LL["lookup_table"] = L["lookup_table"].astype(np.float16).astype(np.float32)
        y = orc.forward_f64(LL, xin.astype(np.float32).reshape(1, K)).reshape(N)
        prev = y.astype(np.float16).astype(np.float64)  # the hand-over between two matvecs is fp16, as in the model
        outs.append(prev)
    return outs


CASES = [  # (bits, dims, sparsity, topX)
    (4, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)], 0.0, 0),
    (4, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)], 0.02, 4),
    (3, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)], 0.02, 4),
    (4, [(512, 132, 0), (128, 200, 4), (192, 64, 8), (64, 512, 0), (512, 132, 0)], 0.01, 3),   # ragged strips, one-strip items
    (4, [(4096, 12288, 0), (4096, 4096, 8192), (4096, 22016, 0), (11008, 4096, 0)], 0.0045, 10, 3),  # LLaMA-7B decoder layer, three times over
    (3, [(4096, 12288, 0), (4096, 4096, 8192), (4096, 22016, 0), (11008, 4096, 0)], 0.0045, 10, 2),
    # more than 32 dense rows: the general dense-row branch (duplicates, channel 0, all rows in one strip)
    (4, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)], 0.02, 33),
    (3, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)], 0.02, 128),
    # a 131072-column item (CTAs own ~16 strips; dense rows in their 9th and later), then an item that reads its last 4096 outputs
    (4, [(128, 131072, 0), (4096, 768, 126976), (768, 256, 0)], 0.0, 128),
]
IDS = [f"w{c[0]}-{len(c[1])}items-K{c[1][0][0]}-s{int(c[2] * 1e4)}-t{c[3]}" for c in CASES]


@pytest.mark.parametrize("case", CASES, ids=IDS)
@pytest.mark.parametrize("mode", ["exact", "fp16"])
def test_sequence_matches_layer_by_layer_and_oracle(case, mode):
    from squeezellm_b200.quant import quant_cuda
    from squeezellm_b200.runtime import DecodeSequence
    bits, dims, sp, topX = case[:4]
    layers, mods = _chain(bits, dims, sp, topX, seed=bits * 100 + len(dims))
    rep_n = case[4] if len(case) > 4 else 1  # the same matrices again (the generator is slow for 22016 channels): a longer chain
    dims, layers, mods = dims * rep_n, layers * rep_n, mods * rep_n
    x = orc.make_vec(dims[0][0], seed=5).reshape(-1).astype(np.float16)
    seq = DecodeSequence(dims[0][0], "cuda", lut_mode=mode)
    vecs, prev = [], seq.input
    for m, (K, N, off) in zip(mods, dims):
        prev = seq.matvec(m, prev[off:off + K])
        vecs.append(prev)
    seq.compile(outputs=vecs)
    seq.x.copy_(torch.from_numpy(x).cuda())
    want = _oracle_chain(layers, dims, x.astype(np.float64), lut_fp16=(mode == "fp16"))
    # the same layers one by one through the module path
    quant_cuda.set_lut_mode(mode)
    try:
        ys, cur = [], torch.from_numpy(x).cuda()
        for m, (K, N, off) in zip(mods, dims):
            cur = m(cur[off:off + K].clone() if ys else cur)  # (a fresh allocation: the module path wants a 16-byte aligned x)
            ys.append(cur)
    finally:
        quant_cuda.set_lut_mode("exact")
    x_half = (x.astype(np.float32) * 0.5).astype(np.float16)
    for rep in range(3):  # replays: the tags of the previous token must not be taken for this one's
        if rep == 2:
            seq.x.copy_(torch.from_numpy(x_half).cuda())
        outs = [o.clone() for o in seq.replay()]
        torch.cuda.synchronize()
        assert not seq.error(), "a bounded in-kernel wait of the sequence gave up"
        if rep == 2:
            want = _oracle_chain(layers, dims, x_half.astype(np.float64), lut_fp16=(mode == "fp16"))
        got_all = [o.float().cpu().numpy().astype(np.float64) for o in outs]
        for i, (L, (K, N, off)) in enumerate(zip(layers, dims)):
            # per item, per element: the oracle applied to the fp16 vector this item actually consumed (seq.x, or the exported slice of
            # its predecessor), so that no hand-over rounding blurs the check
            xin = (x if rep < 2 else x_half).astype(np.float64) if i == 0 else got_all[i - 1][off:off + K]
            LL = dict(L)
            if mode == "fp16":
                LL["lookup_table"] = L["lookup_table"].astype(np.float16).astype(np.float32)
            xin = xin.astype(np.float32).reshape(1, K)
            wi = orc.forward_f64(LL, xin).reshape(N)
            assert np.isfinite(got_all[i]).all(), f"rep {rep} item {i}: non-finite output"
            ratio = bound_ratio(got_all[i], wi, abs_sum(LL, xin).reshape(N), wi, R_F16, eta=ETA_F16)
            assert ratio <= 1.0, f"rep {rep} item {i}: bound ratio {ratio:.3f} against the oracle on the item's own input"
        for i, (o, w) in enumerate(zip(outs, want)):
            got = got_all[i]
            # fp16 hand-overs: one fp16 ulp of an input moves later outputs; compare in the max norm at the north_star tolerance,
            # plus the strict per-element metric for the first item (no hand-over before it)
            err = np.abs(got - w).max() / max(np.abs(w).max(), 1e-30)
            assert err < 2 * REL_TOL, f"rep {rep} item {i}: max-norm error {err:.3e} vs the oracle chain"
            if i == 0 and mode == "exact":
                assert rel_err(got, w) < REL_TOL
            if rep < 2:
                ref = ys[i].float().cpu().numpy().astype(np.float64)
                err2 = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)
                assert err2 < 2 * REL_TOL, f"rep {rep} item {i}: {err2:.3e} vs the layer-by-layer module path"


def test_sequence_in_cuda_graph_and_plain_copies():
    """The two launches of a run are capturable; replays keep working (the token counter lives in device memory)."""
    from squeezellm_b200.runtime import DecodeSequence, GraphedDecodeStep
    bits, dims = 4, [(256, 768, 0), (256, 256, 512), (256, 704, 0), (704, 256, 0)]
    layers, mods = _chain(bits, dims, 0.02, 4, seed=77)
    seq = DecodeSequence(256, "cuda", lut_mode="exact")
    prev = seq.input
    for m, (K, N, off) in zip(mods, dims):
        prev = seq.matvec(m, prev[off:off + K])
    seq.compile(outputs=[prev])
    runner = GraphedDecodeStep(lambda x: seq.replay()[0], seq.x, warmup=2, static_input=True)
    for s in (1, 2, 3):
        x = orc.make_vec(256, seed=s).reshape(-1).astype(np.float16)
        y = runner(torch.from_numpy(x)).clone().float().numpy().astype(np.float64)
        w = _oracle_chain(layers, dims, x.astype(np.float64))[-1]
        assert np.abs(y - w).max() / np.abs(w).max() < 2 * REL_TOL
    assert not seq.error()
