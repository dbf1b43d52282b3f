"""GPU tests of the quantizer (squeezellm_b200.quantize, quant_cuda.kmeans1d / pack_indices): the exact weighted k-means against
the long-double oracle and against the reference's sklearn fits, its contract (order, labels, determinism, row independence,
streams, graphs), the GPU pack against quant.pack_indices, the outlier masks against the reference's, and quantize_linear /
quantize_model end to end against pack2, the fp64 forward oracle and a checkpoint round trip."""
import os

import numpy as np
import pytest
import torch

import kmeans_oracle as kmo
from util import GOLDEN, OUT_ROUNDING, abs_sum, bound_ratio, orc

pytestmark = pytest.mark.gpu

from squeezellm_b200 import checkpoint as ck  # noqa: E402
from squeezellm_b200.quant import QuantLinearLUT, pack_indices, quant_cuda  # noqa: E402
from squeezellm_b200.quantize import (kmeans_codebook, outlier_threshold, quantize_linear, quantize_model,  # noqa: E402
                                      split_outliers)


def spread(w, s):
    w, s = np.asarray(w, np.float64), np.asarray(s, np.float64)
    s = np.where(s.sum(1, keepdims=True) > 0, s, 1.0)
    mu = (s * w).sum(1, keepdims=True) / s.sum(1, keepdims=True)
    return (s * (w - mu) ** 2).sum(1)


def make_rows(n, seed):
    """Gaussian, Student-t, x1e-6 and x1e3 magnitudes, Fisher weights over 1e-12..1e2, masked zeros, duplicates, values
    +-equal around 0, a constant row and an all-zero row (with all-zero weights)."""
    rng = np.random.default_rng(seed)
    fis = lambda: ((np.exp(rng.normal(0, 1.5, n)) * rng.standard_normal(n)) ** 2)
    W, S = [], []
    W.append(rng.standard_normal(n)); S.append(rng.random(n))
    W.append(rng.standard_t(3, n) * 0.02); S.append(fis())
    W.append(rng.standard_normal(n) * 1e-6); S.append(10.0 ** rng.uniform(-12, 2, n))
    W.append(rng.standard_t(4, n) * 1e3); S.append(fis())
    w = rng.standard_normal(n) * 0.02
    w[rng.random(n) < 0.2] = 0.0
    W.append(w); S.append(fis() * (w != 0))
    W.append(rng.choice(np.array([-0.5, -0.25, 0.0, 0.25, 0.5, 1.0]), n)); S.append(rng.random(n) * (rng.random(n) < 0.8))
    W.append(rng.choice(np.array([-0.01, 0.01]), n) * rng.choice([1, 1, 2], n)); S.append(fis())
    W.append(np.full(n, 0.0375)); S.append(rng.random(n))
    W.append(np.zeros(n)); S.append(np.zeros(n))
    return np.array(W, np.float32), np.array(S, np.float32)


def gpu_kmeans(w, s, k):
    c, lab = quant_cuda.kmeans1d(torch.from_numpy(w).cuda(), torch.from_numpy(s).cuda(), k)
    return c.cpu().numpy(), lab.cpu().numpy()


def midpoint_labels(w, c):
    thr = (np.float32(0.5) * (c[:, :-1] + c[:, 1:])).astype(np.float32)
    return (w[:, :, None] > thr[:, None, :]).sum(-1).astype(np.uint8)


def check_contract(w, c, lab):
    assert np.all(np.isfinite(c))
    assert np.all(np.diff(c, axis=1) >= 0)
    assert np.array_equal(lab, midpoint_labels(w, c))


@pytest.mark.parametrize("n", [32, 96, 4096, 5120, 11008, 13824, 22016, 28672])
@pytest.mark.parametrize("k", [8, 16])
def test_kmeans_against_the_oracle(n, k):
    w, s = make_rows(n, seed=n + k)
    c, lab = gpu_kmeans(w, s, k)
    check_contract(w, c, lab)
    opt, _, _ = kmo.kmeans1d(w, s, k)
    got = kmo.kmeans_objective(w, s, c, lab)
    bound = opt * (1 + 1e-6) + 1e-12 * spread(w, s)
    assert np.all(got <= bound), (got / np.maximum(opt, 1e-300), np.nonzero(got > bound))


def test_kmeans_against_sklearn_golden_rows():
    g = np.load(os.path.join(GOLDEN, "quantize_kmeans.npz"))
    ratios = []
    for n in (4096, 11008):
        w, s = g[f"w_{n}"], g[f"s_{n}"]
        for bits in (3, 4):
            c, lab = gpu_kmeans(w, s, 2 ** bits)
            check_contract(w, c, lab)
            got = kmo.kmeans_objective(w, s, c, lab)
            sse = g[f"sse_{n}_{bits}"]
            assert np.all(got <= sse * (1 + 1e-6) + 1e-12 * spread(w, s)), (n, bits, got / sse)
            ratios += list(got[sse > 0] / sse[sse > 0])
    print(f"GPU / sklearn objective: median {np.median(ratios):.4f}, min {np.min(ratios):.4f}, max {np.max(ratios):.4f}")


def test_kmeans_deterministic_and_row_independent():
    n, k = 28672, 16
    rng = np.random.default_rng(5)
    R = 270  # more rows than one workspace chunk holds at this width (240 rows: 512 MB / 2.24 MB per row)
    w = torch.from_numpy((rng.standard_t(3, (R, n)) * 0.02).astype(np.float32)).cuda()
    s = torch.from_numpy(((np.exp(rng.normal(0, 1.5, (R, n))) * rng.standard_normal((R, n))) ** 2).astype(np.float32)).cuda()
    c1, l1 = quant_cuda.kmeans1d(w, s, k)
    c2, l2 = quant_cuda.kmeans1d(w, s, k)
    assert torch.equal(c1, c2) and torch.equal(l1, l2)
    for r in (0, 1, 239, 240, 269):
        c, lab = quant_cuda.kmeans1d(w[r:r + 1].contiguous(), s[r:r + 1].contiguous(), k)
        assert torch.equal(c[0], c1[r]) and torch.equal(lab[0], l1[r]), r
    c, lab = quant_cuda.kmeans1d(w[200:].contiguous(), s[200:].contiguous(), k)  # other rows, other chunk boundaries
    assert torch.equal(c, c1[200:]) and torch.equal(lab, l1[200:])


def test_kmeans_on_three_streams_and_in_a_graph():
    n, k = 4096, 16
    data = [make_rows(n, seed=40 + i) for i in range(3)]
    ins = [(torch.from_numpy(w).cuda(), torch.from_numpy(s).cuda()) for w, s in data]
    want = [quant_cuda.kmeans1d(w, s, k) for w, s in ins]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(3)]
    outs = [None] * 3
    for i, st in enumerate(streams):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            outs[i] = quant_cuda.kmeans1d(*ins[i], k)
    torch.cuda.synchronize()
    for (c, lab), (wc, wl) in zip(outs, want):
        assert torch.equal(c, wc) and torch.equal(lab, wl)

    w_static, s_static = ins[0][0].clone(), ins[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        quant_cuda.kmeans1d(w_static, s_static, k)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gc, gl = quant_cuda.kmeans1d(w_static, s_static, k)
    for i in (1, 2):
        w_static.copy_(ins[i][0]); s_static.copy_(ins[i][1])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(gc, want[i][0]) and torch.equal(gl, want[i][1])


@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("K", [32, 96, 4096, 11008])
@pytest.mark.parametrize("N", [1, 3, 4096])
def test_pack_indices_bit_exact(bits, K, N):
    rng = np.random.default_rng(K + N + bits)
    labels = rng.integers(0, 2 ** bits, size=(N, K), dtype=np.uint8)
    q = quant_cuda.pack_indices(torch.from_numpy(labels).cuda(), bits)
    assert np.array_equal(q.cpu().numpy(), pack_indices(labels.T, bits))
    assert np.array_equal(quant_cuda.unpack_indices(q, bits).cpu().numpy(), labels.T)


@pytest.mark.parametrize("case", ["thr", "sens", "both", "tied", "tied_both"])
def test_outlier_masks_on_the_gpu(case):
    g = np.load(os.path.join(GOLDEN, "quantize_outliers.npz"))
    thr, sens = g[f"{case}_params"]
    dense, outl = split_outliers(torch.from_numpy(g["w"]).cuda(), torch.from_numpy(g[f"{case}_fisher"]).cuda(),
                                 threshold=None if np.isnan(thr) else float(thr), sensitivity=float(sens))
    assert np.array_equal(dense.cpu().numpy(), g[f"{case}_dense"])
    assert np.array_equal(outl.cpu().numpy(), g[f"{case}_outliers"])


def test_outlier_threshold_on_the_gpu():
    g = np.load(os.path.join(GOLDEN, "quantize_iqr.npz"))
    for i in range(4):
        for r in (1.5, 3.0, 10.0):
            assert outlier_threshold(torch.from_numpy(g[f"a{i}"]).cuda(), r) == float(g[f"thr{i}_{r}"])
    # above torch.quantile's 2^24-element limit.  numpy forms the quantile's index in fp32 here, which at 1.7e7 elements can
    # land on the neighbouring order statistic, so this size is compared to numpy's value within 1e-6, not bit for bit
    big = torch.randn(4096, 4160, device="cuda")
    a = big.cpu().numpy()
    q1, q3 = np.quantile(a, 0.25), np.quantile(a, 0.75)
    want = float(max(abs(q1 - 3.0 * (q3 - q1)), abs(q3 + 3.0 * (q3 - q1))))
    assert abs(outlier_threshold(big, 3.0) - want) <= 1e-6 * want


def _layer_dict(m):
    L = dict(bits=m.bits, infeatures=m.infeatures, outfeatures=m.outfeatures, qweight=m.qweight.cpu().numpy(),
             lookup_table=m.lookup_table.cpu().numpy(), full_rows=None, full_row_indices=None)
    for k in ("rows", "cols", "vals"):
        L[k] = getattr(m, k).cpu().numpy() if m.include_sparse else None
    return L


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("mode", ["dense", "threshold", "both"])
@pytest.mark.parametrize("bits", [3, 4])
def test_quantize_linear_matches_pack2_and_the_oracle(dtype, bias, mode, bits):
    torch.manual_seed(bits)
    K, N = 512, 384
    lin = torch.nn.Linear(K, N, bias=bias).to(dtype).cuda()
    with torch.no_grad():
        lin.weight.copy_((torch.distributions.StudentT(3.0).sample((N, K)) * 0.02).to(dtype))
    fisher = (torch.randn(N, K) * torch.exp(torch.randn(N, K))) ** 2
    thr = None if mode == "dense" else outlier_threshold(lin.weight, 3.0)
    sens = 0.45 if mode == "both" else 0.0
    q = quantize_linear(lin, fisher, bits, threshold=thr, sensitivity=sens)
    assert q.qweight.is_cuda and q.include_sparse == (mode != "dense") and q.topX == 0

    # pack2 on the CPU from the same centroids, labels and outlier matrix
    w = lin.weight.detach().float()
    if mode == "dense":
        dense, outl = w, torch.zeros_like(w)
    else:
        dense, outl = split_outliers(w, fisher.cuda(), thr, sens)
    lut, labels = kmeans_codebook(dense, fisher.cuda() * (dense != 0), bits)
    assert torch.equal(lut, q.lookup_table)
    ref = QuantLinearLUT(bits, K, N, bias, include_sparse=mode != "dense")
    cpu_lin = torch.nn.Linear(K, N, bias=bias).to(dtype)
    if bias:
        cpu_lin.bias.data = lin.bias.detach().cpu()
    lut_np, lab_np = lut.cpu().numpy(), labels.cpu().numpy()
    ref.pack2(cpu_lin, ([[(lut_np[c], lab_np[c])] for c in range(N)], outl.cpu()), include_sparse=mode != "dense")
    for name, t in ref.state_dict().items():
        mine = q.state_dict()[name]
        assert mine.dtype == t.dtype and torch.equal(mine.cpu(), t), name
    if mode != "dense":
        assert q.numvals == ref.numvals > 0

    # forward against the fp64 oracle on those buffers (fp32 x: the bias is an fp32 buffer only for fp32 layers)
    if dtype == torch.float32:
        x = orc.make_vec(K, batch=1, seed=bits)
        L = _layer_dict(q)
        b = lin.bias.detach().cpu().numpy() if bias else None
        want = orc.forward_f64(L, x, mul_init=None if b is None else b[None, :])
        y = q(torch.from_numpy(x).cuda()).cpu().numpy()
        r, eta = OUT_ROUNDING["float32"]
        assert bound_ratio(y, want, abs_sum(L, x, b), r=r, eta=eta) <= 1.0


def test_quantize_model_tiny_llama(tmp_path):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                                   num_key_value_heads=4, vocab_size=97, max_position_embeddings=32)
    torch.manual_seed(0)
    model = transformers.LlamaForCausalLM(cfg).eval().half().cuda()
    names = [n for n in ck.find_linear_layers(model) if n != "lm_head"]
    fisher = {f"{n}.weight": torch.rand_like(m.weight, dtype=torch.float32) ** 4
              for n, m in ck.find_linear_layers(model).items()}
    numvals = quantize_model(model, fisher, 4, outlier_range=3.0, sensitivity=0.45)
    found = ck.find_linear_layers(model, kinds=(torch.nn.Linear, QuantLinearLUT))
    assert all(isinstance(found[n], QuantLinearLUT) for n in names)
    assert isinstance(found["lm_head"], torch.nn.Linear) and not isinstance(found["lm_head"], QuantLinearLUT)
    assert sorted(numvals) == sorted(names) and all(v > 0 for v in numvals.values())
    ids = torch.arange(12, device="cuda").reshape(1, 12) % 97
    with torch.no_grad():
        logits = model(ids).logits.float()
    assert torch.isfinite(logits).all()

    path = str(tmp_path / "model.pt")
    ck.save_checkpoint(model, path, 4)
    torch.manual_seed(0)
    fresh = transformers.LlamaForCausalLM(cfg).eval().half()
    ck.load_checkpoint(fresh, path)
    fresh = fresh.cuda()
    src, dst = model.state_dict(), fresh.state_dict()
    assert sorted(src) == sorted(dst)
    for k, v in src.items():
        assert v.dtype == dst[k].dtype and torch.equal(v.cpu(), dst[k].cpu()), k
    with torch.no_grad():
        assert torch.equal(fresh(ids).logits.float(), logits)


def test_error_messages():
    w = torch.randn(8, 64, device="cuda")
    s = torch.rand(8, 64, device="cuda")
    with pytest.raises(ValueError, match="must be the same"):
        kmeans_codebook(w, s[:, :32], 4)
    with pytest.raises(ValueError, match="finite and >= 0"):
        kmeans_codebook(w, -s, 4)
    with pytest.raises(ValueError, match="finite and >= 0"):
        kmeans_codebook(w, s.masked_fill(s > 0.5, float("nan")), 4)
    with pytest.raises(ValueError, match="multiple of 32"):
        kmeans_codebook(w[:, :48], s[:, :48], 4)
    with pytest.raises(ValueError, match="bits=2 must be 3 or 4"):
        kmeans_codebook(w, s, 2)
    with pytest.raises(ValueError, match="CUDA tensors"):
        kmeans_codebook(w.cpu(), s.cpu(), 4)
    with pytest.raises(ValueError, match="on a CUDA device"):
        quantize_linear(torch.nn.Linear(64, 8), torch.rand(8, 64), 4)
    with pytest.raises(ValueError, match="fisher"):
        quantize_linear(torch.nn.Linear(64, 8).cuda(), torch.rand(8, 32), 4)
    with pytest.raises(KeyError, match="fisher_state has no entry"):
        quantize_model(torch.nn.Sequential(torch.nn.Linear(64, 8).cuda()), {}, 4)
