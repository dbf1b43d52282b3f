"""quant_cuda.attn_decode_batch (csrc/attn_decode.cuh, the batched kernel) on the GPU: B sequences in one launch, each at its own
position in its own cache block, checked row by row with the single-row tests' checks (test_attn_decode_gpu.check_call):
  * each row's output within the fp64 bound of `out_bound`, its stored k within one rounding, its stored v bit-exact, every other
    slot of its cache block bitwise unchanged, with the slots past its pos NaN-filled (so a read of one would show in the output);
  * idle rows (pos -1 and pos = capacity) between active ones leave their out row and their whole cache block bitwise untouched;
  * row b bitwise equal to quant_cuda.attn_decode on row b's slices wherever the two split counts agree;
  * repeated runs bitwise equal; a CUDA graph that advances the active rows' positions on the device bitwise equal to eager calls.
Shapes: (n_heads, n_kv) in test_attn_decode_gpu.HEADS, head_dim 64 and 128, fp16 and bf16; B in {2, 5, 8, 63} for the layouts
(32, 32), (32, 8), (8, 2) and (4, 4), and B in {5, 63} for the others (g = 2, 3, 5, 6, 7, 8, 12, 16 and 71), which bounds the module's
time (on 132 SMs, B = 5 splits every one of them over 2 to 8 CTAs and B = 63 over one); the rows take different positions from
{0, 1, 63, 64, 65, 64S - 1, 64S, capacity - 1} (S: the batch's split count)."""
import pytest
import torch

from test_attn_decode_gpu import DTYPES, HEADS, Case, check_call

pytestmark = pytest.mark.gpu

CAP = 1100  # not a multiple of 64: the last block of a full cache is partial
BATCHES = [2, 5, 8, 63]
# (nh, nkv, d, dtype, B): every B for the first four layouts, B = 5 and 63 for the others
ROWS_GRID = [(nh, nkv, d, dt, B) for i, (nh, nkv) in enumerate(HEADS) for d in (64, 128) for dt in DTYPES
             for B in (BATCHES if i < 4 else [5, 63])]


def _quant_cuda():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


class BatchCase:
    """B single-row Cases (each with its own NaN-filled cache past its pos) stacked into the batched layouts."""

    def __init__(self, nh, nkv, d, dt, positions, seed=0, cap=CAP):
        self.rows = [Case(nh, nkv, d, dt, p, seed=seed + 101 * b, cap=cap) for b, p in enumerate(positions)]
        self.nh, self.nkv, self.d, self.dt, self.cap = nh, nkv, d, dt, cap
        self.scale = self.rows[0].scale
        self.cos, self.sin = self.rows[0].cos, self.rows[0].sin
        self.qkv = torch.stack([r.qkv for r in self.rows])
        self.kc = torch.stack([r.kc for r in self.rows])
        self.vc = torch.stack([r.vc for r in self.rows])
        self.pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
        self.out = torch.stack([r.out for r in self.rows])

    def run(self):
        _quant_cuda().attn_decode_batch(self.qkv, self.pos, self.cos, self.sin, self.kc, self.vc, self.out, self.nh, self.nkv, self.scale)

    def scatter(self):
        """Copy each row's results back into its Case (its out and its cache, inside the buffer with the guard band)."""
        for b, r in enumerate(self.rows):
            r.kc.copy_(self.kc[b])
            r.vc.copy_(self.vc[b])
            r.out.copy_(self.out[b])


def ragged(nh, nkv, B, shift=0):
    S = _quant_cuda().attn_decode_batch_splits(nh, nkv, B)
    vals = sorted({0, 1, 63, 64, 65, 64 * S - 1, 64 * S, CAP - 1})
    return [vals[(b + shift) % len(vals)] for b in range(B)]


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.mark.parametrize("nh,nkv,d,dtype,B", ROWS_GRID, ids=[f"{a}x{b}-{d}-{dt}-{B}" for a, b, d, dt, B in ROWS_GRID])
def test_rows_against_fp64(record, nh, nkv, d, dtype, B):
    bc = BatchCase(nh, nkv, d, DTYPES[dtype], ragged(nh, nkv, B, shift=B), seed=B)
    before = [(r.kbuf.clone(), r.vbuf.clone()) for r in bc.rows]
    bc.run()
    bc.scatter()
    worst = 0.0
    for r, (bk, bv) in zip(bc.rows, before):
        ratio = check_call(r, bk, bv)
        assert ratio <= 1.0, (r.pos, ratio)
        worst = max(worst, ratio)
    record("bound_ratio", worst)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_idle_rows_write_nothing(dtype):
    nh, nkv, d = 8, 2, 128
    positions = [-1, 10, CAP, 700, -1, CAP - 1]
    bc = BatchCase(nh, nkv, d, DTYPES[dtype], positions, seed=3)
    before = [(r.kbuf.clone(), r.vbuf.clone()) for r in bc.rows]
    kc0, vc0, out0 = bc.kc.clone(), bc.vc.clone(), bc.out.clone()
    bc.run()
    torch.cuda.synchronize()
    for b, p in enumerate(positions):
        if 0 <= p < CAP:
            continue
        assert torch.equal(bc.out[b].view(torch.int16), out0[b].view(torch.int16)), f"idle row {b} wrote its out row"
        assert torch.equal(bc.kc[b].view(torch.int16), kc0[b].view(torch.int16)), f"idle row {b} wrote its k cache"
        assert torch.equal(bc.vc[b].view(torch.int16), vc0[b].view(torch.int16)), f"idle row {b} wrote its v cache"
    bc.scatter()
    for r, (bk, bv), p in zip(bc.rows, before, positions):
        if 0 <= p < CAP:
            assert check_call(r, bk, bv) <= 1.0


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,d,B", [(8, 2, 64, 2), (8, 2, 128, 5), (32, 8, 128, 2), (4, 4, 64, 4)])
def test_rows_equal_the_single_row_kernel(nh, nkv, d, dtype, B):
    qc = _quant_cuda()
    assert qc.attn_decode_batch_splits(nh, nkv, B) == qc.attn_decode_splits(nh, nkv), "pick shapes whose split counts agree"
    assert qc.attn_decode_batch_splits(nh, nkv, 1) == qc.attn_decode_splits(nh, nkv)
    positions = ragged(nh, nkv, B)
    bc = BatchCase(nh, nkv, d, DTYPES[dtype], positions, seed=7)
    single = BatchCase(nh, nkv, d, DTYPES[dtype], positions, seed=7).rows
    bc.run()
    for b, r in enumerate(single):
        r.run()
        assert torch.equal(bc.out[b].view(torch.int16), r.out.view(torch.int16)), b
        assert torch.equal(bc.kc[b].view(torch.int16), r.kc.view(torch.int16)), b
        assert torch.equal(bc.vc[b].view(torch.int16), r.vc.view(torch.int16)), b


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_bitwise_reproducible(dtype):
    bc = BatchCase(32, 8, 128, DTYPES[dtype], [3001 % CAP, 17, 900, 64, 1], seed=5)
    outs = []
    for _ in range(5):
        bc.run()
        outs.append(bc.out.clone())
    for o in outs[1:]:
        assert torch.equal(o.view(torch.int16), outs[0].view(torch.int16))


@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64)])
def test_graph_replay_advances_pos_on_device(nh, nkv, d):
    """N steps of one captured call + pos[b] += 1 for the active rows, each with new qkv, bitwise equal to N eager calls."""
    N = 12
    positions = [250, -1, 3, 700, CAP - N]
    dt = torch.float16
    g = torch.Generator(device="cuda").manual_seed(9)
    qkvs = torch.randn(N, len(positions), (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
    eager = BatchCase(nh, nkv, d, dt, positions, seed=1)
    graphed = BatchCase(nh, nkv, d, dt, positions, seed=1)
    outs_e, outs_g = [], []
    for i in range(N):
        eager.qkv.copy_(qkvs[i])
        eager.pos.copy_(torch.tensor([p + i if p >= 0 else p for p in positions], dtype=torch.int32))
        eager.run()
        outs_e.append(eager.out.clone())
    qc = _quant_cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        qc.attn_decode_batch(graphed.qkv, graphed.pos, graphed.cos, graphed.sin, graphed.kc, graphed.vc, graphed.out, nh, nkv,
                             graphed.scale)
        graphed.pos.add_((graphed.pos >= 0).to(torch.int32))
    for i in range(N):
        graphed.qkv.copy_(qkvs[i])
        graph.replay()
        outs_g.append(graphed.out.clone())
    torch.cuda.synchronize()
    assert graphed.pos.tolist() == [p + N if p >= 0 else p for p in positions]
    for a, b in zip(outs_e, outs_g):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(eager.kc.view(torch.int16), graphed.kc.view(torch.int16))
    assert torch.equal(eager.vc.view(torch.int16), graphed.vc.view(torch.int16))


def test_module_rejects_mismatched_cuda_tensors():
    bc = BatchCase(8, 2, 64, torch.float16, [5, 9])
    with pytest.raises(RuntimeError, match="k_cache, v_cache and out must have qkv's dtype"):
        _quant_cuda().attn_decode_batch(bc.qkv, bc.pos, bc.cos, bc.sin, bc.kc, bc.vc, bc.out.to(torch.bfloat16), 8, 2, 0.125)
    with pytest.raises(RuntimeError, match="pos must be a CUDA tensor"):
        _quant_cuda().attn_decode_batch(bc.qkv, bc.pos.cpu(), bc.cos, bc.sin, bc.kc, bc.vc, bc.out, 8, 2, 0.125)
