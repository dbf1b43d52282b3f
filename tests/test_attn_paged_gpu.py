"""GPU tests of the paged attention kernels (sqllm_attn_decode_paged, sqllm_attn_extend_paged): on tables of randomly permuted pages,
each row's output and the slots it writes are bitwise those of attn_decode_batch / attn_extend on the row's pages gathered into a
contiguous cache.  Unassigned pages hold NaN and must stay NaN and never reach an output; a row whose table names a page outside the
pool writes nothing."""
import pytest
import torch

from test_attn_decode_gpu import DTYPES, HEADS, rope_tables
from test_attn_extend_gpu import CHUNKS

pytestmark = pytest.mark.gpu

PAGE = 64
CAP = 4160            # 65 pages per sequence
WIDTH = CAP // PAGE
# (nh, nkv, d, dtype, B): B = 2 and 5 for every layout, 63 for the first four
DECODE_GRID = [(nh, nkv, d, dt, B) for i, (nh, nkv) in enumerate(HEADS) for d in (64, 128) for dt in DTYPES
               for B in ([2, 5, 63] if i < 4 else [2, 5])]


def _qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def bits(t):
    return t.view(torch.int16) if t.dtype in (torch.float16, torch.bfloat16) else t


def ragged(nh, nkv, B):
    S = _qc().attn_decode_batch_splits(nh, nkv, B)
    vals = sorted({0, 63, 64, 65, 64 * S - 1, 64 * S + 1, CAP - 1})
    return [vals[b % len(vals)] for b in range(B)]


class Paged:
    """B rows at `positions`: contiguous caches [B, nkv, CAP, d] (NaN past each row's pos) and the same content in page pools whose
    pages are dealt in a random order; `spare` extra pages and every unassigned page hold NaN.  share: row 1 reads row 0's first
    `share` pages (both contiguous copies agree there)."""

    def __init__(self, nh, nkv, d, dt, positions, seed=0, spare=3, share=0):
        g = torch.Generator(device="cuda").manual_seed(seed)
        B = len(positions)
        self.nh, self.nkv, self.d, self.dt, self.B = nh, nkv, d, dt, B
        self.scale = d ** -0.5
        self.cos, self.sin = rope_tables(CAP, d)
        self.kc = torch.randn(B, nkv, CAP, d, generator=g, device="cuda").to(dt)
        self.vc = torch.randn(B, nkv, CAP, d, generator=g, device="cuda").to(dt)
        if share:
            self.kc[1, :, :share * PAGE] = self.kc[0, :, :share * PAGE]
            self.vc[1, :, :share * PAGE] = self.vc[0, :, :share * PAGE]
        for b, p in enumerate(positions):
            self.kc[b, :, max(p, 0) + 1:] = float("nan")
            self.vc[b, :, max(p, 0) + 1:] = float("nan")
        blocks = [max(p, 0) // PAGE + 1 for p in positions]
        n = sum(blocks) - (min(share, blocks[1]) if share else 0) + spare
        self.n_pages = n
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).tolist()
        self.table = torch.full((B, WIDTH), -1, dtype=torch.int32)
        k = 0
        for b in range(B):
            for j in range(blocks[b]):
                if b == 1 and j < share:
                    self.table[1, j] = self.table[0, j]
                else:
                    self.table[b, j] = perm[k]
                    k += 1
        self.kp = torch.full((n, nkv, PAGE, d), float("nan"), dtype=dt, device="cuda")
        self.vp = torch.full_like(self.kp, float("nan"))
        for b in range(B):
            for j in range(blocks[b]):
                pg = int(self.table[b, j])
                self.kp[pg] = self.kc[b, :, j * PAGE:(j + 1) * PAGE]
                self.vp[pg] = self.vc[b, :, j * PAGE:(j + 1) * PAGE]
        self.table = self.table.cuda()
        self.qkv = torch.randn(B, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
        self.out_c = torch.full((B, nh * d), 7.0, dtype=dt, device="cuda")
        self.out_p = self.out_c.clone()

    def run_contiguous(self):
        _qc().attn_decode_batch(self.qkv, self.pos, self.cos, self.sin, self.kc, self.vc, self.out_c, self.nh, self.nkv, self.scale)

    def run_paged(self):
        _qc().attn_decode_paged(self.qkv, self.pos, self.cos, self.sin, self.kp, self.vp, self.table, self.out_p, self.nh, self.nkv,
                                self.scale)

    def gathered(self, b, pool):
        """Row b's pages of `pool` laid out as its contiguous cache [nkv, blocks * PAGE, d]."""
        ids = [int(x) for x in self.table[b].tolist() if x >= 0]
        return torch.cat([pool[i] for i in ids], dim=1) if ids else pool[:0]

    def check_rows(self, rows):
        for b in rows:
            assert torch.equal(bits(self.out_p[b]), bits(self.out_c[b])), f"row {b}: output differs"
            assert not torch.isnan(self.out_p[b]).any()
            k, v = self.gathered(b, self.kp), self.gathered(b, self.vp)
            n = k.shape[1]
            assert torch.equal(bits(k), bits(self.kc[b, :, :n])) and torch.equal(bits(v), bits(self.vc[b, :, :n])), f"row {b}: cache"

    def unassigned_nan(self):
        used = set(int(x) for x in self.table.flatten().tolist() if x >= 0)
        for i in range(self.n_pages):
            if i not in used:
                assert torch.isnan(self.kp[i]).all() and torch.isnan(self.vp[i]).all(), f"unassigned page {i} was written"


@pytest.mark.parametrize("nh,nkv,d,dtype,B", DECODE_GRID, ids=[f"{a}x{b}-d{d}-{t}-B{n}" for a, b, d, t, n in DECODE_GRID])
def test_decode_rows_equal_the_batched_kernel(nh, nkv, d, dtype, B):
    c = Paged(nh, nkv, d, DTYPES[dtype], ragged(nh, nkv, B), seed=B + d)
    c.run_contiguous()
    c.run_paged()
    torch.cuda.synchronize()
    c.check_rows(range(B))
    c.unassigned_nan()


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_decode_rows_sharing_pages(dtype):
    c = Paged(32, 8, 128, DTYPES[dtype], [200, 300, 5], share=3)
    c.run_contiguous()
    c.run_paged()
    torch.cuda.synchronize()
    c.check_rows(range(3))
    c.unassigned_nan()


@pytest.mark.parametrize("bad", [-1, "n_pages", "huge"])
def test_decode_out_of_range_entry_idles_the_row(bad):
    c = Paged(32, 8, 128, torch.float16, [700, 130, -1, 64], seed=3)
    c.table[1, 1] = {-1: -1, "n_pages": c.n_pages, "huge": 2 ** 31 - 1}[bad]  # an entry row 1 reads (130 // 64 = 2 blocks)
    kp, vp = c.kp.clone(), c.vp.clone()
    c.run_contiguous()
    c.run_paged()
    torch.cuda.synchronize()
    c.check_rows([0, 3])
    for b in (1, 2):  # the bad row and the idle row: out untouched
        assert (c.out_p[b] == 7.0).all()
    for b in (1, 2):
        for x in c.table[b].tolist():
            if 0 <= x < c.n_pages:
                assert torch.equal(bits(c.kp[x]), bits(kp[x])) and torch.equal(bits(c.vp[x]), bits(vp[x]))


@pytest.mark.parametrize("nh,nkv,d", [(32, 8, 128), (8, 2, 64), (48, 4, 128)])
def test_decode_graph_replay_equals_eager(nh, nkv, d):
    steps = 4
    pos = [60, 127, 0, -1, 3000]
    c = Paged(nh, nkv, d, torch.float16, [p + steps if p >= 0 else p for p in pos], seed=7)  # pages for every step's slot
    c.pos.copy_(torch.tensor(pos, dtype=torch.int32))
    e = Paged(nh, nkv, d, torch.float16, [p + steps if p >= 0 else p for p in pos], seed=7)
    e.pos.copy_(c.pos)
    Paged(nh, nkv, d, torch.float16, [-1], seed=7).run_paged()  # the first launch's set-up outside the capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            c.run_paged()
            c.pos.add_((c.pos >= 0).to(torch.int32))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(steps):
        graph.replay()
        e.run_paged()
        e.pos.add_((e.pos >= 0).to(torch.int32))
        torch.cuda.synchronize()
        assert torch.equal(bits(c.out_p), bits(e.out_p))
    assert torch.equal(bits(c.kp), bits(e.kp)) and torch.equal(c.pos, e.pos)


class PagedChunk:
    """One sequence's chunk of T tokens at `start`: a contiguous cache [nkv, CAP, d] (NaN from start on) and page pools holding its
    blocks 0 .. (start + T - 1) / 64 in a random order, with spare NaN pages."""

    def __init__(self, nh, nkv, d, dt, start, T, seed=0, spare=3):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.nh, self.nkv, self.d, self.start, self.T = nh, nkv, d, start, T
        self.scale = d ** -0.5
        self.cos, self.sin = rope_tables(CAP, d)
        self.kc = torch.randn(nkv, CAP, d, generator=g, device="cuda").to(dt)
        self.vc = torch.randn(nkv, CAP, d, generator=g, device="cuda").to(dt)
        self.kc[:, start:] = float("nan")
        self.vc[:, start:] = float("nan")
        self.blocks = (start + T - 1) // PAGE + 1
        self.n_pages = self.blocks + spare
        perm = torch.randperm(self.n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
        self.row = torch.full((WIDTH,), -1, dtype=torch.int32)
        self.row[:self.blocks] = torch.tensor(perm[:self.blocks], dtype=torch.int32)
        self.kp = torch.full((self.n_pages, nkv, PAGE, d), float("nan"), dtype=dt, device="cuda")
        self.vp = torch.full_like(self.kp, float("nan"))
        for j in range(self.blocks):
            self.kp[perm[j]] = self.kc[:, j * PAGE:(j + 1) * PAGE]
            self.vp[perm[j]] = self.vc[:, j * PAGE:(j + 1) * PAGE]
        self.row = self.row.cuda()
        self.qkv = torch.randn(T, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.out_c = torch.full((T, nh * d), 7.0, dtype=dt, device="cuda")
        self.out_p = self.out_c.clone()

    def run(self):
        qc = _qc()
        qc.attn_extend(self.qkv, self.start, self.cos, self.sin, self.kc, self.vc, self.out_c, self.nh, self.nkv, self.scale)
        qc.attn_extend_paged(self.qkv, self.start, self.cos, self.sin, self.kp, self.vp, self.row, self.out_p, self.nh, self.nkv,
                             self.scale)


EXT_GRID = [(nh, nkv, d, dt, st, T) for i, (nh, nkv) in enumerate(HEADS[:4]) for d in (64, 128) for dt in DTYPES for st, T in CHUNKS]


@pytest.mark.parametrize("nh,nkv,d,dtype,start,T", EXT_GRID, ids=[f"{a}x{b}-d{d}-{t}-{s}+{n}" for a, b, d, t, s, n in EXT_GRID])
def test_extend_equals_the_contiguous_kernel(nh, nkv, d, dtype, start, T):
    c = PagedChunk(nh, nkv, d, DTYPES[dtype], start, T, seed=start + T)
    c.run()
    torch.cuda.synchronize()
    assert torch.equal(bits(c.out_p), bits(c.out_c))
    assert not torch.isnan(c.out_p).any()
    ids = c.row[:c.blocks].tolist()
    n = start + T
    k = torch.cat([c.kp[i] for i in ids], dim=1)[:, :n]
    v = torch.cat([c.vp[i] for i in ids], dim=1)[:, :n]
    assert torch.equal(bits(k), bits(c.kc[:, :n])) and torch.equal(bits(v), bits(c.vc[:, :n]))
    for i in range(c.n_pages):
        if i not in ids:
            assert torch.isnan(c.kp[i]).all() and torch.isnan(c.vp[i]).all(), f"page {i} outside the table was written"


@pytest.mark.parametrize("start,T", [(0, 65), (100, 300), (4000, 8)])
def test_extend_out_of_range_entry_writes_nothing(start, T):
    c = PagedChunk(32, 8, 128, torch.float16, start, T)
    c.row[(start + T - 1) // PAGE] = c.n_pages
    kp, vp = c.kp.clone(), c.vp.clone()
    _qc().attn_extend_paged(c.qkv, start, c.cos, c.sin, c.kp, c.vp, c.row, c.out_p, c.nh, c.nkv, c.scale)
    torch.cuda.synchronize()
    assert (c.out_p == 7.0).all()
    assert torch.equal(bits(c.kp), bits(kp)) and torch.equal(bits(c.vp), bits(vp))
