"""quant_cuda.attn_extend_batch and attn_extend_batch_paged (csrc/attn_extend.cuh) on the GPU against the single-sequence kernels.

The contract is bitwise: segment i's out rows and the k / v it stores are those of attn_extend (attn_extend_paged) run for its slot alone
with (start_i, T_i).  Per call, the segments go to permuted slots of a cache with more slots than segments; every slot holds random
data before its segment's start and NaN from it on, and slots no segment names hold random data throughout.  Checked:
  * out rows and the whole cache (or page pool) bitwise equal to the single kernels run one segment after another on a copy, so no
    slot or position outside the segments' chunks changes, and the NaN past start + T stays NaN;
  * reversing the segment order gives the same bits per segment; a rerun and a CUDA-graph replay give the same bits;
  * paged: randomly permuted pages, two segments whose prefixes share read-only pages, and a segment with a table entry outside the
    pool, which writes nothing while the others still match.
Segment mixes: one segment; three of one token; (0, 17), (100, 300), (4000, 8), (63, 2), (0, 65); (0, 2048), (CAP - 5, 5); 16 segments
of 16 tokens whose splits (attn_extend_splits) take at least three values, so that the call makes at least three attention launches."""
import math

import pytest
import torch

from test_attn_decode_gpu import HEADS
from test_attn_extend_gpu import CAP, rope_tables

pytestmark = pytest.mark.gpu

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
STARTS16 = [0, 64, 150, 4000, 20, 100, 300, 1000, 2000, 3000, 500, 700, 40, 250, 3500, 4100]
MIXES = {
    "one": [(100, 300)],
    "three_T1": [(0, 1), (63, 1), (4000, 1)],
    "five": [(0, 17), (100, 300), (4000, 8), (63, 2), (0, 65)],
    "long": [(0, 2048), (CAP - 5, 5)],
    "sixteen": [(s, 16) for s in STARTS16],
}
PAGED_HEADS = [(32, 8), (8, 2), (28, 4), (71, 1)]
PAGE = 64


def _qc():
    from squeezellm_b200.quant import quant_cuda
    return quant_cuda


def bits(t):
    return t.view(torch.int16)


class Setup:
    """One call's inputs: segments (slot, start, T) on permuted slots, qkv [sum T, ...], the caches (contiguous [n_slots, n_kv, CAP, d],
    or a pool of pages and a block table [n_slots, width]) and an out buffer filled with 7."""

    def __init__(self, nh, nkv, d, dt, mix, paged, seed=0, share=False):
        g = torch.Generator(device="cuda").manual_seed(seed)
        cg = torch.Generator().manual_seed(seed)
        self.nh, self.nkv, self.d, self.dt, self.paged = nh, nkv, d, dt, paged
        self.scale = 1.0 / math.sqrt(d)
        n = len(mix)
        self.n_slots = n + 2
        slots = torch.randperm(self.n_slots, generator=cg)[:n].tolist()
        self.segs = [(slots[i], s, T) for i, (s, T) in enumerate(mix)]
        rows = sum(T for _, T in mix)
        self.qkv = torch.randn(rows, (nh + 2 * nkv) * d, generator=g, device="cuda").to(dt)
        self.cos, self.sin = rope_tables(CAP, d)
        if not paged:
            self.k = torch.randn(self.n_slots, nkv, CAP, d, generator=g, device="cuda").to(dt)
            self.v = torch.randn(self.n_slots, nkv, CAP, d, generator=g, device="cuda").to(dt)
            for slot, s, _ in self.segs:
                self.k[slot, :, s:] = float("nan")
                self.v[slot, :, s:] = float("nan")
        else:
            width = -(-CAP // PAGE)
            blocks = {slot: -(-(s + T) // PAGE) for slot, s, T in self.segs}
            n_pages = sum(blocks.values()) + 3
            perm = torch.randperm(n_pages, generator=cg).tolist()
            self.table = torch.full((self.n_slots, width), -1, dtype=torch.int32)
            for slot, nb in blocks.items():
                for j in range(nb):
                    self.table[slot, j] = perm.pop()
            self.shared = []
            if share:  # the first two segments with a full block before both starts share those pages (read only)
                (a, sa, _), (b, sb, _) = [x for x in self.segs if x[1] >= PAGE][:2]
                for j in range(min(sa, sb) // PAGE):
                    self.table[b, j] = self.table[a, j]
                    self.shared.append(int(self.table[a, j]))
            self.k = torch.randn(n_pages, nkv, PAGE, d, generator=g, device="cuda").to(dt)
            self.v = torch.randn(n_pages, nkv, PAGE, d, generator=g, device="cuda").to(dt)
            for slot, s, T in self.segs:
                for p in range(s, blocks[slot] * PAGE):
                    pg = int(self.table[slot, p // PAGE])
                    self.k[pg, :, p % PAGE] = float("nan")
                    self.v[pg, :, p % PAGE] = float("nan")
            self.table = self.table.cuda()
        self.k0, self.v0 = self.k.clone(), self.v.clone()

    def rows(self, i):
        r0 = sum(T for _, _, T in self.segs[:i])
        return slice(r0, r0 + self.segs[i][2])

    def fresh(self):
        """Copies of the caches as they were, and an out buffer of 7s."""
        return self.k0.clone(), self.v0.clone(), torch.full((self.qkv.shape[0], self.nh * self.d), 7.0, dtype=self.dt, device="cuda")

    def batch(self, k, v, out, order=None, table=None):
        """The batch call on (k, v, out) with the segments in `order` (default: as given); out rows follow that order."""
        order = list(range(len(self.segs))) if order is None else order
        qkv = torch.cat([self.qkv[self.rows(i)] for i in order])
        o = torch.cat([out[self.rows(i)] for i in order])
        slots, starts, ts = ([self.segs[i][j] for i in order] for j in range(3))
        if self.paged:
            _qc().attn_extend_batch_paged(qkv, slots, starts, ts, self.cos, self.sin, k, v, self.table if table is None else table, o,
                                          self.nh, self.nkv, self.scale)
        else:
            _qc().attn_extend_batch(qkv, slots, starts, ts, self.cos, self.sin, k, v, o, self.nh, self.nkv, self.scale)
        r = 0
        for i in order:  # back to the given order
            T = self.segs[i][2]
            out[self.rows(i)] = o[r:r + T]
            r += T

    def single(self, k, v, out, skip=()):
        """The single-sequence kernel for each segment, one after another."""
        for i, (slot, s, T) in enumerate(self.segs):
            if i in skip:
                continue
            rows = self.rows(i)
            if self.paged:
                _qc().attn_extend_paged(self.qkv[rows], s, self.cos, self.sin, k, v, self.table[slot], out[rows], self.nh, self.nkv,
                                        self.scale)
            else:
                _qc().attn_extend(self.qkv[rows], s, self.cos, self.sin, k[slot], v[slot], out[rows], self.nh, self.nkv, self.scale)

    def nan_past_chunks(self, k):
        """Every position from start + T on of each segment's slot (up to its last block, paged) is still NaN."""
        for slot, s, T in self.segs:
            if not self.paged:
                assert torch.isnan(k[slot, :, s + T:].float()).all()
            else:
                for p in range(s + T, -(-(s + T) // PAGE) * PAGE):
                    assert torch.isnan(k[int(self.table[slot, p // PAGE]), :, p % PAGE].float()).all()


def check_against_single(st):
    k, v, out = st.fresh()
    st.batch(k, v, out)
    kr, vr, outr = st.fresh()
    st.single(kr, vr, outr)
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(outr)), "out rows differ from the single-sequence kernel's"
    assert torch.equal(bits(k), bits(kr)) and torch.equal(bits(v), bits(vr)), "the caches differ from the single kernel's"
    st.nan_past_chunks(k)
    return k, v, out


def _splits(st):
    return [_qc().attn_extend_splits(st.nh, st.nkv, T, s) for _, s, T in st.segs]


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nh,nkv", HEADS, ids=[f"{a}x{b}" for a, b in HEADS])
def test_contiguous_equals_single(nh, nkv, d, dtype):
    for m, (name, mix) in enumerate(MIXES.items()):
        st = Setup(nh, nkv, d, DTYPES[dtype], mix, paged=False, seed=m)
        if name == "sixteen":
            assert len(set(_splits(st))) >= 3, _splits(st)
        k, v, out = check_against_single(st)
        if name in ("five", "sixteen"):
            rk, rv, rout = st.fresh()
            st.batch(rk, rv, rout, order=list(range(len(mix)))[::-1])
            assert torch.equal(bits(rout), bits(out)) and torch.equal(bits(rk), bits(k)) and torch.equal(bits(rv), bits(v)), "order"


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nh,nkv", PAGED_HEADS, ids=[f"{a}x{b}" for a, b in PAGED_HEADS])
def test_paged_equals_single(nh, nkv, d, dtype):
    for m, (name, mix) in enumerate(MIXES.items()):
        st = Setup(nh, nkv, d, DTYPES[dtype], mix, paged=True, seed=m, share=name in ("five", "sixteen"))
        if name == "sixteen":
            assert len(set(_splits(st))) >= 3, _splits(st)
        k, v, out = check_against_single(st)
        if st.shared:
            assert torch.equal(bits(k[st.shared]), bits(st.k0[st.shared])), "a shared prefix page was written"
        if name in ("five", "sixteen"):
            rk, rv, rout = st.fresh()
            st.batch(rk, rv, rout, order=list(range(len(mix)))[::-1])
            assert torch.equal(bits(rout), bits(out)) and torch.equal(bits(rk), bits(k)) and torch.equal(bits(rv), bits(v)), "order"


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("d", [64, 128])
def test_paged_bad_table_entry_writes_nothing(d, dtype):
    """Segment 1's table names a page outside the pool among its blocks: its out rows and its pages stay as they were, the other
    segments match the single kernel."""
    st = Setup(32, 8, d, DTYPES[dtype], MIXES["five"], paged=True, seed=7)
    slot, s, T = st.segs[1]
    table = st.table.clone()
    table[slot, (s + T - 1) // PAGE] = st.k.shape[0]
    k, v, out = st.fresh()
    st.batch(k, v, out, table=table)
    kr, vr, outr = st.fresh()
    st.single(kr, vr, outr, skip=(1,))
    torch.cuda.synchronize()
    assert (out[st.rows(1)] == 7.0).all(), "the segment with a bad table entry wrote its out rows"
    assert torch.equal(bits(out), bits(outr)) and torch.equal(bits(k), bits(kr)) and torch.equal(bits(v), bits(vr))


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_rerun_and_graph_replay(paged, dtype):
    st = Setup(32, 8, 128, DTYPES[dtype], MIXES["sixteen"], paged=paged, seed=3)
    k, v, out = check_against_single(st)
    k2, v2, out2 = st.fresh()
    st.batch(k2, v2, out2)
    assert torch.equal(bits(out2), bits(out)) and torch.equal(bits(k2), bits(k)) and torch.equal(bits(v2), bits(v))
    gk, gv, gout = st.fresh()
    qkv = torch.cat([st.qkv[st.rows(i)] for i in range(len(st.segs))])
    o = torch.empty_like(gout)
    slots, starts, ts = ([x[j] for x in st.segs] for j in range(3))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        if paged:
            _qc().attn_extend_batch_paged(qkv, slots, starts, ts, st.cos, st.sin, gk, gv, st.table, o, st.nh, st.nkv, st.scale)
        else:
            _qc().attn_extend_batch(qkv, slots, starts, ts, st.cos, st.sin, gk, gv, o, st.nh, st.nkv, st.scale)
    gk.copy_(st.k0)
    gv.copy_(st.v0)
    o.fill_(7.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(o), bits(out)) and torch.equal(bits(gk), bits(k)) and torch.equal(bits(gv), bits(v))
