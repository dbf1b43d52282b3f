// lutgemv_v1.cuh - lutgemv_kernel ("v1"), the round-1 one-vector GEMV: the kernel of the deterministic fused mode
// (sqllm_set_deterministic / SQLLM_DETERMINISTIC=1).  lutgemv2_kernel (lutgemv_v2.cuh) runs every other one-vector GEMV.
// v1 (DESIGN.md has the full story and the measurements):
//   * ONE launch per GEMV.  The [units x strips] iteration space (unit = one packed row for 4-bit,
//     one 3-row / 32-input group for 3-bit; strip = 64 output columns) is flattened strip-major and
//     cut into equal contiguous chunks, one per CTA (stream-K): every SM gets the same number of
//     bytes whatever the shape.  A CTA touches at most MAXSEG strips.
//   * Warp roles: 8 consumer warps + 1 sparse warp, 72 registers, 3 CTAs per SM.
//       - consumers: each lane streams its own 16 bytes per unit row with cp.async into a private ring in shared memory,
//         PF positions ahead (the first PF before the programmatic dependency on the previous kernel resolves - PDL - so
//         the weight traffic of GEMV n+1 overlaps the tail of GEMV n), pulls the word-quad into registers and turns every
//         4-bit index into an LDS address with a single PRMT (the per-strip LUT is staged transposed
//         [value][column-slot] in a 4 KB aligned table so that every lane owns one shared-memory bank: conflict-free
//         gathers); products go into pairs of fp32 accumulators (two fma.rn.f32 per pair).  No tensor cores: this is a gather-bound GEMV.
//       - sparse warp: CSR rows spread evenly over all CTAs, staged with 16-byte cp.async, x gathered in batches,
//         per-row sums in storage order; plus a k-slice of the topX dense rows.
//   * Only the slice of x a CTA needs is staged (fp32, converted from fp16 or bf16 on the way in).
//   * Flush: per-strip partials in the workspace and one ticket per contributor; the last contributor of a strip sums them in a
//     fixed order, adds the bias and stores y.
#pragma once
#include "common.cuh"

namespace {

constexpr int NW = 8;                     // consumer warps per CTA
constexpr int WARP_SPARSE = NW;           // warp index of the CSR / dense-row warp
constexpr int THREADS = (NW + 1) * 32;
constexpr int CTAS_PER_SM = 3;            // resident CTAs per SM the register budget must allow and the plan asks for (shared memory
                                          // admits 3; at 4 the 56-register cap makes the compiler rematerialise table addresses inside
                                          // the loop: measured slower)
constexpr int PF4 = 8;                    // 128-bit loads in flight per lane, 4-bit path
constexpr int PF3 = 3;                    // 3-row groups in flight per lane, 3-bit path
constexpr int MAXSEG = 4;                 // strips a CTA may touch
constexpr int SU = 2 * NW;                // units per pipeline stage (one pair per consumer warp)
constexpr int CSR_CH = 1024;              // CSR elements staged per chunk
constexpr int STAGE = CSR_CH * 16;        // staging buffer: a chunk of CSR cols + vals (8 KB), then the dense-row partials (8 KB)
constexpr int HYB_R = 11;                 // dense rows: k-rows per lane slot requested before the dependency wait

struct Params {
    const uint32_t *qw;
    const float *lut;
    const void *x;      // [K], x_dt
    void *out;          // y, y_dt
    const float *bias;  // may be null
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX;
    int K, N;
    int R;        // units per strip
    int strips;
    int T;        // strips * R
    int chunk;    // units per CTA (even)
    int maxseg;   // strips a CTA of this launch can touch (sizes the LUT tables)
    int x_direct; // 1: x staged at its natural index (CTA covers whole strips), 0: compact, indexed by unit offset
    int xfloats;  // floats in the x staging buffer
    int hc;       // CTAs that take a slice of the dense rows
    int hrows;    // k-rows per such CTA
    int x_dt, y_dt;     // SQLLM_DT_* of x (fp32, fp16 or bf16) and of y (fp32 or 16-bit)
    int maxc;     // max dense contributors per strip
    float *ws_part;   // [strips][maxc+1][64]
    int *ws_cnt;      // [strips]
    float *ws_hyb;    // [hc][topX]
    int has_stage;   // bytes of the shared-memory staging buffer: 0 or STAGE
    int csr_al16;    // cols / vals are 16-byte aligned: stage them with 16-byte cp.async
    int csr_rpc;     // CSR rows (output channels) handled per CTA: rows are spread evenly over all CTAs
    float *ws_csr;   // [N] CSR row sums
    unsigned long long *trace;  // debug timeline (only written when built with -DSQLLM_TRACE and non-null)
};

// ---- per-bit-width constants and the shared memory carve-up (offsets from a 4 KB aligned base) ---
template <int BITS>
struct Cfg {
    static constexpr int L = 1 << BITS;
    static constexpr int TAB = L * STRIP * 4;              // 4096 (w4) / 2048 (w3) bytes per strip table
    static constexpr int ROWS_PER_UNIT = BITS == 4 ? 1 : 3;
    static constexpr int XU = BITS == 4 ? 8 : 32;          // inputs per unit
    // every consumer thread owns PF slots of POS_BYTES (its 4 columns of one unit) in the weight ring, laid out [slot][row-in-unit][thread]
    static constexpr int PF = BITS == 4 ? PF4 : PF3;
    static constexpr int POS_BYTES = ROWS_PER_UNIT * 16;
    static constexpr int RING_BYTES = PF * NW * 32 * POS_BYTES;
    // layout: [tables maxseg*TAB][part maxseg][misc][x][csr stage][weight ring]
    __host__ __device__ static int off_part(int maxseg) { return maxseg * TAB; }
    __host__ __device__ static int off_misc(int maxseg) { return off_part(maxseg) + maxseg * NW * STRIP * 4; }
    // misc: 256 B unused (kept so that the carve-up - and with it occupancy, plan and workspace size - stays as it was measured)
    // + 16 ints (64 B) + dense-row totals float[maxseg + 1][MAX_TOPX_FUSED]
    __host__ __device__ static int off_x(int maxseg) { return off_misc(maxseg) + 256 + 64 + (maxseg + 1) * MAX_TOPX_FUSED * 4; }
    __host__ __device__ static int off_cstage(int maxseg, int xfloats) { return off_x(maxseg) + ((xfloats * 4 + 15) & ~15); }
    __host__ __device__ static int off_stage(int maxseg, int xfloats, int csr) {  // csr: bytes of staging (CSR 8 KB [+ dense-row partials 8 KB])
        return (off_cstage(maxseg, xfloats) + csr + 127) & ~127;
    }
    __host__ __device__ static int total(int maxseg, int xfloats, int csr) { return 4096 + off_stage(maxseg, xfloats, csr) + RING_BYTES; }
};

__device__ __forceinline__ float ldcg_f32(const float *p) { return __ldcg(p); }
// Ticket: one gpu-scope acq_rel atomic.  The release half publishes everything the calling thread wrote - and, by
// cumulativity, what the threads it synchronised with (bar.sync / __syncwarp) wrote before that barrier; the acquire half makes
// the other contributors' published partials visible to whoever draws the last ticket (and, through the next barrier, to its
// whole group).  This replaces the fence / atomic / fence triple (a fence costs about a microsecond on a busy GPU).
__device__ __forceinline__ int ticket_take(int *counter) {
    int old;
    asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;" : "=r"(old) : "l"(counter) : "memory");
    return old;
}

// Walks, in order, the positions (unit pairs) one consumer warp owns: offset 2*warp + SU*p from the CTA's first unit.  Within a
// segment (= strip) consecutive positions are SU units apart, so callers keep running pointers and only `seek` at segment ends.
struct Cursor {
    int seg;   // current segment; == nseg when exhausted
    int left;  // positions left in this segment (including the current one)
    int rr;    // unit index inside the strip of the current position (the lane adds its own 0/1)
    __device__ __forceinline__ void seek(int from_seg, int warp2, int r0, int R, int len, int nseg) {
        for (int sg = from_seg; sg < nseg; ++sg) {
            const int b = sg == 0 ? 0 : sg * R - r0, e = min(len, (sg + 1) * R - r0);   // offsets [b, e) belong to segment sg
            const int pf = b <= warp2 ? 0 : (b - warp2 + SU - 1) / SU;                   // first position with offset >= b
            const int pl = e <= warp2 ? 0 : (e - warp2 + SU - 1) / SU;                   // positions with offset < e
            if (pl > pf) { seg = sg; left = pl - pf; rr = warp2 + SU * pf + r0 - sg * R; return; }
        }
        seg = nseg; left = 0; rr = 0;
    }
};

// =================================================================================================
// 4-bit: one 128-bit word-quad (4 columns x 8 inputs) -> 32 gathers + 16 packed FMAs.
//   E/O hold the even/odd nibbles of a word in separate bytes, already OR-ed with bits 12..15 of the
//   table address; PRMT then builds the complete LDS address: {ls.b3, ls.b2, E.b_n, ls.b0}.
// =================================================================================================
__device__ __forceinline__ void consume4(const uint4 q, const int jsel, const uint32_t lsb, const uint32_t segc,
                                         const uint32_t xaddr, uint64_t (&acc)[4]) {
    const float4 xa = lds_v4(xaddr), xb = lds_v4(xaddr + 16);
    const uint64_t x01 = pack2(xa.x, xa.y), x23 = pack2(xa.z, xa.w), x45 = pack2(xb.x, xb.y), x67 = pack2(xb.z, xb.w);
    // half-warp 1 walks its 4 columns in the order 1,0,3,2 so that the two half-warps never hit the same bank
    const uint32_t w[4] = {jsel ? q.y : q.x, jsel ? q.x : q.y, jsel ? q.w : q.z, jsel ? q.z : q.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const uint32_t E = (w[t] & 0x0F0F0F0Fu) | segc;
        const uint32_t O = ((w[t] >> 4) & 0x0F0F0F0Fu) | segc;
        const uint32_t l = lsb ^ (uint32_t)(t << 6);  // slot of column t (the lane's bank), see set_seg
        const float e0 = lds_f32(__byte_perm(E, l, 0x7604)), o0 = lds_f32(__byte_perm(O, l, 0x7604));
        const float e1 = lds_f32(__byte_perm(E, l, 0x7614)), o1 = lds_f32(__byte_perm(O, l, 0x7614));
        const float e2 = lds_f32(__byte_perm(E, l, 0x7624)), o2 = lds_f32(__byte_perm(O, l, 0x7624));
        const float e3 = lds_f32(__byte_perm(E, l, 0x7634)), o3 = lds_f32(__byte_perm(O, l, 0x7634));
        ffma2(acc[t], pack2(e0, o0), x01);
        ffma2(acc[t], pack2(e1, o1), x23);
        ffma2(acc[t], pack2(e2, o2), x45);
        ffma2(acc[t], pack2(e3, o3), x67);
    }
}

template <int BITS> struct Words;
template <> struct Words<4> { uint4 a; };
template <> struct Words<3> { uint4 a, b, c; };

__device__ __forceinline__ void consume(const Words<4> &g, const int jsel, const uint32_t lsb, const uint32_t segc,
                                        const uint32_t (&)[4], const uint32_t xaddr, uint64_t (&acc)[4]) {
    consume4(g.a, jsel, lsb, segc, xaddr, acc);
}
__device__ __forceinline__ void consume(const Words<3> &g, const int jsel, const uint32_t, const uint32_t,
                                        const uint32_t (&lsv)[4], const uint32_t xaddr, uint64_t (&acc)[4]) {
    uint64_t xp[16];
#pragma unroll
    for (int v = 0; v < 8; ++v) {
        const float4 f = lds_v4(xaddr + 16 * v);
        xp[2 * v] = pack2(f.x, f.y);
        xp[2 * v + 1] = pack2(f.z, f.w);
    }
    const uint32_t a[4] = {jsel ? g.a.y : g.a.x, jsel ? g.a.x : g.a.y, jsel ? g.a.w : g.a.z, jsel ? g.a.z : g.a.w};
    const uint32_t b[4] = {jsel ? g.b.y : g.b.x, jsel ? g.b.x : g.b.y, jsel ? g.b.w : g.b.z, jsel ? g.b.z : g.b.w};
    const uint32_t c[4] = {jsel ? g.c.y : g.c.x, jsel ? g.c.x : g.c.y, jsel ? g.c.w : g.c.z, jsel ? g.c.z : g.c.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) consume3_col(a[t], b[t], c[t], lsv[t], xp, acc[t]);
}

// ---- who contributes to a strip, and the per-column final reduction ----------------------
__device__ __forceinline__ bool strip_has_hybrid(const Params &p, int strip) {
    if (!p.full_rows) return false;
    bool h = false;
    for (int j = 0; j < p.topX; ++j) {
        const int c = __ldg(p.fri + j);
        h |= (c >= 0 && c < p.N && c / STRIP == strip);
    }
    return h;
}
// Contributors that take a ticket on strip `strip`: nd dense CTAs (stream-K), ncsr CTAs whose CSR row
// range touches the strip and - if a dense row lands in it - all hc dense-row contributors.
__device__ __forceinline__ int strip_contributors(const Params &p, int strip, int &nd, bool &hyb) {
    const int first = (int)(((long long)strip * p.R) / p.chunk);
    const int lastc = (int)((((long long)strip + 1) * p.R - 1) / p.chunk);
    nd = lastc - first + 1;
    hyb = strip_has_hybrid(p, strip);
    int ncsr = 0;
    if (p.rows) {
        const int c0 = strip * STRIP, c1 = min(p.N, c0 + STRIP) - 1;
        ncsr = c1 / p.csr_rpc - c0 / p.csr_rpc + 1;
    }
    return nd + ncsr + (hyb ? p.hc : 0);
}
// One warp: fixed-order totals of the dense-row partials ws_hyb[hc][topX] -> tot[topX] (shared memory).  All partials are
// pulled through the staging buffer in one go (one latency), then lanes = (slot, j) sum contributors slot, slot+nsl, ... and the
// slots are folded in fixed order: deterministic.  Callers guarantee every contributor has published (ticket) and fenced.
__device__ __forceinline__ void hybrid_totals(const Params &p, uint32_t stage_u32, const float *stage, float *tot, int lane) {
    const int tp = p.topX, tot_f = p.hc * tp;
    const int n16 = tot_f >> 2;  // ws_hyb and the staging buffer are 16-byte aligned
    for (int e = lane; e < n16; e += 32) cp_async16(stage_u32 + 16 * e, p.ws_hyb + 4 * e);
    for (int e = 4 * n16 + lane; e < tot_f; e += 32) cp_async4(stage_u32 + 4 * e, p.ws_hyb + e);
    cp_async_commit();
    cp_async_wait_all();
    __syncwarp();
    const int nsl = tp <= 16 ? 32 / tp : 1;
    for (int jb = 0; jb < (tp <= 16 ? 1 : tp); jb += 32) {
        const int sl = tp <= 16 ? lane / tp : 0, j = tp <= 16 ? lane - sl * tp : jb + lane;
        float t = 0.f;
        if (sl < nsl && j < tp)
            for (int b = sl; b < p.hc; b += nsl) t += stage[b * tp + j];
        for (int q = 1; q < nsl; ++q) {
            const float v = __shfl_sync(0xffffffffu, t, (j + q * tp) & 31);
            if (sl == 0) t += v;
        }
        if (sl == 0 && j < tp) tot[j] = t;
    }
    __syncwarp();
}
__device__ __forceinline__ void store_y(const Params &p, int col, float v) {
    if (p.y_dt == SQLLM_DT_F16) reinterpret_cast<__half *>(p.out)[col] = __float2half_rn(v);
    else if (p.y_dt == SQLLM_DT_BF16) reinterpret_cast<__nv_bfloat16 *>(p.out)[col] = __float2bfloat16_rn(v);
    else reinterpret_cast<float *>(p.out)[col] = v;
}
__device__ __forceinline__ void final_store(const Params &p, int strip, int c, int nd, const float *hyb_tot) {
    const int col = strip * STRIP + c;
    if (col >= p.N) return;
    const float *base = p.ws_part + (size_t)strip * p.maxc * STRIP + c;
    float tot = 0.f;
    for (int s = 0; s < nd; ++s) tot += ldcg_f32(base + s * STRIP);
    if (p.rows) tot += ldcg_f32(p.ws_csr + col);
    if (hyb_tot)
        for (int j = 0; j < p.topX; ++j)
            if (__ldg(p.fri + j) == col) tot += hyb_tot[j];
    if (p.bias) tot += p.bias[col];
    store_y(p, col, tot);
}
// one warp takes a ticket on `strip` and, if it is the last contributor, reduces and stores the strip's 64 columns
__device__ __forceinline__ void warp_ticket(const Params &p, int strip, int lane, uint32_t hstage_u32, const float *hstage, float *hyb_tot) {
    int nd;
    bool hyb;
    const int expected = strip_contributors(p, strip, nd, hyb);
    int fin = 0;
    __syncwarp();
    if (lane == 0) {
        fin = (ticket_take(p.ws_cnt + strip) == expected - 1);
        if (fin) p.ws_cnt[strip] = 0;
    }
    fin = __shfl_sync(0xffffffffu, fin, 0);
    if (fin) {
        if (hyb) hybrid_totals(p, hstage_u32, hstage, hyb_tot, lane);
        final_store(p, strip, lane, nd, hyb ? hyb_tot : nullptr);
        final_store(p, strip, lane + 32, nd, hyb ? hyb_tot : nullptr);
    }
}

__device__ __forceinline__ float load_x(const Params &p, int k) {  // read-only path: x stays in L1 across the gathers
    if (p.x_dt == SQLLM_DT_F16) return __half2float(__ldg(reinterpret_cast<const __half *>(p.x) + k));
    if (p.x_dt == SQLLM_DT_BF16) return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short *>(p.x) + k) << 16);
    return __ldg(reinterpret_cast<const float *>(p.x) + k);
}

// =================================================================================================
// Sparse warp.  CSR rows (= output channels) are spread evenly over ALL CTAs (csr_rpc consecutive rows each, ~9 for a 4096-wide
// layer) and so are the k-rows of the topX dense rows; each warp therefore has a few hundred elements at most and every
// step is lane-parallel: row pointers live one-per-lane (shuffles / ballots instead of serial scans), cols/vals are staged
// with cp.async, x is gathered in batches of independent loads, per-row sums are taken in storage order (deterministic).
// Everything static (row pointers, cols/vals, dense-row values) is requested BEFORE griddepcontrol.wait.
// Results: ws_csr[row] / dense-row partials + a ticket on the strips touched.
// =================================================================================================
template <int BITS>
__device__ __forceinline__ void sparse_warp(const Params &p, unsigned char *sm, const uint32_t sm_u32, const int lane, float *hyb_tot,
                                            const int nseg, const int s0) {
    using C = Cfg<BITS>;
    const int N = p.N;
    const int cso = C::off_cstage(p.maxseg, p.xfloats);
    int *scols = reinterpret_cast<int *>(sm + cso);
    float *svals = reinterpret_cast<float *>(sm + cso + CSR_CH * 4);
    const uint32_t scols_u32 = sm_u32 + cso, svals_u32 = scols_u32 + CSR_CH * 4;

    // ---------------- phase A: static data ----------------
    float hfr[HYB_R];
    const bool hyb_on = p.full_rows && (int)blockIdx.x < p.hc;
    const bool hyb_multi = hyb_on && p.topX <= 32;  // 32/topX k-rows per warp step: lane = (row slot, column j)
    int kb = 0, ke = 0, nsl = 1, rs = 0, hj = lane;
    if (hyb_on) { kb = blockIdx.x * p.hrows; ke = min(p.K, kb + p.hrows); }
    if (hyb_multi) {
        nsl = 32 / p.topX;
        rs = lane / p.topX;
        hj = lane - rs * p.topX;
#pragma unroll
        for (int i = 0; i < HYB_R; ++i) {
            const int k = kb + rs + nsl * i;
            hfr[i] = (rs < nsl && k < ke) ? __ldg(p.full_rows + (size_t)k * p.topX + hj) : 0.f;
        }
    }
    // CSR: this CTA's rows [ra, rb) (rows are spread evenly over all CTAs), processed in groups of <= 31 rows / <= CSR_CH elements;
    // the first group is pre-staged before the dependency wait
    const int ra = p.rows ? min(N, (int)blockIdx.x * p.csr_rpc) : 0, rb = p.rows ? min(N, ra + p.csr_rpc) : 0;
    int r = ra, rp = 0, m = 0, base = 0, cnt = 0;
    auto group_begin = [&]() {  // row pointers one per lane, group size by ballot, then stage cols/vals
        rp = __ldg(p.rows + min(r + lane, rb));
        base = __shfl_sync(0xffffffffu, rp, 0);
        const bool ok = lane <= min(31, rb - r) && rp - base <= CSR_CH - 4;
        m = __popc(__ballot_sync(0xffffffffu, ok)) - 1;  // rp is non-decreasing: the ok lanes are a prefix that includes lane 0
        const int last = m > 0 ? __shfl_sync(0xffffffffu, rp, m) : base;
        if (p.csr_al16 && m > 0) {
            // 16-byte copies from the element-aligned-down start: up to 3 leading elements of earlier rows ride along (valid data,
            // never summed); the last quad is clipped with the src-size operand, so nothing past `last` is read
            base &= ~3;
            cnt = last - base;
            for (int e = 4 * lane; e < cnt; e += 128) {
                const int nb = min(16, 4 * (cnt - e));
                cp_async16_clip(scols_u32 + 4 * e, p.cols + base + e, nb);
                cp_async16_clip(svals_u32 + 4 * e, p.vals + base + e, nb);
            }
        } else {
            cnt = m > 0 ? last - base : 0;
            for (int e = lane; e < cnt; e += 32) {
                cp_async4(scols_u32 + 4 * e, p.cols + base + e);
                cp_async4(svals_u32 + 4 * e, p.vals + base + e);
            }
        }
        cp_async_commit();
    };
    if (r < rb) group_begin();

    TRACE(13, lane == 0);
    if (lane == 0) pdl_wait();
    __syncwarp();
    TRACE(14, lane == 0);

    // ---------------- phase B: needs x and the workspace ----------------
    // (1) topX dense rows: CTA b < hc takes k-rows [kb, ke)
    if (hyb_on) {
        for (int jb = 0; jb < (hyb_multi ? 1 : p.topX); jb += 32) {
            float a = 0.f;
            int j;
            if (hyb_multi) {
                j = hj;
                float hx[HYB_R];
#pragma unroll
                for (int i = 0; i < HYB_R; ++i) {
                    const int k = kb + rs + nsl * i;
                    hx[i] = (rs < nsl && k < ke) ? load_x(p, k) : 0.f;
                }
#pragma unroll
                for (int i = 0; i < HYB_R; ++i) a += hfr[i] * hx[i];
                for (int k = kb + rs + nsl * HYB_R; rs < nsl && k < ke; k += nsl)
                    a += __ldg(p.full_rows + (size_t)k * p.topX + hj) * load_x(p, k);
                // fold the row slots onto slot 0 in fixed order
                for (int sl = 1; sl < nsl; ++sl) {
                    const float v = __shfl_sync(0xffffffffu, a, (hj + sl * p.topX) & 31);
                    if (rs == 0) a += v;
                }
                if (rs != 0) j = p.topX;  // only slot 0 publishes
            } else {
                j = jb + lane;
                if (j < p.topX) {
                    const float *fr = p.full_rows + (size_t)kb * p.topX + j;
#pragma unroll 8
                    for (int k = kb; k < ke; ++k, fr += p.topX) a += __ldg(fr) * load_x(p, k);
                }
            }
            if (j < p.topX) p.ws_hyb[(size_t)blockIdx.x * p.topX + j] = a;
        }
    }
    TRACE(15, lane == 0);

    // (2) CSR outliers
    while (r < rb) {
        if (m == 0) {  // a single row longer than the staging buffer: straight from global memory, whole warp
            const int e1 = __shfl_sync(0xffffffffu, rp, 1);
            float a = 0.f;
            for (int e = base + lane; e < e1; e += 32) a += __ldg(p.vals + e) * load_x(p, __ldg(p.cols + e));
            a = warp_sum(a);
            if (lane == 0) p.ws_csr[r] = a;
            r += 1;
        } else {
            cp_async_wait_all();
            __syncwarp();
            // products vals[e] * x[cols[e]] in place; gathers go out in batches of 8 independent loads per lane
            for (int e0 = lane; e0 < cnt; e0 += 32 * 8) {
                float xv[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int e = e0 + 32 * j;
                    xv[j] = e < cnt ? load_x(p, scols[e]) : 0.f;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int e = e0 + 32 * j;
                    if (e < cnt) svals[e] *= xv[j];
                }
            }
            __syncwarp();
            // lane i < m owns row r+i: [a0, a1) in the staged arrays
            const int a0 = rp - base, a1 = __shfl_down_sync(0xffffffffu, rp, 1) - base;
            const int n = lane < m ? a1 - a0 : 0;
            if (lane < m && n <= 64) {  // short row: sequential sum in storage order (two interleaved chains)
                float ea = 0.f, eb = 0.f;
                int e = a0;
                for (; e + 1 < a1; e += 2) { ea += svals[e]; eb += svals[e + 1]; }
                if (e < a1) ea += svals[e];
                p.ws_csr[r + lane] = ea + eb;
            }
            unsigned longm = __ballot_sync(0xffffffffu, n > 64);  // long rows: the whole warp on each, fixed xor tree
            while (longm) {
                const int i = __ffs(longm) - 1;
                longm &= longm - 1;
                const int b0 = __shfl_sync(0xffffffffu, a0, i), b1 = __shfl_sync(0xffffffffu, a1, i);
                float a = 0.f;
                for (int e = b0 + lane; e < b1; e += 32) a += svals[e];
                a = warp_sum(a);
                if (lane == 0) p.ws_csr[r + i] = a;
            }
            __syncwarp();
            r += m;
        }
        if (r < rb) group_begin();
    }
    // publish: one fence for everything this warp wrote (CSR row sums, dense-row partials), then one ticket per strip touched
    const uint32_t hstage_u32 = svals_u32 + CSR_CH * 4;
    const float *hstage = svals + CSR_CH;
    __syncwarp();
    if (p.rows && ra < rb)
        for (int strip = ra / STRIP; strip <= (rb - 1) / STRIP; ++strip) warp_ticket(p, strip, lane, hstage_u32, hstage, hyb_tot);
    if (hyb_on) {  // every distinct strip that owns a dense-row output channel
        for (int j0 = 0; j0 < p.topX; ++j0) {
            const int cj0 = __ldg(p.fri + j0);
            if (cj0 < 0 || cj0 >= N) continue;
            const int strip = cj0 / STRIP;
            bool seen = false;
            for (int j = 0; j < j0; ++j) {
                const int cj = __ldg(p.fri + j);
                seen |= (cj >= 0 && cj < N && cj / STRIP == strip);
            }
            if (!seen) warp_ticket(p, strip, lane, hstage_u32, hstage, hyb_tot);
        }
    }
}

// =================================================================================================
// The kernel
// =================================================================================================
template <int BITS>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM) lutgemv_kernel(const Params p) {
    using C = Cfg<BITS>;
    extern __shared__ unsigned char smem_raw[];
    // 4 KB aligned base, computed in the 32-bit shared window and pinned in a register (an opaque mov: otherwise the
    // compiler rematerialises it - S2UR + uniform adds - at every use once registers get tight)
    const uint32_t raw_u32 = smem_u32(smem_raw);
    uint32_t sm_u32 = (raw_u32 + 4095u) & ~4095u;
    asm volatile("mov.u32 %0, %0;" : "+r"(sm_u32));
    unsigned char *sm = smem_raw + (sm_u32 - raw_u32);
    const int maxseg = p.maxseg;
    float *part = reinterpret_cast<float *>(sm + C::off_part(maxseg));
    int *misc = reinterpret_cast<int *>(sm + C::off_misc(maxseg) + 256);
    float *hyb_tot = reinterpret_cast<float *>(sm + C::off_misc(maxseg) + 320);
    float *xs = reinterpret_cast<float *>(sm + C::off_x(maxseg));
    const uint32_t xs_u32 = sm_u32 + C::off_x(maxseg);
    const uint32_t stage_u32 = sm_u32 + C::off_stage(maxseg, p.xfloats, p.has_stage);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i16 = lane & 15, jsel = lane >> 4;  // column group (4 columns) and unit-of-the-pair of this lane
    const int N = p.N, R = p.R;

    // ---- this CTA's chunk of the flattened [strip][unit] space ----
    const int g0 = min((int)blockIdx.x * p.chunk, p.T);
    const int g1 = min(g0 + p.chunk, p.T);
    const int len = g1 - g0;
    const int s0 = g0 / R;
    const int r0 = g0 - s0 * R;
    const int nseg = len > 0 ? (g1 - 1) / R - s0 + 1 : 0;

    TRACE(0, tid == 0);
#ifdef SQLLM_TRACE
    if (p.trace && tid == 0) { unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid)); p.trace[(size_t)blockIdx.x * 32 + 12] = smid + 1; }
#endif
    pdl_launch_dependents();  // the next kernel in the stream may start its own (independent) prologue now
    __syncthreads();
    TRACE(1, tid == 0);

    constexpr int PF = C::PF;
    // ---- weight ring: slot u of this thread lives at ring_u32 + ((u * ROWS_PER_UNIT + row) * NW*32 + tid) * 16 (consecutive threads are
    // contiguous: coalesced fills, conflict-free 128-bit reads).  Exactly one group is committed per position, valid or not,
    // so "at most PF-1 groups pending" always means "the oldest position has landed".  A running global pointer follows the
    // load cursor; it is re-derived only when the cursor enters a new segment.
    const uint32_t ring_u32 = stage_u32 + tid * 16;
    constexpr uint32_t SLOT_STRIDE = C::ROWS_PER_UNIT * NW * 32 * 16;
    const int warp2 = 2 * warp;
    Cursor cl;
    cl.seg = 0; cl.left = 0; cl.rr = 0;
    const uint32_t *lptr = p.qw;
    bool lvalid = false;
    const size_t lstep = (size_t)SU * C::ROWS_PER_UNIT * N;  // words between consecutive positions of a warp
    auto cl_setup = [&]() {
        const int col0 = (s0 + cl.seg) * STRIP + 4 * i16;
        lvalid = cl.seg < nseg && col0 < N;  // lanes past a ragged last strip fetch nothing (their LUT columns are zero)
        if (lvalid) lptr = p.qw + (size_t)((cl.rr + jsel) * C::ROWS_PER_UNIT) * N + col0;
    };
    auto cpa_issue = [&](uint32_t dst) {
        if (lvalid) {
#pragma unroll
            for (int r = 0; r < C::ROWS_PER_UNIT; ++r) cp_async16(dst + r * (NW * 32 * 16), lptr + (size_t)r * N);
        }
        cp_async_commit();
        if (cl.seg < nseg) {
            lptr += lstep;
            if (--cl.left == 0) {
                cl.seek(cl.seg + 1, warp2, r0, R, len, nseg);
                cl_setup();
            }
        }
    };
    auto cpa_fetch = [&](Words<BITS> &w, uint32_t src) {
        w.a = lds_u4(src);
        if constexpr (BITS == 3) {
            w.b = lds_u4(src + NW * 32 * 16);
            w.c = lds_u4(src + 2 * NW * 32 * 16);
        }
    };
    if (warp == WARP_SPARSE) {
        sparse_warp<BITS>(p, sm, sm_u32, lane, hyb_tot + maxseg * MAX_TOPX_FUSED, nseg, s0);
        TRACE(10, lane == 0);
    } else {
        // ---- the first PF weight fetches of every lane go out before anything else.  They do not depend on the previous
        //      kernel, so under PDL the ring of the next GEMV fills while this SM is still busy. ----
        cl.seek(0, warp2, r0, R, len, nseg);
        cl_setup();
#pragma unroll
        for (int u = 0; u < PF; ++u) cpa_issue(ring_u32 + u * SLOT_STRIDE);
        // ---- consumers: stage the LUTs of this CTA's strips, transposed to [value][slot].  One 128-bit load per (column, value
        //      quad); a warp takes 32 columns whose slots fall in 32 different banks, so the four scalar stores are conflict-free.
        //      (4-byte cp.async would cost 16 shared-memory wavefronts per warp instruction - measured.) ----
        constexpr int IPS = STRIP * C::L / 4;                 // (column, quad) items per strip: 256 (w4) / 128 (w3)
        constexpr int LQ = (MAXSEG * IPS + NW * 32 - 1) / (NW * 32);  // items per thread at most
        float4 lq[LQ];
#pragma unroll
        for (int n = 0; n < LQ; ++n) {
            const int it = tid + n * (NW * 32), seg = it / IPS, vw = (it % IPS) >> 5;
            const int c = ((lane >> 1) << 2) | ((vw & 1) << 1) | (lane & 1), q = vw >> 1;
            const int col = (s0 + seg) * STRIP + c;
            lq[n] = (seg < nseg && col < N) ? __ldg(reinterpret_cast<const float4 *>(p.lut + (size_t)col * C::L) + q)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int e = tid; e < maxseg * NW * STRIP; e += NW * 32) part[e] = 0.f;
#pragma unroll
        for (int n = 0; n < LQ; ++n) {
            const int it = tid + n * (NW * 32), seg = it / IPS, vw = (it % IPS) >> 5;
            const int c = ((lane >> 1) << 2) | ((vw & 1) << 1) | (lane & 1), q = vw >> 1;
            const int slot = ((c & 3) << 4) | (c >> 2);
            if (seg < nseg) {
                float *t = reinterpret_cast<float *>(sm + seg * C::TAB) + (4 * q) * STRIP + slot;
                t[0] = lq[n].x; t[STRIP] = lq[n].y; t[2 * STRIP] = lq[n].z; t[3 * STRIP] = lq[n].w;
            }
        }

        TRACE(2, tid == 0);
        // Everything below reads data the previous kernel may have produced (x, workspace).  One thread waits on the
        // programmatic dependency; the other consumers sleep on a hardware barrier instead of each polling it.
        if (tid == 0) pdl_wait();
        named_bar_sync(6, NW * 32);
        TRACE(3, tid == 0);

        // ---- stage the slice(s) of x this CTA needs, as fp32 ----
        for (int seg = 0; seg < nseg; ++seg) {
            const int ua = seg == 0 ? r0 : 0;                               // first unit of the segment inside its strip
            const int ub = min(R, r0 + len - seg * R);                      // one past the last
            const int dst_unit = p.x_direct ? ua : (seg * R + ua - r0);     // compact: indexed by unit offset
            const int nfl = (ub - ua) * C::XU;
            const int src_f = ua * C::XU, dst_f = dst_unit * C::XU;
            if (p.x_dt == SQLLM_DT_F16) {
                const __half *xh = reinterpret_cast<const __half *>(p.x) + src_f;
                for (int e = tid; e < nfl / 4; e += NW * 32) {  // 4 halves in, one float4 out per thread: conflict-free stores
                    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(xh) + e);
                    const __half2 *h = reinterpret_cast<const __half2 *>(&u);
                    const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]);
                    reinterpret_cast<float4 *>(xs + dst_f)[e] = make_float4(f0.x, f0.y, f1.x, f1.y);
                }
            } else if (p.x_dt == SQLLM_DT_BF16) {
                const __nv_bfloat16 *xb = reinterpret_cast<const __nv_bfloat16 *>(p.x) + src_f;
                for (int e = tid; e < nfl / 4; e += NW * 32) {  // the same, 4 bf16 in
                    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(xb) + e);
                    const float2 f0 = bf16x2_to_f32x2(u.x), f1 = bf16x2_to_f32x2(u.y);
                    reinterpret_cast<float4 *>(xs + dst_f)[e] = make_float4(f0.x, f0.y, f1.x, f1.y);
                }
            } else {
                const float *xf = reinterpret_cast<const float *>(p.x) + src_f;
                for (int e = tid; e < nfl / 4; e += NW * 32) cp_async16(xs_u32 + 4 * dst_f + 16 * e, xf + 4 * e);
            }
        }
        cp_async_commit();
        cp_async_wait_all();
        named_bar_sync(5, NW * 32);  // consumers only: LUTs, x slice, zeroed partials visible
        TRACE(4, tid == 0);
    }

    if (warp < NW) {
        // =========================== consumer warps ===========================
        // Everything in this loop is addressed through 32-bit shared-window addresses (no generic pointers: those make
        // the compiler rematerialise the window base through S2UR inside the loop when registers are tight).
        uint64_t acc[4] = {0ull, 0ull, 0ull, 0ull};
        uint32_t lsb = 0u, segc = 0u;
        uint32_t lsv[4] = {0u, 0u, 0u, 0u};
        const uint32_t part_u32 = sm_u32 + C::off_part(maxseg) + (warp * STRIP + 4 * i16) * 4;
        const uint32_t lane_slot = (uint32_t)((jsel << 6) | (i16 << 2));  // column 0 of this lane: slot ((0^jsel)<<4 | i16), x4 bytes

        auto set_seg = [&](int seg) {
            const uint32_t tb = sm_u32 + seg * C::TAB;
            // 4-bit: byte 1 of the address comes from the nibble | segc (table 4 KB aligned); 3-bit: bits 8..10 are free (2 KB aligned)
            lsb = (BITS == 4 ? (tb & 0xFFFF0000u) : tb) | lane_slot;
            segc = ((tb >> 8) & 0xF0u) * 0x01010101u;
            if constexpr (BITS == 3) {
                // 3-bit: the four per-column slot addresses are pinned in registers for the whole segment.  Left to itself the
                // compiler folds the `^ (t << 6)` into a second LOP3 per lookup (96 extra instructions per 128-weight position).
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    lsv[t] = lsb ^ (uint32_t)(t << 6);
                    asm volatile("mov.u32 %0, %0;" : "+r"(lsv[t]));
                }
            }
        };
        auto deposit = [&](int seg) {
            float s[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) s[t] = sum2(acc[t]);
            // lane (i, j=1) holds column t^1 in slot t: hand it to lane (i, j=0)
            const float v0 = __shfl_xor_sync(0xffffffffu, s[1], 16);
            const float v1 = __shfl_xor_sync(0xffffffffu, s[0], 16);
            const float v2 = __shfl_xor_sync(0xffffffffu, s[3], 16);
            const float v3 = __shfl_xor_sync(0xffffffffu, s[2], 16);
            if (jsel == 0)
                asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(part_u32 + seg * (NW * STRIP * 4)), "f"(s[0] + v0),
                             "f"(s[1] + v1), "f"(s[2] + v2), "f"(s[3] + v3) : "memory");
#pragma unroll
            for (int t = 0; t < 4; ++t) acc[t] = 0ull;
        };

        const uint32_t xlane = xs_u32 + (C::XU * 4) * jsel;
        const bool xdir = p.x_direct != 0;
        // Outer loop: the segments (strips) this warp has positions in; inner loop: a fixed trip
        // count of positions with nothing but running pointers: wait for the slot, pull it into registers, do the math,
        // refill the slot PF positions ahead.
        Cursor cc;
        cc.seek(0, warp2, r0, R, len, nseg);
        uint32_t slot = ring_u32;
        const uint32_t slot_end = ring_u32 + PF * SLOT_STRIDE;
        while (cc.seg < nseg) {
            set_seg(cc.seg);
            uint32_t xptr = xlane + (C::XU * 4) * (xdir ? cc.rr : cc.rr + cc.seg * R - r0);
            for (int i = cc.left; i > 0; --i) {
                cp_async_wait_pending<PF - 1>();
                Words<BITS> cur;
                cpa_fetch(cur, slot);
                consume(cur, jsel, lsb, segc, lsv, xptr, acc);
                cpa_issue(slot);  // the words are in registers (consumed above): the slot can be overwritten
                slot += SLOT_STRIDE;
                if (slot == slot_end) slot = ring_u32;
                xptr += SU * C::XU * 4;
            }
            deposit(cc.seg);
            cc.seek(cc.seg + 1, warp2, r0, R, len, nseg);
        }
        TRACE(6, tid == 0);
    }

    __syncthreads();  // all partials of this CTA are in shared memory
    TRACE(7, tid == 0);

    // =========================== flush ===========================
    if (tid < MAXSEG * STRIP) {
        const int seg = tid >> 6, c = tid & 63;
        const bool active = seg < nseg;
        int strip = 0, nd = 1, expected = 1;
        bool hyb = false;
        if (active) {
            strip = s0 + seg;
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < NW; ++w) tot += part[(seg * NW + w) * STRIP + c];
            expected = strip_contributors(p, strip, nd, hyb);
            if (expected == 1) {  // this CTA is the strip's only contributor: store directly
                const int col = strip * STRIP + c;
                if (col < N) {
                    if (p.bias) tot += p.bias[col];
                    store_y(p, col, tot);
                }
            } else {
                const int slot = (int)blockIdx.x - (int)(((long long)strip * R) / p.chunk);
                p.ws_part[((size_t)strip * p.maxc + slot) * STRIP + c] = tot;
            }
        }
        // ticket: 64 threads (2 warps) per segment; sync them with a named barrier per segment
        const bool ticketed = active && expected > 1;
        named_bar_sync(seg + 1, 64);
        if (c == 0) {
            int fin = 0;
            if (ticketed) {
                fin = (ticket_take(p.ws_cnt + strip) == expected - 1);
                if (fin) p.ws_cnt[strip] = 0;
            }
            misc[seg] = fin;
        }
        named_bar_sync(seg + 1, 64);
        if (misc[seg]) {
            float *ht = hyb_tot + seg * MAX_TOPX_FUSED;
            if (hyb) {  // the first warp of this segment's pair stages and sums the dense-row partials, then both warps use them
                const int cso = C::off_cstage(maxseg, p.xfloats);
                if ((c >> 5) == 0) hybrid_totals(p, sm_u32 + cso + CSR_CH * 8, reinterpret_cast<const float *>(sm + cso + CSR_CH * 8), ht, lane);
                named_bar_sync(seg + 1, 64);
            }
            final_store(p, strip, c, nd, hyb ? ht : nullptr);
        }
        TRACE(11, tid == 0);
    }
}

}  // namespace
