// lutgemv_v2.cuh - round-2 kernel: ONE fat CTA per SM, TMA-fed weight ring, one strip table at a time, optional fp16 pair tables.
//
// Same job as lutgemv_kernel (v1): y[c] (+)= sum_k LUT[c][idx(k,c)] * x[k]  (+ CSR outliers + topX dense rows), replacing
// squeezellm/quant_cuda_kernel.cu:741-880 (LUT GEMV), :1040-1059 (SPMV_ATOMIC), :1092-1123 (DenseMatVecKernel).
// What changed and why:
//   * grid = #SMs, 23 warps per CTA: 16 consumer warps, 1 TMA producer warp, 2 table-builder warps, 4 sparse warps.  v1 ran 3 CTAs x 8 consumer warps per SM;
//     most of its executed instructions on a 4096x4096 layer were per-CTA prologue/epilogue bookkeeping.
//   * weights arrive as 2-D TMA boxes (cp.async.bulk.tensor.2d): stages are aligned to the CTA's strip segments, so a full stage is
//     ONE box of 64 columns x 32 units (8 KB / 24 KB) issued by one lane of the producer warp; the ragged last stage of a segment
//     goes out as 2-unit boxes, one per lane (second tensor map), so nothing is over-fetched.  (One 256-byte cp.async.bulk
//     per row instead was much slower: the TMA unit retires small copies slowly.)
//     Nothing of this touches the LSU pipe, which bounds the gather loop (32 gathers + 4 word reads + 2-4 x reads per 1024 weights).
//   * the CTA walks its strips one after the other with TWO table buffers in shared memory: the builder warps prepare the next strip's
//     table in the background and move each finished strip's sums (red.shared.add by the consumer warps) on to global memory; the
//     consumers never meet a CTA-wide barrier inside the loop.  Only two tables resident is what makes room for the
//   * fp16 PAIR table (MODE 1): entry [a | b<<BITS] = half2(LUT[a], LUT[b]) - one PRMT-built (4-bit: the byte of the packed word IS
//     the entry number) shared-memory lookup serves TWO weights, and the products are fp16 x fp16 -> fp32 accumulate with
//     exact products (fhfma2; tests/perf/microbench2.cu measures the loop).  The only rounding is LUT -> fp16 (2^-11 relative per centroid); it needs fp16 x.
//   * x is staged whole in its own type (fp32, fp16 or bf16: the XT template parameter; 16-bit pairs are widened to fp32 in registers),
//     the sparse warps gather it from shared memory (sparse3: nothing else of theirs goes through shared memory).
// The warp roles' per-segment work is text #included by this kernel and the sequence kernel (lutgemv_seq.cuh), each text opening with
// the names its includer defines: the producer's lutgemv_stream.inc, the builders' lutgemv_tables.inc and lutgemv_finish.inc, the
// consumers' lutgemv_segment.inc (DESIGN §3.4).
#pragma once
#include "common.cuh"

namespace {

namespace v2 {

constexpr int NWC = 16;                         // consumer warps
constexpr int WARP_PROD = NWC;                  // TMA producer
constexpr int WARP_BLD = NWC + 1;               // first of the 2 table-builder warps
constexpr int NBW = 2;
constexpr int WARP_SP = WARP_BLD + NBW;         // first of the sparse warps
constexpr int NSPW = 4;                         // sparse warps: their shared-memory accesses queue behind the consumers' (the LSU pipe is
                                                // saturated), so outlier work is latency-bound per warp - four warps, four times the progress
constexpr int THREADS2 = (NWC + 1 + NBW + NSPW) * 32;  // 736 (641..768 threads: 80 registers per thread)
constexpr int NCT = NWC * 32;                   // consumer threads
constexpr int NBT = NBW * 32;                   // builder threads: one per column slot of a strip
constexpr int SU2 = 2 * NWC;                    // units per stage (one pair per consumer warp)
constexpr int MAXD = 16;                        // ring depth limit (mbarrier slots)
constexpr int HYB_R2 = 11;
static_assert(NBT == STRIP, "one builder thread per column of a strip");
// shared-memory carve-up, offsets from a 128-byte aligned base
constexpr int OFF_BAR = 0;                      // full[s] at +8s, empty[s] at +128+8s, tfull[b] at +256+8b, tfree[b] at +272+8b
constexpr int OFF_SACC = 512;                   // float [2][64]: per-strip sums of the consumer warps (red.shared.add), ping-pong by strip parity
constexpr int OFF_LUT = OFF_SACC + 2 * STRIP * 4;            // 2 x raw fp32 LUT rows of a strip (64 columns x 16 values), staged ahead by the builders
constexpr int LUTBUF = STRIP * (16 * 4 + 16);                // a strip's raw LUT rows, one per column SLOT, row stride L*4 + 16 bytes (see lut_prefetch)
constexpr int OFF_FIN = OFF_LUT + 2 * LUTBUF;                // finishers: float sown[8][64] (own strip sums), int sdj[128], float sden[128], int sdn (dense rows)
constexpr int OFF_X = OFF_FIN + 4096;                        // x (fp16 or fp32), then [ring stages][table 0][table 1][ring stages]
static_assert(OFF_X % 128 == 0, "x must stay 128-byte aligned");

struct P2 {
    const uint32_t *qw;
    const float *lut;
    const void *x;
    void *out;           // accumulate mode: float* mul ; fused: fp32 or 16-bit y (y16_t of x's type)
    const float *bias;
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX, K, N, R, T, chunk, nstage;
    unsigned smem_raw;   // shared-window address of the dynamic shared memory the host planned the carve-up for (checked by the kernel)
    int y_is_half;
    int hc, hrows, csr_rpc;
    float *ws_acc;       // fused: [N] fp32 accumulator, zero between launches
    unsigned long long *ws_hbox;  // fused: [grid][64] partial strip sums of a CTA's first segment when the strip starts in an earlier CTA
    unsigned long long *ws_cbox;  // fused: [N] outlier (CSR) row sums; both {float value, u32 valid}, all zero between launches
    unsigned long long *ws_dbox;  // sequence kernel: [topX][MAX_GRID_V2] dense-row partial sums, one tagged word per (dense row, contributing CTA)
    int *ws_cnt;         // fused: [16] error flag (a bounded wait gave up; sqllm_workspace_error)
    int strips;          // output strips of 64 columns
    int nown_ctas;       // exchange: CTAs that own at least one strip (each announces itself once on every rank)
    int xw_world, xw_rank, xw_members, xw_nfull;
    const unsigned long long *xw_base;
    unsigned long long xw_out_off, xw_flag_off, xw_state_off, xw_err_off;
    unsigned long long *trace;
};

template <int BITS, int MODE>
struct C2 {
    static constexpr int L = 1 << BITS;
    static constexpr int ENT = MODE ? L * L : L;             // table rows
    static constexpr int TAB = ENT * STRIP * 4;              // 4 KB / 2 KB exact, 64 KB / 16 KB pair
    static constexpr int ROWS = BITS == 4 ? 1 : 3;           // packed rows per unit
    static constexpr int XU = BITS == 4 ? 8 : 32;            // inputs per unit
    static constexpr int UNIT = ROWS * STRIP * 4;            // bytes of one unit in a stage
    static constexpr int SU = SU2;                           // units per stage
    static constexpr bool ROT = false;                       // no 64-unit stages (G2), so the sequence kernel runs 32-unit ones
    static constexpr int STAGE = SU2 * UNIT;                 // 8 KB / 24 KB
    static constexpr int NTB = TAB <= 16384 ? 4 : 2;         // sequence kernel: table buffers (and strip accumulators), 4 x 4 KB exact, 2 x 64 KB for the 4-bit pair table
};
// The one-GEMV kernel's plan (lutgemv2_kernel; the sequence kernel keeps C2's).  4-bit exact (ROT): a stage is 64 units, two positions per
// consumer warp behind one full-barrier wait, and a table buffer holds the strip table twice - copy 0 for the even half-warps, copy 1
// (4 KB above, entry of slot s at slot s ^ 16: bank-rotated by 16) for the odd ones, so that both read column t of their lane with
// word t and still hit 32 different banks.  Every other mode: 32-unit stages and one copy, as C2.
template <int BITS, int MODE>
struct G2 : C2<BITS, MODE> {
    static constexpr bool ROT = BITS == 4 && MODE == 0;
    static constexpr int SU = ROT ? 2 * SU2 : SU2;           // units per stage
    static constexpr int STAGE = SU * C2<BITS, MODE>::UNIT;  // 16 KB 4-bit exact ; 8 KB / 24 KB otherwise
    static constexpr int TAB = (ROT ? 2 : 1) * C2<BITS, MODE>::TAB;
    // ring depth limit.  ROT: 3 stages (48 KB per SM).  Measured on the 7B chain (DESIGN §6), a shallow ring is faster: with 132 SMs
    // each holding 128 KB of requests at once, the launch's last CTAs finish later than with 48 KB.
    static constexpr int RING = ROT ? 3 : MAXD;
};

// Shared-memory carve-up of lutgemv2_kernel and lutgemv_seq_kernel, from the 128-byte aligned base:
//   [fixed OFF_X][x: xbytes][front][ring stages 0 .. n_lo)[ntab tables, each aligned to its own size][ring stages n_lo .. nstage)
// The kernels place their buffers by it and the host sizes the launch and the ring by it: both must see the same addresses.
struct Carve {
    uint32_t lo_base;  // ring stage s < n_lo lives at lo_base + s * stage
    uint32_t tab0;     // table b lives at tab0 + b * tab
    uint32_t tab_end;
    int lo_cap;        // ring stages that fit below the tables
    int n_lo;
    uint32_t hi_base;  // ring stage s >= n_lo lives at hi_base + s * stage
    uint32_t end;      // end of the used window
    __host__ __device__ __forceinline__ Carve(uint32_t base, uint32_t xbytes, uint32_t front, uint32_t tab, int ntab, uint32_t stage, int nstage)
        : lo_base(base + OFF_X + xbytes + front),
          tab0((lo_base + tab - 1u) & ~(tab - 1u)),
          tab_end(tab0 + (uint32_t)ntab * tab),
          lo_cap((int)((tab0 - lo_base) / stage)),
          n_lo(nstage < lo_cap ? nstage : lo_cap),
          hi_base(tab_end - (uint32_t)n_lo * stage),
          end(hi_base + (uint32_t)nstage * stage) {}
    // host: the ring depth for a window of `bytes` from `raw` - the stages that fit below and above the tables, at most `cap` and
    // MAXD; -1: the tables themselves do not fit
    int depth(uint32_t raw, int bytes, uint32_t stage, int cap) const {
        const long long hi_room = (long long)raw + bytes - (long long)tab_end;
        if (hi_room < 0) return -1;
        return (int)std::min<long long>(std::min(cap, MAXD), lo_cap + hi_room / stage);
    }
};

__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
// acc_lo += lo16(w) * lo16(x) ; acc_hi += hi16(w) * hi16(x).  Hopper has no fp16 x fp16 -> fp32 FMA: the halves are widened
// (exact) and go through fma.rn.f32.  An fp16 x fp16 product is exact in fp32, so the single rounding is the accumulation's.
__device__ __forceinline__ void fhfma2(float &acc_lo, float &acc_hi, uint32_t w, uint32_t x) {
    asm("{\n.reg .b16 wl, wh, xl, xh;\n.reg .f32 fwl, fwh, fxl, fxh;\nmov.b32 {wl, wh}, %2;\nmov.b32 {xl, xh}, %3;\n"
        "cvt.f32.f16 fwl, wl;\ncvt.f32.f16 fwh, wh;\ncvt.f32.f16 fxl, xl;\ncvt.f32.f16 fxh, xh;\n"
        "fma.rn.f32 %0, fwl, fxl, %0;\nfma.rn.f32 %1, fwh, fxh, %1;\n}"
        : "+f"(acc_lo), "+f"(acc_hi) : "r"(w), "r"(x));
}
// the two 16-bit x values of a word (fp16 or bf16: XT) as a packed fp32 pair, exactly
template <typename XT>
__device__ __forceinline__ uint64_t x2_to_f32x2(uint32_t h) {
    const float2 f = x16x2_to_f32x2<XT>(h);
    return pack2(f.x, f.y);
}
__device__ __forceinline__ uint32_t f32x2_to_half2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&h);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Table build, by the NCT consumer threads.  Column c of the strip lives in slot ((c & 3) << 4) | (c >> 2): lane i16 of a half-warp
// owns columns 4*i16..4*i16+3, i.e. slots i16, 16+i16, 32+i16, 48+i16, so at every step the 32 lanes of a warp hit 32 different banks.
//   exact : row v, slot s  = LUT[c][v]                                  (fp32)
//   pair  : row a | b<<BITS = half2(lo = LUT[c][a], hi = LUT[c][b])      (a: the even input of the pair, b: the odd one)
// Columns past N read as zeros (ragged last strip: whatever index the stale stage bytes hold, the product is 0).
// ---------------------------------------------------------------------------------------------------------------------------
// Tables are built by the two builder warps (thread = slot = one column of the strip) from the strip's raw LUT rows, which they stage
// in shared memory first (lut_prefetch, zero-filled past N): a build never waits on global memory, and it runs in the background -
// the consumers only ever wait on an mbarrier that is normally long complete.  (First v2 build: the consumers rebuilt the table
// themselves at every strip boundary; that left a bubble per switch with the warps stalled on the LUT loads.)
// ---------------------------------------------------------------------------------------------------------------------------
// Mailboxes (fused mode).  A sum that one CTA produces and another CTA needs - the partial strip sums of a CTA whose first
// segment continues a strip started earlier, and every outlier row sum (the CSR rows are spread evenly over the CTAs) - is written
// ONCE, as one 64-bit word {fp32 value, valid = 1}, and the strip's owner polls that word.  A 64-bit access is single-copy atomic, so
// the value needs no fence and no separate flag: the word validates itself.  Before: red.add into the accumulator, MEMBAR, flag
// increment on the producer; acquire-poll of the flag, then a second round trip for the accumulator on the owner - three L2 round
// trips under load between the last weight of a launch and its last y, now one.  The owner writes the word back to zero
// (next launch's producers only write after the grid dependency resolved).  The dense-row sums travel the same way since the second
// half of round 2: one word per (contributing CTA, dense row) - rows that feed the same channel are combined in the contributing warp -
// summed by the owner of the channel's strip; and the owner's OWN strip sums never leave the SM (sown, a shared-memory row per owned
// strip).  Before: red.add into the global accumulator + MEMBAR.GPU + one announcement per strip on the producers, an acquire-poll and a
// load of the accumulator behind it on the owner.
// ---------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// `tag` is what makes a word valid: 1 for the one-GEMV kernel (the owner writes the word back to zero), a value unique to the (token, GEMV)
// for the sequence kernel (lutgemv_seq.cuh), where words are never reset (keep = true): a stale word simply carries an older tag.
__device__ __forceinline__ unsigned long long box_word(float v, uint32_t tag = 1u) { return ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v); }
// value of a mailbox word read speculatively as `w`; spins (bounded: 2 s, then the workspace error word) until it is valid; clears it
__device__ __forceinline__ float box_take(unsigned long long w, unsigned long long *ptr, int *err, const uint32_t tag = 1u, const bool keep = false) {
    if ((uint32_t)(w >> 32) != tag) {
        unsigned long long t0, t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        do {
            w = ld_relaxed_u64(ptr);
            if ((uint32_t)(w >> 32) == tag) break;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile int *>(err) = 1; break; }
        } while (true);
    }
    if (!keep) st_relaxed_u64(ptr, 0ull);
    return __uint_as_float((uint32_t)w);
}

// Staging layout: the row of column c sits at slot(c) * (L*4 + 16) bytes.  The builders read it with 16-byte loads, lane = slot: with the
// rows packed by column (stride 4 columns x 64 B = 256 B between adjacent lanes) every LDS.128 was an 8-way bank conflict, and the
// pair-table build re-reads the row for each of its 16 outer steps, so these conflicts cost LSU time the gathers need.  With an 80-byte
// (4-bit) / 48-byte (3-bit) stride the 8 lanes of each 128-byte phase cover all 32 banks.
template <int BITS>
__device__ __forceinline__ void lut_prefetch(const P2 &p, const uint32_t lutbuf, const int strip, const int bt) {
    constexpr int L = 1 << BITS;
    constexpr int N16 = STRIP * L / 4;  // 16-byte pieces: 256 (w4) / 128 (w3)
#pragma unroll
    for (int e = bt; e < N16; e += NBT) {
        const int c = e / (L / 4), q = e % (L / 4), col = strip * STRIP + c;
        const int slot = ((c & 3) << 4) | (c >> 2);
        const bool ok = col < p.N;
        cp_async16_clip(lutbuf + slot * (L * 4 + 16) + 16 * q, p.lut + (ok ? (size_t)strip * STRIP * L + 4 * (size_t)e : 0), ok ? 16 : 0);
    }
    cp_async_commit();
}

// ROT (G2): also the bank-rotated second copy of the exact table, C2::TAB bytes above the first.
template <int BITS, int MODE, bool ROT = false>
__device__ __forceinline__ void build_table(const uint32_t tab, const uint32_t lutbuf, const int slot) {
    using C = C2<BITS, MODE>;
    const uint32_t row = lutbuf + slot * (C::L * 4 + 16);    // the staged LUT row of the column this slot serves (slot s <-> column (s & 15) * 4 + (s >> 4))
    const uint32_t a0 = tab + (slot << 2);                   // a warp's 32 lanes = 32 consecutive slots: conflict-free stores
    float v[C::L];
#pragma unroll
    for (int q = 0; q < C::L / 4; ++q) {
        const float4 f = lds_v4(row + 16 * q);
        v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
    }
    if constexpr (MODE == 0) {
#pragma unroll
        for (int e = 0; e < C::L; ++e) sts_u32(a0 + e * (STRIP * 4), __float_as_uint(v[e]));
        if constexpr (ROT) {
            const uint32_t a1 = tab + C::TAB + ((slot ^ 16) << 2);
#pragma unroll
            for (int e = 0; e < C::L; ++e) sts_u32(a1 + e * (STRIP * 4), __float_as_uint(v[e]));
        }
    } else {
        uint32_t H[C::L / 2];  // H[m] = half2(LUT[2m], LUT[2m+1])
#pragma unroll
        for (int m = 0; m < C::L / 2; ++m) H[m] = f32x2_to_half2(v[2 * m], v[2 * m + 1]);
#pragma unroll
        for (int b = 0; b < C::L; ++b) {
#pragma unroll
            for (int a = 0; a < C::L; ++a) {
                // row a | b << BITS : low half <- LUT[a] = half (a & 1) of H[a >> 1], high half <- LUT[b] = half (b & 1) of H[b >> 1]
                const uint32_t sel = (uint32_t)(((5 + 2 * (b & 1)) << 12) | ((4 + 2 * (b & 1)) << 8) | ((2 * (a & 1) + 1) << 4) | (2 * (a & 1)));
                sts_u32(a0 + ((a | (b << BITS)) << 8), __byte_perm(H[a >> 1], H[b >> 1], sel));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Per-position math.  A lane holds 4 adjacent columns x one unit; slot addresses l[t] (column t ^ jsel of the lane) are fixed
// for the whole kernel because there is one table.  Accumulators: exact -> 4 packed (even k, odd k) fp32 pairs; pair -> 8 fp32.
// ---------------------------------------------------------------------------------------------------------------------------
struct Acc {
    uint64_t a[4];
    float f[8];
};

// What a lane pulls out of a stage for one position: its 16 bytes (x 3 rows for 3-bit) and - 4-bit only, 8 inputs - its slice of x
// (X16: x is staged in a 16-bit type, fp16 or bf16).
template <int BITS, bool X16> struct FetchX;
template <> struct FetchX<4, true> { uint4 q, xh; };
template <> struct FetchX<4, false> { uint4 q; float4 xa, xb; };
template <bool X16> struct FetchX<3, X16> { uint4 a, b, c; };
template <int BITS, typename XT> using Fetch = FetchX<BITS, x_is16<XT>>;

template <int BITS, typename XT>
__device__ __forceinline__ void fetch2(Fetch<BITS, XT> &F, const uint32_t unit_addr, const uint32_t xaddr) {
    if constexpr (BITS == 4) {
        F.q = lds_u4(unit_addr);
        if constexpr (x_is16<XT>) F.xh = lds_u4(xaddr);
        else { F.xa = lds_v4(xaddr); F.xb = lds_v4(xaddr + 16); }
    } else {
        F.a = lds_u4(unit_addr);
        F.b = lds_u4(unit_addr + STRIP * 4);
        F.c = lds_u4(unit_addr + 2 * STRIP * 4);
    }
}

// 4-bit, exact fp32 table (v1's loop): E/O = even/odd nibbles in separate bytes, OR-ed with bits 12..15 of the table address.
template <typename XT>
__device__ __forceinline__ void consume4_exact(const Fetch<4, XT> &F, const int jsel, const uint32_t (&l)[4], const uint32_t segc, Acc &A) {
    uint64_t x01, x23, x45, x67;
    if constexpr (x_is16<XT>) {
        x01 = x2_to_f32x2<XT>(F.xh.x); x23 = x2_to_f32x2<XT>(F.xh.y); x45 = x2_to_f32x2<XT>(F.xh.z); x67 = x2_to_f32x2<XT>(F.xh.w);
    } else {
        x01 = pack2(F.xa.x, F.xa.y); x23 = pack2(F.xa.z, F.xa.w); x45 = pack2(F.xb.x, F.xb.y); x67 = pack2(F.xb.z, F.xb.w);
    }
    const uint4 q = F.q;
    const uint32_t w[4] = {jsel ? q.y : q.x, jsel ? q.x : q.y, jsel ? q.w : q.z, jsel ? q.z : q.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const uint32_t E = (w[t] & 0x0F0F0F0Fu) | segc;
        const uint32_t O = ((w[t] >> 4) & 0x0F0F0F0Fu) | segc;
        const float e0 = lds_f32(__byte_perm(E, l[t], 0x7604)), o0 = lds_f32(__byte_perm(O, l[t], 0x7604));
        const float e1 = lds_f32(__byte_perm(E, l[t], 0x7614)), o1 = lds_f32(__byte_perm(O, l[t], 0x7614));
        const float e2 = lds_f32(__byte_perm(E, l[t], 0x7624)), o2 = lds_f32(__byte_perm(O, l[t], 0x7624));
        const float e3 = lds_f32(__byte_perm(E, l[t], 0x7634)), o3 = lds_f32(__byte_perm(O, l[t], 0x7634));
        ffma2(A.a[t], pack2(e0, o0), x01);
        ffma2(A.a[t], pack2(e1, o1), x23);
        ffma2(A.a[t], pack2(e2, o2), x45);
        ffma2(A.a[t], pack2(e3, o3), x67);
    }
}
// 4-bit, fp16 pair table (64 KB aligned): byte j of a packed word = (index of input 2j) | (index of input 2j+1) << 4 = the entry number.
__device__ __forceinline__ void consume4_pair(const Fetch<4, __half> &F, const int jsel, const uint32_t (&l)[4], Acc &A) {
    const uint4 q = F.q, xh = F.xh;  // halves (x0,x1) (x2,x3) (x4,x5) (x6,x7)
    const uint32_t w[4] = {jsel ? q.y : q.x, jsel ? q.x : q.y, jsel ? q.w : q.z, jsel ? q.z : q.w};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const uint32_t p0 = lds_u32(__byte_perm(w[t], l[t], 0x7604)), p1 = lds_u32(__byte_perm(w[t], l[t], 0x7614));
        const uint32_t p2 = lds_u32(__byte_perm(w[t], l[t], 0x7624)), p3 = lds_u32(__byte_perm(w[t], l[t], 0x7634));
        fhfma2(A.f[t], A.f[t + 4], p0, xh.x);
        fhfma2(A.f[t], A.f[t + 4], p1, xh.y);
        fhfma2(A.f[t], A.f[t + 4], p2, xh.z);
        fhfma2(A.f[t], A.f[t + 4], p3, xh.w);
    }
}
// 3-bit pair table (16 KB aligned): the three words of a group are a 96-bit stream of 32 3-bit fields (quant.py:185-203), so pair
// p = (input 2p, input 2p+1) is the 6-bit field at stream bit 6p.  Moved to bits 8..13 by one shift (a funnel shift for pairs 5, 10).
template <int SH>
__device__ __forceinline__ uint32_t fld8(uint32_t w) {
    if constexpr (SH < 8) return w << (8 - SH);
    else if constexpr (SH == 8) return w;
    else return w >> (SH - 8);
}
#define LKP(e, word_expr) e = lds_u32((((word_expr)) & 0x3F00u) | lsv)
__device__ __forceinline__ void consume3_pair_col(const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t lsv,
                                                  const uint32_t (&xh)[16], float &fa, float &fb) {
    uint32_t e;
    LKP(e, fld8<0>(w0));  fhfma2(fa, fb, e, xh[0]);
    LKP(e, fld8<6>(w0));  fhfma2(fa, fb, e, xh[1]);
    LKP(e, fld8<12>(w0)); fhfma2(fa, fb, e, xh[2]);
    LKP(e, fld8<18>(w0)); fhfma2(fa, fb, e, xh[3]);
    LKP(e, fld8<24>(w0)); fhfma2(fa, fb, e, xh[4]);
    LKP(e, __funnelshift_r(w0, w1, 22)); fhfma2(fa, fb, e, xh[5]);   // stream bits 30..35
    LKP(e, fld8<4>(w1));  fhfma2(fa, fb, e, xh[6]);
    LKP(e, fld8<10>(w1)); fhfma2(fa, fb, e, xh[7]);
    LKP(e, fld8<16>(w1)); fhfma2(fa, fb, e, xh[8]);
    LKP(e, fld8<22>(w1)); fhfma2(fa, fb, e, xh[9]);
    LKP(e, __funnelshift_r(w1, w2, 20)); fhfma2(fa, fb, e, xh[10]);  // stream bits 60..65
    LKP(e, fld8<2>(w2));  fhfma2(fa, fb, e, xh[11]);
    LKP(e, fld8<8>(w2));  fhfma2(fa, fb, e, xh[12]);
    LKP(e, fld8<14>(w2)); fhfma2(fa, fb, e, xh[13]);
    LKP(e, fld8<20>(w2)); fhfma2(fa, fb, e, xh[14]);
    LKP(e, fld8<26>(w2)); fhfma2(fa, fb, e, xh[15]);
}
#undef LKP

template <int BITS, int MODE, typename XT>
__device__ __forceinline__ void math2(const Fetch<BITS, XT> &F, const int jsel, const uint32_t (&l)[4], const uint32_t segc, const uint32_t xaddr, Acc &A) {
    if constexpr (BITS == 4) {
        if constexpr (MODE == 0) consume4_exact<XT>(F, jsel, l, segc, A);
        else consume4_pair(F, jsel, l, A);
    } else {
        const uint4 ga = F.a, gb = F.b, gc = F.c;
        const uint32_t a[4] = {jsel ? ga.y : ga.x, jsel ? ga.x : ga.y, jsel ? ga.w : ga.z, jsel ? ga.z : ga.w};
        const uint32_t b[4] = {jsel ? gb.y : gb.x, jsel ? gb.x : gb.y, jsel ? gb.w : gb.z, jsel ? gb.z : gb.w};
        const uint32_t c[4] = {jsel ? gc.y : gc.x, jsel ? gc.x : gc.y, jsel ? gc.w : gc.z, jsel ? gc.z : gc.w};
        if constexpr (MODE == 0) {
            uint64_t xp[16];
            if constexpr (x_is16<XT>) {
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const uint4 h = lds_u4(xaddr + 16 * v);
                    xp[4 * v] = x2_to_f32x2<XT>(h.x); xp[4 * v + 1] = x2_to_f32x2<XT>(h.y);
                    xp[4 * v + 2] = x2_to_f32x2<XT>(h.z); xp[4 * v + 3] = x2_to_f32x2<XT>(h.w);
                }
            } else {
#pragma unroll
                for (int v = 0; v < 8; ++v) {
                    const float4 f = lds_v4(xaddr + 16 * v);
                    xp[2 * v] = pack2(f.x, f.y);
                    xp[2 * v + 1] = pack2(f.z, f.w);
                }
            }
#pragma unroll
            for (int t = 0; t < 4; ++t) consume3_col(a[t], b[t], c[t], l[t], xp, A.a[t]);
        } else {
            uint32_t xh[16];
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                const uint4 h = lds_u4(xaddr + 16 * v);
                xh[4 * v] = h.x; xh[4 * v + 1] = h.y; xh[4 * v + 2] = h.z; xh[4 * v + 3] = h.w;
            }
#pragma unroll
            for (int t = 0; t < 4; ++t) consume3_pair_col(a[t], b[t], c[t], l[t], xh, A.f[t], A.f[t + 4]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Outlier warps (NSPW per CTA), shared by lutgemv2_kernel and the sequence kernel.  CSR rows (= output channels) are spread evenly over
// the CTAs (csr_rpc consecutive rows each, split between the CTA's sparse warps); warp 0 also takes the CTA's k-slice of the topX dense
// rows.  Nothing but x goes through shared memory: the LSU pipe is what bounds the kernel, so every dependent shared-memory access of
// these warps queues for hundreds of cycles behind the consumers' gathers.  (Before: the (col, val) pairs were staged in 256-element
// chunks with cp.async, the products formed in place and the rows summed from there - four or more dependent shared-memory round trips
// per chunk; on a 4096x4096 layer the outlier warps finished after the last consumer warp and set the layer's critical path,
// tests/perf/seq_trace.cu.)  Here:
//   * LPR lanes share a row (LPR from the average row length), 32 / LPR rows per pass; a lane keeps its <= T (col, val) pairs of the
//     pass in REGISTERS, loaded straight from global memory (the warp's whole non-zero range is prefetched into L2 at entry) -
//     everything static, so the first pass is in registers before x arrives and the loads of pass k+1 are issued before pass k is summed;
//   * after x: one round of x gathers (the only shared-memory accesses), FMAs, a shuffle tree over the LPR lanes, and one result per
//     row: a 64-bit mailbox word {sum, boxtag} (fused mode; rows without outliers store 0: the strip's owner waits for all its rows) or
//     one red.add into `acc_out` (accumulate mode: the 12 symbols);
//   * the part of a row beyond T x LPR elements is summed by the whole warp (skewed rows).
// `boxtag` is 1 for the one-GEMV kernel (the owner resets the words) and the (token, GEMV) tag for the sequence kernel (box_word).
// Dense rows: this CTA's k-slice of full_rows, prefetched into L2 at entry, the first HYB_R2 per row slot in registers before x arrives
// (the rest is read after x: from L2, not from HBM - every owner of a dense-row channel waits for the slowest CTA's warp 0); one mailbox word per
// (CTA, dense row), rows on the same channel combined (fused), or one red.add per dense row into its channel (accumulate).
// ---------------------------------------------------------------------------------------------------------------------------
template <typename XT>
__device__ __forceinline__ float xs_load(const uint32_t xs_u32, const int k) {
    if constexpr (x_is16<XT>) {
        unsigned short h;
        asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(xs_u32 + 2 * k));
        if constexpr (std::is_same<XT, __nv_bfloat16>::value) return __uint_as_float((uint32_t)h << 16);
        else return __half2float(__ushort_as_half(h));
    } else {
        return lds_f32(xs_u32 + 4 * k);
    }
}

template <typename XT, bool FUSED>
__device__ __forceinline__ void sparse3(const P2 &p, const uint32_t base, const int spw, const int lane, float *acc_out, const uint32_t boxtag) {
    const int N = p.N;
    const uint32_t xs_u32 = base + OFF_X;
    // ---------------- static: dense-row slice ----------------
    float hfr[HYB_R2];
    const bool hyb_on = p.full_rows && spw == 0 && (int)blockIdx.x < p.hc;
    const bool hyb_multi = hyb_on && p.topX <= 32;  // 32/topX k-rows per warp step: lane = (row slot, column j)
    int kb = 0, ke = 0, nsl = 1, rs = 0, hj = lane;
    if (hyb_on) {
        kb = blockIdx.x * p.hrows; ke = min(p.K, kb + p.hrows);
        // the slice is contiguous ([kb, ke) x topX floats): into L2 now, so that the rows read after x arrives are L2 hits
        const char *f0 = reinterpret_cast<const char *>(p.full_rows + (size_t)kb * p.topX);
        for (int i = lane; i < (int)(((size_t)(ke - kb) * p.topX * 4 + 127) / 128); i += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(f0 + 128 * i));
    }
    if (hyb_multi) {
        nsl = 32 / p.topX;
        rs = lane / p.topX;
        hj = lane - rs * p.topX;
#pragma unroll
        for (int i = 0; i < HYB_R2; ++i) {
            const int k = kb + rs + nsl * i;
            hfr[i] = (rs < nsl && k < ke) ? __ldg(p.full_rows + (size_t)k * p.topX + hj) : 0.f;
        }
    }
    // ---------------- static: this warp's CSR rows [r, rb) of the CTA's [ca, cb) ----------------
    int r = 0, rb = 0;
    if (p.rows) {
        const int ca = min(N, (int)blockIdx.x * p.csr_rpc), cb = min(N, ca + p.csr_rpc);
        // warp 0 has the dense rows and then takes no CSR rows: the outlier sums are what the owners of ALL strips wait for, they must
        // not queue behind the dense-row work
        const int tot = cb - ca, w0 = p.full_rows ? 0 : tot / NSPW, rest = tot - w0;
        r = spw == 0 ? ca : ca + w0 + (int)((long long)rest * (spw - 1) / (NSPW - 1));
        rb = spw == 0 ? ca + w0 : ca + w0 + (int)((long long)rest * spw / (NSPW - 1));
    }
    const int nr = rb - r;
    int LPR = 4;
    if (nr > 0) {
        const int e_lo = __ldg(p.rows + r), e_hi = __ldg(p.rows + rb);
        for (int e = (e_lo & ~31) + 32 * lane; e < e_hi; e += 32 * 32) {
            asm volatile("prefetch.global.L2 [%0];" ::"l"(p.cols + e));
            asm volatile("prefetch.global.L2 [%0];" ::"l"(p.vals + e));
        }
        const int avg = (e_hi - e_lo) / nr;
        LPR = avg > 128 ? 32 : avg > 64 ? 16 : avg > 32 ? 8 : avg > 8 ? 4 : 2;
    }
    const int RPP = 32 / LPR, part = lane & (LPR - 1), rslot = lane / LPR;
    const int npass = (nr + RPP - 1) / RPP;
    constexpr int T = 8;  // (col, val) pairs per lane and pass
    auto load_ptrs = [&](int pass, int &a0, int &a1) {
        const int row = r + pass * RPP + rslot;
        a0 = a1 = 0;
        if (pass < npass && row < rb) { a0 = __ldg(p.rows + row); a1 = __ldg(p.rows + row + 1); }
    };
    auto load_elems = [&](int a0, int a1, int (&cc)[T], float (&vv)[T]) {
#pragma unroll
        for (int t = 0; t < T; ++t) {
            const int e = a0 + part + t * LPR;
            const bool ok = e < a1;
            cc[t] = ok ? __ldg(p.cols + e) : 0;
            vv[t] = ok ? __ldg(p.vals + e) : 0.f;
        }
    };
    int a0c, a1c, a0n, a1n, a0nn, a1nn;
    int cc[T], cn[T];
    float vv[T], vn[T];
    load_ptrs(0, a0c, a1c);
    load_ptrs(1, a0n, a1n);
    load_elems(a0c, a1c, cc, vv);

    named_bar_sync(2, NCT + NSPW * 32);  // x is in shared memory (and the previous kernel has completed: the consumers waited on it)

    // ---------------- dense rows ----------------
    if (hyb_on) {
        for (int jb = 0; jb < (hyb_multi ? 1 : p.topX); jb += 32) {
            float a = 0.f;
            int j;
            if (hyb_multi) {
                j = hj;
#pragma unroll
                for (int i = 0; i < HYB_R2; ++i) {
                    const int k = kb + rs + nsl * i;
                    if (rs < nsl && k < ke) a += hfr[i] * xs_load<XT>(xs_u32, k);
                }
                for (int k = kb + rs + nsl * HYB_R2; rs < nsl && k < ke; k += nsl)
                    a += __ldg(p.full_rows + (size_t)k * p.topX + hj) * xs_load<XT>(xs_u32, k);
                for (int sl = 1; sl < nsl; ++sl) {  // fold the row slots onto slot 0 in fixed order
                    const float v = __shfl_sync(0xffffffffu, a, (hj + sl * p.topX) & 31);
                    if (rs == 0) a += v;
                }
                if (rs != 0) j = p.topX;  // only slot 0 publishes
                if constexpr (FUSED) {
                    // dense rows that feed the SAME channel travel as one word (the first of them carries the sum): the owner of that channel's
                    // strip then reads hc words, not hc per row - a checkpoint without dense rows loads as topX rows on channel 0 (llama.py:182)
                    const int cme = (rs == 0 && hj < p.topX) ? __ldg(p.fri + hj) : -1 - lane;
                    bool first = true;
                    float tot = a;
                    for (int j2 = 0; j2 < p.topX; ++j2) {
                        const int c2 = __shfl_sync(0xffffffffu, cme, j2);
                        const float a2 = __shfl_sync(0xffffffffu, a, j2);
                        if (c2 == cme && j2 < hj) first = false;
                        if (c2 == cme && j2 > hj) tot += a2;
                    }
                    a = tot;
                    if (!first) j = p.topX;
                }
            } else {
                j = jb + lane;
                if (j < p.topX) {
                    const float *fr = p.full_rows + (size_t)kb * p.topX + j;
                    for (int k = kb; k < ke; ++k, fr += p.topX) a += __ldg(fr) * xs_load<XT>(xs_u32, k);
                }
            }
            if constexpr (FUSED) {
                // this CTA's part of dense row j: one self-validating word, no RED + fence + flag (the owner of the channel's strip sums the
                // hc words of row j, the finishers of lutgemv2_kernel / lutgemv_seq_kernel)
                if (j < p.topX) st_relaxed_u64(p.ws_dbox + (size_t)j * MAX_GRID_V2 + blockIdx.x, box_word(a, boxtag));
            } else if (j < p.topX) {
                const int c = __ldg(p.fri + j);
                if (c >= 0 && c < N) atomicAdd(acc_out + c, a);
            }
        }
    }
    // ---------------- CSR passes ----------------
    for (int pass = 0; pass < npass; ++pass) {
        load_ptrs(pass + 2, a0nn, a1nn);
        load_elems(a0n, a1n, cn, vn);
        float s0 = 0.f, s1 = 0.f;
        {
            float xv[T];
#pragma unroll
            for (int t = 0; t < T; ++t) xv[t] = a0c + part + t * LPR < a1c ? xs_load<XT>(xs_u32, cc[t]) : 0.f;  // (padding: no gather)
#pragma unroll
            for (int t = 0; t < T; t += 2) { s0 = fmaf(vv[t], xv[t], s0); s1 = fmaf(vv[t + 1], xv[t + 1], s1); }
        }
        float tot = s0 + s1;
        for (int d = 1; d < LPR; d <<= 1) tot += __shfl_xor_sync(0xffffffffu, tot, d);
        // rows longer than T * LPR: the whole warp sums the remainder, row after row
        unsigned longm = __ballot_sync(0xffffffffu, part == 0 && a1c - a0c > T * LPR);
        while (longm) {
            const int i = __ffs(longm) - 1;
            longm &= longm - 1;
            const int b0 = __shfl_sync(0xffffffffu, a0c, i) + T * LPR, b1 = __shfl_sync(0xffffffffu, a1c, i);
            float a = 0.f, b = 0.f;
            for (int e = b0 + lane; e < b1; e += 128) {
                const int c0 = __ldg(p.cols + e), c1 = e + 32 < b1 ? __ldg(p.cols + e + 32) : 0, c2 = e + 64 < b1 ? __ldg(p.cols + e + 64) : 0,
                          c3 = e + 96 < b1 ? __ldg(p.cols + e + 96) : 0;
                const float v0 = __ldg(p.vals + e), v1 = e + 32 < b1 ? __ldg(p.vals + e + 32) : 0.f, v2 = e + 64 < b1 ? __ldg(p.vals + e + 64) : 0.f,
                            v3 = e + 96 < b1 ? __ldg(p.vals + e + 96) : 0.f;
                a = fmaf(v0, xs_load<XT>(xs_u32, c0), a);
                if (e + 32 < b1) b = fmaf(v1, xs_load<XT>(xs_u32, c1), b);
                if (e + 64 < b1) a = fmaf(v2, xs_load<XT>(xs_u32, c2), a);
                if (e + 96 < b1) b = fmaf(v3, xs_load<XT>(xs_u32, c3), b);
            }
            a = warp_sum(a + b);
            if (lane == i) tot += a;
        }
        const int row = r + pass * RPP + rslot;
        if constexpr (FUSED) {
            if (part == 0 && row < rb) st_relaxed_u64(p.ws_cbox + row, box_word(tot, boxtag));
        } else {
            if (part == 0 && row < rb && a1c > a0c) atomicAdd(acc_out + row, tot);
        }
        a0c = a0n; a1c = a1n; a0n = a0nn; a1n = a1nn;
#pragma unroll
        for (int t = 0; t < T; ++t) { cc[t] = cn[t]; vv[t] = vn[t]; }
    }
}

// The calling CTA's part of GEMV `p`: units [g0, g0 + len) of the strip-major [strip][unit] space, from unit r0 of strip s0, in nseg
// segments (a segment is the CTA's part of one strip).
struct Span {
    int g0, len, s0, r0, nseg;
    __device__ __forceinline__ explicit Span(const P2 &p) {
        const int R = p.R;
        g0 = min((int)blockIdx.x * p.chunk, p.T);
        const int g1 = min(g0 + p.chunk, p.T);
        len = g1 - g0;
        s0 = g0 / R;
        r0 = g0 - s0 * R;
        nseg = len > 0 ? (g1 - 1) / R - s0 + 1 : 0;
    }
};

// By one producer lane each: a 1/grid slice of the GEMV's look-up table and row pointers into L2.  A decode step finds none of a layer's
// arrays there, and the CTAs of a launch start at different times, so the late ones find what the early ones asked for.
template <int BITS>
__device__ __forceinline__ void warm_l2(const P2 &p, const int N, const int lane) {
    const int G = (int)gridDim.x;
    const size_t lut_lines = ((size_t)N * (1 << BITS) * 4 + 127) / 128, per = (lut_lines + G - 1) / G;
    for (size_t i = (size_t)blockIdx.x * per + lane; i < min(lut_lines, ((size_t)blockIdx.x + 1) * per); i += 32)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(p.lut) + 128 * i));
    if (p.rows) {
        const size_t row_lines = ((size_t)(N + 1) * 4 + 127) / 128, rper = (row_lines + G - 1) / G;
        for (size_t i = (size_t)blockIdx.x * rper + lane; i < min(row_lines, ((size_t)blockIdx.x + 1) * rper); i += 32)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(p.rows) + 128 * i));
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Strip finishing (fused mode), by the builder warps of lutgemv2_kernel and lutgemv_seq_kernel (thread bt = column bt of a strip).
// A strip is finished (converted to y) by the CTA in whose range it STARTS.  A CTA that only holds a later part of it (that can only
// be its first segment) hands its sums to that owner through its mailbox row (ws_hbox); the owner's own strip sums never leave the SM:
// sown[u][column] for the u-th owned strip (a strip inside one CTA is exactly one segment), SOWN of them, the rest through the global
// accumulator.  (The first round-2 build sent all of them through the global accumulator: a RED and, in the finishing pass, a load that
// had to wait for it - two L2 round trips between the last weight and y when the last segment is short.)
// A mailbox word carries the kernel's tag (box_word): 1 in lutgemv2_kernel, reset by the owner; the (token, GEMV) tag in the sequence
// kernel, never reset.  The finishing pass itself is one text, lutgemv_finish.inc, #included by both kernels (DESIGN §3.4).
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int SOWN = 8;
constexpr int FAST = 4;  // owned strips whose outlier-sum words the finishing pass requests ahead, before it needs them

// Strip sums of segment s (at `a` in shared memory, back to zero) -> the strip's owner; FUSED = false: one red.add per column.
// ofs = sp.r0 != 0 (segment s is owned strip s - ofs), given by the caller: the sequence kernel has it once per GEMV.
template <bool FUSED>
__device__ __forceinline__ void flush_strip(const P2 &p, const uint32_t a, const int s, const int ofs, const Span &sp, const int N,
                                            const uint32_t base, const int bt, float *const acc_out, const uint32_t tag) {
    const float v = lds_f32(a);
    sts_u32(a, 0u);
    const int strip = sp.s0 + s, col = strip * STRIP + bt;
    if constexpr (FUSED) {
        const uint32_t sown = base + OFF_FIN;   // float [SOWN][64]
        if (s == 0 && sp.r0 != 0) st_relaxed_u64(p.ws_hbox + (size_t)blockIdx.x * STRIP + bt, box_word(v, tag));
        else if (s - ofs < SOWN) sts_u32(sown + 4u * (uint32_t)((s - ofs) * STRIP + bt), __float_as_uint(v));
        else if (col < N) atomicAdd(acc_out + col, v);
    } else {
        if (col < N) atomicAdd(acc_out + col, v);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// The kernel.  MODE 0: exact fp32 table ; MODE 1: fp16 pair table (needs fp16 x).  XT: x's element type (float, __half or
// __nv_bfloat16), in which it is given and staged; a 16-bit y (p.y_is_half) is y16_t<XT>.
// ---------------------------------------------------------------------------------------------------------------------------
template <int BITS, int MODE, typename XT, bool FUSED>
__global__ void __launch_bounds__(THREADS2, 1) lutgemv2_kernel(const P2 p, const __grid_constant__ CUtensorMap tm_big,
                                                               const __grid_constant__ CUtensorMap tm_small,
                                                               const __grid_constant__ CUtensorMap tm_mid) {
    using C = G2<BITS, MODE>;
    using Y16 = y16_t<XT>;
    static_assert(MODE == 0 || std::is_same<XT, __half>::value, "the pair table multiplies fp16 by fp16: it needs fp16 x");
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    if (raw != p.smem_raw) __trap();  // the host planned the carve-up (table alignment) for another window address
    uint32_t base = (raw + 127u) & ~127u;
    asm volatile("mov.u32 %0, %0;" : "+r"(base));  // pinned: keeps the compiler from rematerialising it through S2UR
    unsigned char *sm = smem_raw + (base - raw);
    const uint32_t bar_u32 = base + OFF_BAR;
    const uint32_t xs_u32 = base + OFF_X;
    const int nstage = p.nstage;
    constexpr int NTB = 2;       // table buffers and strip accumulators: segment s uses s & 1
    constexpr int TFREE = 272;   // tfree[b] at bar_u32 + TFREE + 8b
    auto tab_of = [](int s) { return s & 1; };
    const Carve cv(base, (uint32_t)((p.K * (int)sizeof(XT) + 127) & ~127), 0u, C::TAB, NTB, C::STAGE, nstage);
    const uint32_t lo_base = cv.lo_base, tab0 = cv.tab0, hi_base = cv.hi_base;
    const int n_lo = cv.n_lo;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = p.N, R = p.R;
    const Span sp(p);
    const int len = sp.len, s0 = sp.s0, r0 = sp.r0, nseg = sp.nseg;

    TRACE(0, tid == 0);
    if (tid == 0) {
        for (int s = 0; s < nstage; ++s) {
            mbar_init(bar_u32 + 8 * s, 1);          // full: the producer's arrive.expect_tx
            mbar_init(bar_u32 + 128 + 8 * s, NWC);  // empty: one arrive per consumer warp
        }
        for (int b = 0; b < NTB; ++b) {
            mbar_init(bar_u32 + 256 + 8 * b, NBW);    // tfull: table b is built (one arrive per builder warp)
            mbar_init(bar_u32 + TFREE + 8 * b, NWC);  // tfree: every consumer warp is done with table b and has deposited its strip sums
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_launch_dependents();
    if (warp == WARP_PROD) {
        // Cold-start latencies (a decode step finds none of a layer's arrays in L2): ask for the tensor-map descriptors now, and pull this
        // CTA's slice of the look-up table and row pointers into L2 (the CTAs inherit their SM from the previous kernel's CTAs).
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_big)) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_small)) : "memory");
            if constexpr (C::ROT) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_mid)) : "memory");
        }
        warm_l2<BITS>(p, N, lane);
    }
    __syncthreads();
    float *const acc_out = FUSED ? p.ws_acc : reinterpret_cast<float *>(p.out);

    if (warp == WARP_PROD) {
        // =========================== TMA producer: weights never depend on the previous kernel ===========================
        // (Also tried: cp.async.bulk.prefetch.tensor into L2 16-24 stages ahead of the ring - slower on every shape, like the
        // L2 prefetch experiment of round 1.)
        const uint64_t pol = l2_evict_first_policy();
        const CUtensorMap *const tmap_big = &tm_big, *const tmap_small = &tm_small, *const tmap_mid = &tm_mid;
        int slot = 0;
        uint32_t ph = 0;
        bool refill = false;
        for (int seg = 0; seg < nseg; ++seg) {
#include "lutgemv_stream.inc"
        }
    } else if (warp >= WARP_SP) {
        sparse3<XT, FUSED>(p, base, warp - WARP_SP, lane, acc_out, 1u);
        TRACE(10, lane == 0);
    } else if (warp >= WARP_BLD) {
        // =========================== table builders (2 warps, thread = column slot) ===========================
        // Segment s uses table buffer s & 1 and strip accumulator s & 1; the loop over the segments is lutgemv_tables.inc.
        const int bt = tid - WARP_BLD * 32;
        const uint32_t lutbuf = base + OFF_LUT, sacc = base + OFF_SACC;
        sts_u32(sacc + 4 * bt, 0u);
        sts_u32(sacc + 4 * (STRIP + bt), 0u);
        bool dep_ok = false;
        auto dep_wait = [&]() { if (!dep_ok) { pdl_wait(); dep_ok = true; } };  // builders never read x: they only need this before writing
        const uint32_t sown = base + OFF_FIN;   // float [SOWN][64]
        auto sacc_of = [&](int s) { return sacc + 4 * ((s & 1) * STRIP + bt); };
        auto tfree_wait = [&](int s) { mbar_wait(bar_u32 + TFREE + 8 * (s & 1), (uint32_t)((s >> 1) & 1)); };
        auto reuse_wait = [&](int s) {  // the previous user of segment s's buffer: segment s - 2
            dep_wait();                 // from here on we write global memory: the previous kernel must be done
            mbar_wait(bar_u32 + TFREE + 8 * (s & 1), (uint32_t)(((s >> 1) - 1) & 1));
        };
        auto flush = [&](int s) { flush_strip<FUSED>(p, sacc_of(s), s, r0 != 0 ? 1 : 0, sp, N, base, bt, acc_out, 1u); };
        // The raw LUT rows of the first two strips are requested at once (one cold round trip, not two); later strips two ahead.
        if (nseg > 0) lut_prefetch<BITS>(p, lutbuf, s0, bt);
        if (nseg > 1) lut_prefetch<BITS>(p, lutbuf + LUTBUF, s0 + 1, bt);
#include "lutgemv_tables.inc"
        dep_wait();
        if constexpr (!FUSED) {
            for (int s = max(0, nseg - NTB); s < nseg; ++s) {  // the last two segments
                tfree_wait(s);
                flush(s);
            }
        } else {
            // the finishing pass (lutgemv_finish.inc): every mailbox word is written back to zero by its owner; no word per column
            // besides the mailboxes'; y is fp32 or y16_t, in this rank's vector or, with the exchange, in every rank's
            auto err_word = [&]() { return p.ws_cnt + 16; };
            constexpr uint32_t boxtag = 1u;
            constexpr bool box_keep = false;
            auto res_load = [](uint32_t *rw, uint32_t &, int, int, int) { for (int u = 0; u < FAST; ++u) rw[u] = 0u; };
            auto res_word = [](int) { return 0u; };
            auto make_store_y = [&]() {
                const int w = p.xw_world ? N / p.xw_members : 0;
                return [&, w](int col, float yv, uint32_t) {
                    if (p.bias) yv += __ldg(p.bias + col);
                    if (p.xw_world == 0) {
                        if (p.y_is_half) reinterpret_cast<Y16 *>(p.out)[col] = f32_to<Y16>(yv);
                        else reinterpret_cast<float *>(p.out)[col] = yv;
                    } else {
                        // local column col of the stacked shard = column j of member m; it lands at [m][rank*w + j] of the
                        // [members][n_full] vector in EVERY rank's arena
                        const int mm = col / w, j = col - mm * w;
                        const unsigned long long e = (unsigned long long)mm * p.xw_nfull + (unsigned long long)p.xw_rank * w + j;
                        for (int pr = 0; pr < p.xw_world; ++pr) {
                            unsigned char *dst = reinterpret_cast<unsigned char *>(__ldg(p.xw_base + pr) + p.xw_out_off);
                            if (p.y_is_half) *reinterpret_cast<Y16 *>(dst + 2 * e) = f32_to<Y16>(yv);
                            else *reinterpret_cast<float *>(dst + 4 * e) = yv;
                        }
                    }
                };
            };
#include "lutgemv_finish.inc"
            if (p.xw_world) {
                // exchange: every owning CTA publishes its stores on every rank (system-scope release); CTA 0 (it always owns strip 0)
                // then holds the grid open until every owning CTA of every rank has published on ours: when this grid completes, the
                // local vector is whole.  Counters only grow (expected arrivals so far live next to the flag).
                named_bar_sync(3, NBT);
                if (bt == 0) {
                    const unsigned long long self = __ldg(p.xw_base + p.xw_rank);
                    if (nown > 0) {
                        __threadfence_system();
                        for (int pr = 0; pr < p.xw_world; ++pr)
                            atomicAdd_system(reinterpret_cast<unsigned long long *>(__ldg(p.xw_base + pr) + p.xw_flag_off), 1ull);
                    }
                    if (blockIdx.x == 0) {
                        const unsigned long long target = *reinterpret_cast<volatile unsigned long long *>(self + p.xw_state_off) +
                                                          (unsigned long long)p.xw_world * p.nown_ctas;
                        unsigned long long seen, t0, t1;
                        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
                        const bool broken = *reinterpret_cast<volatile unsigned int *>(self + p.xw_err_off) != 0u;
                        if (!broken) do {
                            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(self + p.xw_flag_off) : "memory");
                            if (seen >= target) break;
                            __nanosleep(100);
                            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                            if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile unsigned int *>(self + p.xw_err_off) = 1u; break; }
                        } while (true);
                        *reinterpret_cast<volatile unsigned long long *>(self + p.xw_state_off) = target;
                    }
                }
            }
        }
        TRACE(9, bt == 0);
    } else {
        // =========================== consumers ===========================
        const int i16 = lane & 15, jsel = lane >> 4;
        TRACE(2, tid == 0);
        if (tid == 0) pdl_wait();  // everything below reads what the previous kernel may have produced (x)
        named_bar_sync(1, NCT);
        TRACE(3, tid == 0);
        {   // stage x whole, in its own type
            const int n16 = p.K * (int)sizeof(XT) / 16;
            for (int e = tid; e < n16; e += NCT) cp_async16(xs_u32 + 16 * e, reinterpret_cast<const unsigned char *>(p.x) + 16 * (size_t)e);
            cp_async_commit();
            cp_async_wait_all();
        }
        named_bar_sync(2, NCT + NSPW * 32);  // x visible to consumers and the sparse warp
        TRACE(4, tid == 0);

        Acc A;
#pragma unroll
        for (int t = 0; t < 4; ++t) A.a[t] = 0ull;
#pragma unroll
        for (int t = 0; t < 8; ++t) A.f[t] = 0.f;
        const uint32_t slotb[4] = {(uint32_t)((((0 ^ jsel) << 4) | i16) << 2), (uint32_t)((((1 ^ jsel) << 4) | i16) << 2),
                                   (uint32_t)((((2 ^ jsel) << 4) | i16) << 2), (uint32_t)((((3 ^ jsel) << 4) | i16) << 2)};
        const uint32_t sacc_lane = base + OFF_SACC + (4 * i16) * 4;
        auto sacc_row = [&](int b) { return sacc_lane + b * (STRIP * 4); };
        auto tab_phase = [](int s) { return (uint32_t)((s >> 1) & 1); };
        const uint32_t lane_in_stage = (uint32_t)((2 * warp + jsel) * C::UNIT + i16 * 16);
        int slot = 0;
        uint32_t par = 0;
        auto stage_of = [&](int sl) { return (sl < n_lo ? lo_base : hi_base) + sl * C::STAGE + lane_in_stage; };
        auto advance = [&]() { if (++slot == nstage) { slot = 0; par ^= 1u; } };
        for (int seg = 0; seg < nseg; ++seg) {
#include "lutgemv_segment.inc"
        }
        TRACE(6, tid == 0);
    }

    TRACE(11, tid == 0);
}

}  // namespace v2

}  // namespace
