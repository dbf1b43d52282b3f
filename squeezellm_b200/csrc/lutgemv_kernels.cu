// lutgemv_kernels.cu - H100 (sm_90a) dense-and-sparse LUT GEMV, written from scratch.
//
// Replaces (behaviour, not code) squeezellm/quant_cuda_kernel.cu of SqueezeAILab/SqueezeLLM:
//   VecQuant{3,4}MatMulKernelNUQPerChannel[Batched]  (:741-1038)   LUT GEMV
//   SPMV_ATOMIC[_BATCHED]                            (:1040-1089)  CSR outliers
//   DenseMatVecKernel[Batched]                       (:1092-1164)  topX dense rows
// and the 12 host launchers (:132-738), behind the C ABI of include/sqllm_b200.h.  Prefill-sized fp16 / bf16 inputs have a
// tensor-core LUT-GEMM of their own (lutgemm_tc.cuh, sqllm_lutgemm_fused_dt), a few fp16 / bf16 rows a multi-row GEMV with a cluster
// split-K (lutgemv_rows.cuh, sqllm_lutgemv_rows_dt).  The input gradient dx = dy . W^T has a transposed LUT-GEMM on the tensor cores
// (lutgemm_tc_t.cuh) and one on the CUDA cores (lutgemm_t.cuh), both behind sqllm_lutgemm_t.  The gradients of the codebook,
// the CSR values and the dense rows come from G = x^T . dy, bucketed by the packed indices: on the tensor cores
// (lut_grad_tc.cuh) or the CUDA cores (lut_grad.cuh), both behind sqllm_lut_grad.
//
// Two GEMV kernels live here.  lutgemv2_kernel (lutgemv_v2.cuh) runs every one-vector GEMV in the accumulate and the default
// (fast) fused mode, whatever its width: a layer narrower than one strip is a layer whose only strip is ragged.
// lutgemv_kernel below ("v1") is the kernel of the deterministic fused mode (sqllm_set_deterministic / SQLLM_DETERMINISTIC=1).
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
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint, no -lcuda)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>
#include <mutex>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "sqllm_b200.h"

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
constexpr int STRIP = 64;                 // output columns per strip (16 lanes x 4 columns)
constexpr int SU = 2 * NW;                // units per pipeline stage (one pair per consumer warp)
constexpr int CSR_CH = 1024;              // CSR elements staged per chunk
constexpr int STAGE = CSR_CH * 16;        // staging buffer: a chunk of CSR cols + vals (8 KB), then the dense-row partials (8 KB)
constexpr int MAX_TOPX_FUSED = SQLLM_FUSED_MAX_TOPX;
constexpr int HYB_R = 11;                 // dense rows: k-rows per lane slot requested before the dependency wait
constexpr int MAX_STRIPS = 16320;         // per-strip tickets in the workspace header (out_features <= 1,044,480)
constexpr int MAX_N_FUSED = SQLLM_FUSED_MAX_OUT;  // fused path: the scratch accumulator lives at a fixed place in the workspace
constexpr size_t WS_ACC_OFF = 65536;       // [64 KB, 64 KB + 4*MAX_N_FUSED): fp32 accumulator (zero between launches)
constexpr int MAX_GRID_V2 = 256;           // v2 runs one CTA per SM
constexpr size_t WS_HBOX_OFF = WS_ACC_OFF + (size_t)MAX_N_FUSED * 4;       // v2 mailboxes: [MAX_GRID_V2][64] x 8 bytes (partial strip sums)
constexpr size_t WS_CBOX_OFF = WS_HBOX_OFF + (size_t)MAX_GRID_V2 * 64 * 8;  // ... and [MAX_N_FUSED] x 8 bytes (outlier row sums); zero between launches
constexpr size_t WS_DBOX_OFF = WS_CBOX_OFF + (size_t)MAX_N_FUSED * 8;          // ... and [MAX_TOPX_FUSED][MAX_GRID_V2] x 8 bytes (dense-row parts, one per contributing CTA)
constexpr size_t WS_HEADER = WS_DBOX_OFF + (size_t)MAX_TOPX_FUSED * MAX_GRID_V2 * 8;  // tickets + accumulator + mailboxes: never shared with data of any shape

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

// ---- small PTX helpers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float lds_f32(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ float4 lds_v4(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ uint4 lds_u4(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ uint4 ldg_stream(const void *p) {  // read-once weights: no L1 allocation
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16_clip(uint32_t dst, const void *src, int src_bytes) {  // reads src_bytes (<= 16), zero-fills the rest
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_pending() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
// Two fp32 FMAs on a register pair.  Hopper has no packed fp32 FMA, so each half is one fma.rn.f32: the same rounding,
// lane for lane, as a packed instruction would give, and the pair keeps two independent accumulation chains per column.
__device__ __forceinline__ void ffma2(uint64_t &acc, uint64_t a, uint64_t b) {
    asm("{\n.reg .f32 a0, a1, b0, b1, c0, c1;\n"
        "mov.b64 {a0, a1}, %1;\nmov.b64 {b0, b1}, %2;\nmov.b64 {c0, c1}, %0;\n"
        "fma.rn.f32 c0, a0, b0, c0;\nfma.rn.f32 c1, a1, b1, c1;\n"
        "mov.b64 %0, {c0, c1};\n}" : "+l"(acc) : "l"(a), "l"(b));
}
__device__ __forceinline__ float sum2(uint64_t v) {
    float lo, hi;
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
    return lo + hi;
}
// Element types of x in the GEMV kernels: float, __half or __nv_bfloat16.  A 16-bit y has x's 16-bit type (fp16 for fp32 x).
template <typename XT> constexpr bool x_is16 = !std::is_same<XT, float>::value;
template <typename XT> using y16_t = typename std::conditional<std::is_same<XT, __nv_bfloat16>::value, __nv_bfloat16, __half>::type;
template <typename T> __device__ __forceinline__ T f32_to(float v);
template <> __device__ __forceinline__ __half f32_to<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 f32_to<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
// the two bf16 values of a word (lo, hi) as fp32, exactly: a bf16 is the upper half of its fp32 (one shift, one mask)
__device__ __forceinline__ float2 bf16x2_to_f32x2(uint32_t h) { return make_float2(__uint_as_float(h << 16), __uint_as_float(h & 0xFFFF0000u)); }
// ... and of either 16-bit type
template <typename XT>
__device__ __forceinline__ float2 x16x2_to_f32x2(uint32_t h) {
    if constexpr (std::is_same<XT, __nv_bfloat16>::value) return bf16x2_to_f32x2(h);
    else return __half22float2(*reinterpret_cast<const __half2 *>(&h));
}
__device__ __forceinline__ float warp_sum(float v) {  // fixed xor tree -> deterministic
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}
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
#ifdef SQLLM_TRACE
__device__ __forceinline__ void trace_mark(unsigned long long *trace, int slot) {
    if (trace) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        trace[(size_t)blockIdx.x * 32 + slot] = t;
    }
}
#define TRACE(slot, cond) do { if (cond) trace_mark(p.trace, slot); } while (0)
#else
#define TRACE(slot, cond) do { } while (0)
#endif

// mbarrier / TMA bulk copy / PDL
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_tile2d_g2s(uint32_t dst, const CUtensorMap *map, int col, int row, uint32_t bar, uint64_t pol) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;"
                 ::"r"(dst), "l"(map), "r"(col), "r"(row), "r"(bar), "l"(pol) : "memory");
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
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

// =================================================================================================
// 3-bit: one group = 3 words per column = 32 inputs (10 | straddler | 10 | straddler | 10), the layout
// of squeezellm/quant.py:185-203.  Each index is moved to bits 8..10 (table row stride 256 B) by one
// shift (a funnel shift for the two straddlers) and merged with the lane's slot address by one LOP3.
// =================================================================================================
template <int SH>  // field at bit position SH of w -> bits 8..10
__device__ __forceinline__ uint32_t fld(uint32_t w) {
    if constexpr (SH < 8) return w << (8 - SH);
    else if constexpr (SH == 8) return w;
    else return w >> (SH - 8);
}
#define LK3(dst, word_expr, lsv) dst = lds_f32((((word_expr)) & 0x700u) | (lsv))

__device__ __forceinline__ void consume3_col(const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t lsv,
                                             const uint64_t (&xp)[16], uint64_t &acc) {
    float a, b;
    // inputs 0..9 from w0 (bits 3k), 10 straddles w0/w1
    LK3(a, fld<0>(w0), lsv);  LK3(b, fld<3>(w0), lsv);  ffma2(acc, pack2(a, b), xp[0]);
    LK3(a, fld<6>(w0), lsv);  LK3(b, fld<9>(w0), lsv);  ffma2(acc, pack2(a, b), xp[1]);
    LK3(a, fld<12>(w0), lsv); LK3(b, fld<15>(w0), lsv); ffma2(acc, pack2(a, b), xp[2]);
    LK3(a, fld<18>(w0), lsv); LK3(b, fld<21>(w0), lsv); ffma2(acc, pack2(a, b), xp[3]);
    LK3(a, fld<24>(w0), lsv); LK3(b, fld<27>(w0), lsv); ffma2(acc, pack2(a, b), xp[4]);
    LK3(a, __funnelshift_r(w0, w1, 22), lsv);            // input 10: bits 30,31 of w0 + bit 0 of w1
    LK3(b, fld<1>(w1), lsv);                             // input 11
    ffma2(acc, pack2(a, b), xp[5]);
    LK3(a, fld<4>(w1), lsv);  LK3(b, fld<7>(w1), lsv);  ffma2(acc, pack2(a, b), xp[6]);
    LK3(a, fld<10>(w1), lsv); LK3(b, fld<13>(w1), lsv); ffma2(acc, pack2(a, b), xp[7]);
    LK3(a, fld<16>(w1), lsv); LK3(b, fld<19>(w1), lsv); ffma2(acc, pack2(a, b), xp[8]);
    LK3(a, fld<22>(w1), lsv); LK3(b, fld<25>(w1), lsv); ffma2(acc, pack2(a, b), xp[9]);
    LK3(a, fld<28>(w1), lsv);                            // input 20
    LK3(b, __funnelshift_r(w1, w2, 23), lsv);            // input 21: bit 31 of w1 + bits 0,1 of w2
    ffma2(acc, pack2(a, b), xp[10]);
    LK3(a, fld<2>(w2), lsv);  LK3(b, fld<5>(w2), lsv);  ffma2(acc, pack2(a, b), xp[11]);
    LK3(a, fld<8>(w2), lsv);  LK3(b, fld<11>(w2), lsv); ffma2(acc, pack2(a, b), xp[12]);
    LK3(a, fld<14>(w2), lsv); LK3(b, fld<17>(w2), lsv); ffma2(acc, pack2(a, b), xp[13]);
    LK3(a, fld<20>(w2), lsv); LK3(b, fld<23>(w2), lsv); ffma2(acc, pack2(a, b), xp[14]);
    LK3(a, fld<26>(w2), lsv); LK3(b, fld<29>(w2), lsv); ffma2(acc, pack2(a, b), xp[15]);
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

// test hook: unpack exactly like the GEMV path (same shift/mask expressions)
__global__ void unpack_kernel(int bits, const uint32_t *__restrict__ q, int K, int N, uint8_t *__restrict__ idx) {
    const size_t n = (size_t)K * N;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(e / N), c = (int)(e % N);
        uint32_t v;
        if (bits == 4) {
            const uint32_t w = q[(size_t)(k >> 3) * N + c];
            const int n8 = k & 7;
            const uint32_t EO = (n8 & 1) ? ((w >> 4) & 0x0F0F0F0Fu) : (w & 0x0F0F0F0Fu);
            v = __byte_perm(EO, 0u, 0x4440 | (n8 >> 1)) & 0xFFu;
        } else {
            const int g = k >> 5, j = k & 31;
            const uint32_t *pq = q + (size_t)(3 * g) * N + c;
            const uint32_t w0 = pq[0], w1 = pq[N], w2 = pq[2 * (size_t)N];
            uint32_t f;  // field moved to bits 8..10, as in consume3_col
            if (j < 10) f = (3 * j < 8) ? (w0 << (8 - 3 * j)) : (w0 >> (3 * j - 8));
            else if (j == 10) f = __funnelshift_r(w0, w1, 22);
            else if (j < 21) { const int s = 1 + 3 * (j - 11); f = (s < 8) ? (w1 << (8 - s)) : (w1 >> (s - 8)); }
            else if (j == 21) f = __funnelshift_r(w1, w2, 23);
            else { const int s = 2 + 3 * (j - 22); f = (s < 8) ? (w2 << (8 - s)) : (w2 >> (s - 8)); }
            v = (f & 0x700u) >> 8;
        }
        idx[e] = (uint8_t)v;
    }
}

#include "lutgemv_v2.cuh"
#include "lutgemv_seq.cuh"
#include "lutgemm_batched.cuh"
#include "lutgemv_rows.cuh"
#include "lutgemm_tc.cuh"
#include "lutgemm_t.cuh"
#include "lutgemm_tc_t.cuh"
#include "lut_grad.cuh"
#include "lut_grad_tc.cuh"
#include "fisher.cuh"
#include "kmeans1d.cuh"
#include "dequant.cuh"

// shared-window address at which a kernel without static shared memory sees its dynamic shared memory (the v2 carve-up aligns
// tables to their own size - up to 64 KB - so the host needs the real address, not a worst case; the kernel re-checks it)
__global__ void smem_base_probe(unsigned *out) {
    extern __shared__ unsigned char probe_smem[];
    *out = smem_u32(probe_smem);
}

// =================================================================================================
// Host side
// =================================================================================================
thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

// Process-wide state (mode switches, lazily read environment knobs, per-device state) is guarded by g_state_mu: the entry
// points may be called from several host threads.  Switching a mode (sqllm_set_deterministic / sqllm_set_lut_mode) while other
// threads are launching is allowed but takes effect per call; do not switch while a CUDA graph that should keep the old mode is
// being captured.
std::recursive_mutex g_state_mu;

struct DevInfo {
    int sm = 0;
    unsigned smem_raw = 0;               // shared-window address of dynamic shared memory; 0 until smem_window probes it
    std::vector<const void *> smem_set;  // kernels whose dynamic shared-memory limit dev_setup has raised
};
DevInfo g_dev[64];

// d.smem_raw from smem_base_probe, once per device.  The probe is synchronous and refused during stream capture: only v2 and sequence
// plans ask for it, and the first of them on a device must come before any capture - any warm-up does.  Caller holds g_state_mu.
int smem_window(DevInfo &d) {
    if (d.smem_raw) return SQLLM_OK;
    unsigned *d_out = nullptr, h_out = 0;
    cudaError_t pe = cudaMalloc(&d_out, sizeof(unsigned));
    if (pe == cudaSuccess) {
        smem_base_probe<<<1, 1, 1024>>>(d_out);
        pe = cudaMemcpy(&h_out, d_out, sizeof(unsigned), cudaMemcpyDeviceToHost);
        cudaFree(d_out);
    }
    if (pe != cudaSuccess || h_out == 0) {
        cudaGetLastError();
        return fail(SQLLM_ECUDA, "shared-memory probe failed (first call inside a stream capture? run one call before capturing): %s", cudaGetErrorString(pe));
    }
    d.smem_raw = h_out;
    return SQLLM_OK;
}

// A kernel and the dynamic shared memory it is launched with.
struct KernelSmem {
    const void *fn = nullptr;
    int bytes = 0;
    KernelSmem() = default;
    template <typename... P>
    KernelSmem(void (*f)(P...), int b) : fn((const void *)f), bytes(b) {}
};

// The device set-up of every launch, under g_state_mu: resolves the current device (its SM count is read once), raises the dynamic
// shared-memory limit of each kernel in `ks` (once per device), and returns the SM count in *sm and the shared-memory window in
// *smem_raw where asked (the window is probed on the first request, see smem_window).  `ks` is a braced list of KernelSmem, or an array.
template <typename List = std::initializer_list<KernelSmem>>
int dev_setup(const List &ks, int *sm = nullptr, unsigned *smem_raw = nullptr) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(SQLLM_ECUDA, "cudaGetDevice failed");
    if (dev < 0 || dev >= 64) return fail(SQLLM_EINVAL, "device ordinal %d out of range", dev);
    DevInfo &d = g_dev[dev];
    if (d.sm == 0 && (cudaDeviceGetAttribute(&d.sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sm <= 0)) {
        d.sm = 0;
        return fail(SQLLM_ECUDA, "cannot query SM count");
    }
    for (const KernelSmem &k : ks) {
        if (std::find(d.smem_set.begin(), d.smem_set.end(), k.fn) != d.smem_set.end()) continue;
        if (cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.bytes) != cudaSuccess)
            return fail(SQLLM_ECUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError()));
        d.smem_set.push_back(k.fn);
    }
    if (smem_raw) {
        const int rc = smem_window(d);
        if (rc) return rc;
        *smem_raw = d.smem_raw;
    }
    if (sm) *sm = d.sm;
    return SQLLM_OK;
}

// The one attribute of a cudaLaunchKernelEx launch: programmatic stream serialisation for the GEMV kernels that wait on the grid
// dependency (their prologue and weight stream overlap the previous kernel), cooperative for the sequence kernel (every CTA waits on
// every other one: they must all be resident), or a cluster of `cluster` CTAs along x for the kernels whose CTAs reduce through each
// other's shared memory.
struct LaunchAttr {
    int cluster;
    bool cooperative;
};
constexpr LaunchAttr PDL{0, false}, COOPERATIVE{0, true};
constexpr LaunchAttr cluster_of(int n) { return {n, false}; }

template <typename... P, typename... A>
cudaError_t launch_ex(void (*fn)(P...), dim3 grid, int block, int smem, cudaStream_t st, LaunchAttr la, const A &...args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr;
    if (la.cluster > 0) {
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = la.cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    } else if (la.cooperative) {
        attr.id = cudaLaunchAttributeCooperative;
        attr.val.cooperative = 1;
    } else {
        attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr.val.programmaticStreamSerializationAllowed = 1;
    }
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, fn, args...);
}

// The layer's buffers in a kernel's parameter struct (every one names them qw, lut, rows, cols, vals, full_rows, fri, topX): the
// dense rows only when both full_rows and topX > 0 are given, so that p.topX > 0 means "the layer has dense rows".
template <typename P>
void set_layer(P &p, const sqllm_lutgemv_args &a) {
    const bool hyb = a.full_rows && a.topX > 0;
    p.qw = reinterpret_cast<const uint32_t *>(a.qweight);
    p.lut = a.lookup_table;
    p.rows = a.rows; p.cols = a.cols; p.vals = a.vals;
    p.full_rows = hyb ? a.full_rows : nullptr;
    p.fri = hyb ? a.full_row_indices : nullptr;
    p.topX = hyb ? a.topX : 0;
}

// SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16
bool dt_valid(int dt) { return dt == SQLLM_DT_F32 || dt == SQLLM_DT_F16 || dt == SQLLM_DT_BF16; }
// the (x, y) dtype pairs of the one-GEMV entry points (sqllm_lutgemv_fused_dt, sqllm_lutgemv_fused_exchange_dt): y is fp32 or the
// 16-bit type of x, and that is fp16 for fp32 x
bool fused_dt_pair(int x_dt, int y_dt) {
    const int y16 = x_dt == SQLLM_DT_BF16 ? SQLLM_DT_BF16 : SQLLM_DT_F16;
    return dt_valid(x_dt) && (y_dt == SQLLM_DT_F32 || y_dt == y16);
}
int fused_dt_fail(int x_dt, int y_dt) {
    return fail(SQLLM_EINVAL, "x_dtype=%d, y_dtype=%d: x must be SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16, y SQLLM_DT_F32 or the "
                              "16-bit type of x (SQLLM_DT_F16 for fp32 x)", x_dt, y_dt);
}

// The descriptor checks every GEMV / GEMM entry point shares, in this order: in_features a positive multiple of k_mult (64 or 32),
// out_features a positive multiple of n_mult (4, or 1 for "positive"), the packed matrix and codebook given, and dense rows only with
// their indices.  Each entry point makes its own checks after these.
int check_layer(const sqllm_lutgemv_args *a, int k_mult, int n_mult) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    if (a->bits != 3 && a->bits != 4) return fail(SQLLM_EINVAL, "bits must be 3 or 4 (got %d)", a->bits);
    if (a->in_features <= 0 || a->in_features % k_mult)
        return fail(SQLLM_EINVAL, "in_features=%d must be a positive multiple of %d", a->in_features, k_mult);
    if (a->out_features <= 0 || a->out_features % n_mult) {
        if (n_mult == 1) return fail(SQLLM_EINVAL, "out_features=%d must be positive", a->out_features);
        return fail(SQLLM_EINVAL, "out_features=%d must be a positive multiple of %d", a->out_features, n_mult);
    }
    if (!a->qweight || !a->lookup_table) return fail(SQLLM_EINVAL, "qweight / lookup_table must not be null");
    if (a->topX < 0) return fail(SQLLM_EINVAL, "topX < 0");
    if (a->full_rows && a->topX > 0 && !a->full_row_indices) return fail(SQLLM_EINVAL, "full_rows given without full_row_indices");
    return SQLLM_OK;
}

int g_det = -1;
int det_mode() {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    if (g_det < 0) { const char *e = getenv("SQLLM_DETERMINISTIC"); g_det = (e && e[0] == '1') ? 1 : 0; }
    return g_det;
}
// g_det - fused mode: 1 = v1, deterministic per-strip tickets (SQLLM_DETERMINISTIC=1 or sqllm_set_deterministic), 0 = v2 (default)
int g_last_grid = 0;
unsigned long long *g_trace = nullptr;
size_t g_trace_stride = 0;

// ---- 2-D tensor maps for the packed matrix (one per (pointer, shape, box)), created through the driver entry point ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct TmKey {
    const void *ptr; int rows, cols, box_rows;
    bool operator==(const TmKey &o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows; }
};
struct TmHash {
    size_t operator()(const TmKey &k) const {
        return std::hash<const void *>()(k.ptr) ^ ((size_t)k.rows * 1000003u) ^ ((size_t)k.cols * 10007u) ^ (size_t)k.box_rows;
    }
};
std::mutex g_tm_mutex;
std::unordered_map<TmKey, CUtensorMap, TmHash> g_tm_cache;
EncodeTiledFn g_encode = nullptr;

int get_tensor_map(const void *qweight, int rows, int cols, int box_rows, CUtensorMap &out) {
    std::lock_guard<std::mutex> lock(g_tm_mutex);
    const TmKey key{qweight, rows, cols, box_rows};
    auto it = g_tm_cache.find(key);
    if (it != g_tm_cache.end()) { out = it->second; return SQLLM_OK; }
    if (!g_encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
            return fail(SQLLM_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
        g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    }
    const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)cols * 4};
    const cuuint32_t box[2] = {(cuuint32_t)STRIP, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    const CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<void *>(qweight), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(SQLLM_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    if (g_tm_cache.size() > 8192) g_tm_cache.clear();
    g_tm_cache.emplace(key, m);
    out = m;
    return SQLLM_OK;
}

struct Plan {
    int R, strips, T, chunk, G, maxc, hc, hrows, smem, maxseg, x_direct, xfloats;
    size_t ws_cnt_off, ws_hyb_off, ws_part_off, ws_csr_off, ws_bytes;
    int csr_rpc, has_stage;
};

// stage: bytes of the shared-memory staging buffer when the layer has CSR outliers or dense rows: STAGE for a launch (smaller only
// in sqllm_workspace_bytes)
int make_plan(int bits, int K, int N, int topX, bool has_csr_in, int stage, Plan &pl) {
    std::lock_guard<std::recursive_mutex> state_lock(g_state_mu);  // lazily initialised statics below
    const bool has_csr = has_csr_in || topX > 0;  // from here on: "a staging buffer is needed"
    pl.has_stage = has_csr ? stage : 0;
    int sm = 0;
    const int rc = dev_setup({{lutgemv_kernel<4>, 227 * 1024}, {lutgemv_kernel<3>, 227 * 1024}}, &sm);
    if (rc) return rc;
    const int XU = bits == 4 ? 8 : 32;
    pl.R = bits == 4 ? K / 8 : K / 32;
    pl.strips = (N + STRIP - 1) / STRIP;
    const long long T = (long long)pl.strips * pl.R;
    if (T > 0x3fffffff) return fail(SQLLM_EINVAL, "problem too large");
    pl.T = (int)T;
    if (pl.strips > MAX_STRIPS || N > MAX_N_FUSED) return fail(SQLLM_EINVAL, "out_features=%d exceeds the workspace header (max %d)", N, MAX_N_FUSED);

    // One wave: a plan whose shared memory lets fewer than CTAS_PER_SM CTAs onto an SM would run a second one.  Plan for
    // CTAS_PER_SM, ask the occupancy calculator, and fall back to fewer CTAs per SM if it disagrees.
    int use_cps = CTAS_PER_SM;
replan:
    const int G0 = sm * use_cps;
    int chunk = (int)(2 * ((T + 2LL * G0 - 1) / (2LL * G0)));  // an even number of units: a consumer warp's pair never straddles the end
    if (chunk > 3 * pl.R) chunk = 3 * pl.R;  // a CTA may touch at most MAXSEG strips
    if (chunk < 2) chunk = 2;
    int maxseg = (chunk - 2) / pl.R + 2;      // worst case over start offsets (even offsets, even R)
    if (maxseg > MAXSEG) maxseg = MAXSEG;
    const bool direct = (long long)chunk * XU >= K;
    const int xfl = direct ? K : chunk * XU;
    pl.x_direct = direct ? 1 : 0;
    const int smem = bits == 4 ? Cfg<4>::total(maxseg, xfl, pl.has_stage) : Cfg<3>::total(maxseg, xfl, pl.has_stage);
    if (smem > 227 * 1024) return fail(SQLLM_EINVAL, "in_features=%d needs %d B of shared memory (> 227 KB)", K, smem);
    {
        static std::unordered_map<unsigned long long, int> occ_cache;
        const unsigned long long key = ((unsigned long long)smem << 8) | (unsigned long long)bits;
        int occ = -1;
        auto it = occ_cache.find(key);
        if (it != occ_cache.end()) occ = it->second;
        if (occ < 0) {
            const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bits == 4 ? lutgemv_kernel<4> : lutgemv_kernel<3>, THREADS, smem);
            if (e != cudaSuccess) return fail(SQLLM_ECUDA, "occupancy query failed: %s", cudaGetErrorString(e));
            occ_cache[key] = occ;
        }
        if (occ < 1) return fail(SQLLM_EINVAL, "kernel does not fit an SM (shared memory %d B)", smem);
        if (occ < use_cps) { use_cps = occ; goto replan; }
    }
    pl.smem = smem;
    pl.maxseg = maxseg;
    pl.xfloats = xfl;
    pl.chunk = chunk;
    pl.G = (int)((T + chunk - 1) / chunk);
    pl.maxc = (pl.R - 1) / chunk + 2;
    pl.hc = 0;
    pl.hrows = 0;
    int hc = 0;
    if (topX > 0) {
        // dense-row contributors: as few k-rows per CTA as the grid allows, down to what one warp requests before the dependency
        // wait (HYB_R steps of 32/topX rows), and no more partials (hc*topX floats) than the 2*CSR_CH-float staging buffer of the
        // finisher holds
        const int rows_pre = HYB_R * (topX <= 32 ? 32 / topX : 1);
        hc = std::min({pl.G, (K + rows_pre - 1) / rows_pre, 2 * CSR_CH / topX});
        if (hc < 1) hc = 1;
        pl.hrows = (K + hc - 1) / hc;
        pl.hc = (K + pl.hrows - 1) / pl.hrows;
    }
    pl.csr_rpc = (N + pl.G - 1) / pl.G;
    if (pl.csr_rpc < 1) pl.csr_rpc = 1;
    // Fixed header: [256, 256+4*MAX_STRIPS) per-strip tickets.  Tickets must never share bytes with data regions of ANY shape
    // (the workspace is reused across layers of different sizes).
    size_t off = WS_HEADER;
    pl.ws_cnt_off = 256;
    pl.ws_hyb_off = off; off += (size_t)hc * topX * 4;
    off = (off + 255) & ~(size_t)255;
    pl.ws_part_off = off; off += (size_t)pl.strips * pl.maxc * STRIP * 4;
    off = (off + 255) & ~(size_t)255;
    pl.ws_csr_off = off; off += (size_t)N * 4;
    pl.ws_bytes = off;
    return SQLLM_OK;
}

// the descriptor checks of sqllm_lutgemv, the fused one-GEMV entry points and the sequence: the shared ones with in_features a
// multiple of 64 and out_features a multiple of 4, then a 16-byte aligned matrix and codebook
int check_common(const sqllm_lutgemv_args *a) {
    const int rc = check_layer(a, 64, 4);
    if (rc) return rc;
    if (reinterpret_cast<uintptr_t>(a->qweight) & 15) return fail(SQLLM_EINVAL, "qweight must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(a->lookup_table) & 15) return fail(SQLLM_EINVAL, "lookup_table must be 16-byte aligned");
    return SQLLM_OK;
}

int launch(const sqllm_lutgemv_args *a, const Plan &pl, Params &p, cudaStream_t st) {
    std::lock_guard<std::recursive_mutex> state_lock(g_state_mu);
    set_layer(p, *a);
    p.K = a->in_features; p.N = a->out_features;
    p.R = pl.R; p.strips = pl.strips; p.T = pl.T; p.chunk = pl.chunk;
    p.maxseg = pl.maxseg; p.x_direct = pl.x_direct; p.xfloats = pl.xfloats;
    p.hc = p.topX > 0 ? pl.hc : 0; p.hrows = pl.hrows; p.maxc = pl.maxc;
    p.has_stage = pl.has_stage;
    p.csr_rpc = pl.csr_rpc;
    p.csr_al16 = (a->rows && ((reinterpret_cast<uintptr_t>(a->cols) | reinterpret_cast<uintptr_t>(a->vals)) & 15) == 0) ? 1 : 0;
    p.trace = g_trace;
    if (g_trace) g_trace += g_trace_stride;
    g_last_grid = pl.G;
    const cudaError_t e = launch_ex(a->bits == 4 ? lutgemv_kernel<4> : lutgemv_kernel<3>, pl.G, THREADS, pl.smem, st, PDL, p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}


// =================================================================================================
// v2 (lutgemv_v2.cuh): plan + launch.  One CTA per SM; all process-wide state behind one mutex / atomics.
// =================================================================================================
int g_lut_mode = -1;     // 0: exact fp32 table, 1: fp16 pair table when x is fp16 (SQLLM_LUT_MODE=fp16 / sqllm_set_lut_mode)

int lut_mode() {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    if (g_lut_mode < 0) {
        const char *e = getenv("SQLLM_LUT_MODE");
        g_lut_mode = (e && (!strcmp(e, "fp16") || !strcmp(e, "pair") || !strcmp(e, "1"))) ? 1 : 0;
    }
    return g_lut_mode;
}

typedef void (*K2)(const v2::P2, const CUtensorMap, const CUtensorMap);
struct K2Info { K2 fn; int tab, stage; };
// fused: variant 0: exact, fp32 x ; 1: exact, fp16 x ; 2: fp16 pair table, fp16 x ; 3: exact, bf16 x.  Accumulate mode (the 12
// symbols): variant 0 only.
constexpr int K2_VARIANTS = 4;
K2Info k2_lookup(int bits, int variant, bool fused) {
#define K2E(B, M, XT, F) K2Info{v2::lutgemv2_kernel<B, M, XT, F>, v2::C2<B, M>::TAB, v2::C2<B, M>::STAGE}
    if (bits == 4) {
        if (!fused) return K2E(4, 0, float, false);
        if (variant == 0) return K2E(4, 0, float, true);
        if (variant == 1) return K2E(4, 0, __half, true);
        if (variant == 3) return K2E(4, 0, __nv_bfloat16, true);
        return K2E(4, 1, __half, true);
    }
    if (!fused) return K2E(3, 0, float, false);
    if (variant == 0) return K2E(3, 0, float, true);
    if (variant == 1) return K2E(3, 0, __half, true);
    if (variant == 3) return K2E(3, 0, __nv_bfloat16, true);
    return K2E(3, 1, __half, true);
#undef K2E
}

// Stream-K plan of one layer for the v2 and sequence kernels, on a grid of at most `sm` CTAs, and the layer's buffers: fills the
// shape and buffer fields of p and returns the grid in G.
int plan_layer(const sqllm_lutgemv_args &a, int sm, v2::P2 &p, int &G) {
    const int K = a.in_features, N = a.out_features;
    set_layer(p, a);
    p.K = K; p.N = N;
    p.R = a.bits == 4 ? K / 8 : K / 32;
    p.strips = (N + STRIP - 1) / STRIP;
    const long long T = (long long)p.strips * p.R;
    if (T > 0x3fffffff) return fail(SQLLM_EINVAL, "problem too large");
    p.T = (int)T;
    p.chunk = std::max(2, (int)(2 * ((T + 2LL * sm - 1) / (2LL * sm))));
    G = (int)((T + p.chunk - 1) / p.chunk);
    p.csr_rpc = (N + G - 1) / G;
    p.hc = p.hrows = 0;
    if (p.topX > 0) {
        p.hrows = (K + G - 1) / G;
        p.hc = (K + p.hrows - 1) / p.hrows;
    }
    return SQLLM_OK;
}

// The two tensor maps over the packed matrix: 64 columns x (32 units | 2 units) boxes.
int tensor_maps(const sqllm_lutgemv_args &a, CUtensorMap &big, CUtensorMap &small) {
    const int rows_per_unit = a.bits == 4 ? 1 : 3, qrows = a.in_features / 32 * a.bits;
    // (a matrix shorter than one full stage never issues the big box; its map is clamped so that the encoder accepts it)
    const int rc = get_tensor_map(a.qweight, qrows, a.out_features, qrows < v2::SU2 * rows_per_unit ? 2 * rows_per_unit : v2::SU2 * rows_per_unit, big);
    return rc ? rc : get_tensor_map(a.qweight, qrows, a.out_features, 2 * rows_per_unit, small);
}

int launch2(const sqllm_lutgemv_args *a, int variant, bool fused, v2::P2 &p, cudaStream_t st) {
    const K2Info ki = k2_lookup(a->bits, variant, fused);
    KernelSmem all[2 * (1 + K2_VARIANTS)];  // every v2 kernel: accumulate mode and each fused variant, both widths
    int nk = 0;
    for (int b = 3; b <= 4; ++b) {
        all[nk++] = {k2_lookup(b, 0, false).fn, 227 * 1024};
        for (int v = 0; v < K2_VARIANTS; ++v) all[nk++] = {k2_lookup(b, v, true).fn, 227 * 1024};
    }
    int sm = 0;
    unsigned raw = 0;
    int rc = dev_setup(all, &sm, &raw);
    if (rc) return rc;
    int G = 0;
    if ((rc = plan_layer(*a, sm, p, G))) return rc;
    if (fused && p.N > MAX_N_FUSED) return fail(SQLLM_EINVAL, "out_features=%d exceeds the fused accumulator (max %d)", p.N, MAX_N_FUSED);
    if (fused && G > MAX_GRID_V2) return fail(SQLLM_EINVAL, "grid of %d CTAs exceeds the mailbox area (%d)", G, MAX_GRID_V2);
    const unsigned base = (raw + 127u) & ~127u;
    const unsigned xbytes = (unsigned)((p.K * (variant == 0 ? 4 : 2) + 127) & ~127);  // this layer's x, in its own dtype
    // one GEMV: the ring needs no more stages than the CTA's chunk fills
    const int n = v2::Carve(base, xbytes, 0u, ki.tab, 2, ki.stage, 0).depth(raw, 227 * 1024, ki.stage, (p.chunk + v2::SU2 - 1) / v2::SU2 + 1);
    if (n < 0) return fail(SQLLM_EINVAL, "in_features=%d does not fit the shared-memory carve-up of this table mode", p.K);
    if (n < 2) return fail(SQLLM_EINVAL, "in_features=%d leaves no room for a weight ring in shared memory", p.K);
    const int smem = (int)(v2::Carve(base, xbytes, 0u, ki.tab, 2, ki.stage, n).end - raw);
    p.nstage = n;
    p.smem_raw = raw;
    p.nown_ctas = 0;
    if (p.xw_world)
        for (int b = 0; b < G; ++b) {  // CTAs in whose range at least one strip starts
            const long long c0 = (long long)b * p.chunk, c1 = std::min<long long>(p.T, c0 + p.chunk);
            if ((c0 + p.R - 1) / p.R < (c1 + p.R - 1) / p.R) ++p.nown_ctas;
        }
    {
        std::lock_guard<std::recursive_mutex> lk(g_state_mu);
        p.trace = g_trace;
        if (g_trace) g_trace += g_trace_stride;
        g_last_grid = G;
    }
    CUtensorMap tm_big, tm_small;
    if ((rc = tensor_maps(*a, tm_big, tm_small))) return rc;
    const cudaError_t e = launch_ex(ki.fn, G, v2::THREADS2, smem, st, PDL, p, tm_big, tm_small);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}


// ---- sequences (lutgemv_seq.cuh): plan + descriptors at create time, two launches per run -----------------------------
typedef void (*KSeq)(const seq::SeqCfg);
struct KSeqInfo { KSeq fn; int tab, stage, ntb; };
// bf16 x always takes the exact table (the pair table multiplies fp16 by fp16), whatever `mode` says
KSeqInfo kseq_lookup(int bits, int mode, bool multi, bool bf16) {
#define KSE(B, M, X) KSeqInfo{seq::lutgemv_seq_kernel<B, M, X>, v2::C2<B, M>::TAB, v2::C2<B, M>::STAGE, v2::C2<B, M>::NTB}
#define KSB(B, X) KSeqInfo{seq::lutgemv_seq_kernel<B, 0, X, __nv_bfloat16>, v2::C2<B, 0>::TAB, v2::C2<B, 0>::STAGE, v2::C2<B, 0>::NTB}
    if (bf16) {
        if (bits == 4) return multi ? KSB(4, true) : KSB(4, false);
        return multi ? KSB(3, true) : KSB(3, false);
    }
    if (bits == 4) {
        if (mode == 0) return multi ? KSE(4, 0, true) : KSE(4, 0, false);
        return multi ? KSE(4, 1, true) : KSE(4, 1, false);
    }
    if (mode == 0) return multi ? KSE(3, 0, true) : KSE(3, 0, false);
    return multi ? KSE(3, 1, true) : KSE(3, 1, false);
#undef KSB
#undef KSE
}
constexpr int SEQ_MAX_ITEMS = 1023;  // the mailbox tag keeps 10 bits for the item

size_t seq_item_len(const sqllm_seq_item &it) {  // elements of the item's full-length output vector
    const int members = it.members > 0 ? it.members : 1;
    const int nfull = it.out_features_full > 0 ? it.out_features_full : it.a.out_features / members;
    return (size_t)members * nfull;
}
}  // namespace

struct sqllm_sequence {
    int n = 0, bits = 0, mode = 0, world = 1, rank = 0, grid = 0, smem = 0;
    seq::SeqCfg cfg;
    KSeq fn = nullptr;
    void *d_descs = nullptr, *d_exports = nullptr, *d_ws = nullptr, *d_arena = nullptr;
    bool own_arena = false;
};

namespace {
int seq_fail_free(sqllm_sequence *s, int rc) {
    if (s) sqllm_sequence_destroy(s);
    return rc;
}
}  // namespace

extern "C" size_t sqllm_sequence_arena_bytes(const sqllm_seq_item *items, int n_items) {
    if (!items || n_items <= 0) return 0;
    size_t off = 0;
    for (int i = 0; i < n_items; ++i) off += (seq_item_len(items[i]) * 4 + 127) / 128 * 128;
    return off;
}

extern "C" int sqllm_sequence_create(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, sqllm_sequence **out) {
    return sqllm_sequence_create_dt(items, n_items, opt, SQLLM_DT_F16, out);
}

extern "C" int sqllm_sequence_create_dt(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, int dtype, sqllm_sequence **out) {
    if (dtype != SQLLM_DT_F16 && dtype != SQLLM_DT_BF16) return fail(SQLLM_EINVAL, "sequence: dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", dtype);
    const bool bf = dtype == SQLLM_DT_BF16;
    const char *const tn = bf ? "bf16" : "fp16";
    if (!items || !opt || !out || n_items <= 0) return fail(SQLLM_EINVAL, "sequence: null / empty arguments");
    if (n_items > SEQ_MAX_ITEMS) return fail(SQLLM_EINVAL, "sequence: at most %d items (got %d)", SEQ_MAX_ITEMS, n_items);
    const int world = opt->world > 0 ? opt->world : 1, rank = opt->rank;
    if (world > 64 || rank < 0 || rank >= world) return fail(SQLLM_EINVAL, "sequence: bad world / rank (%d / %d)", world, rank);
    if (world > 1 && (!opt->arena || !opt->peer_base)) return fail(SQLLM_EINVAL, "sequence: several GPUs need a peer-visible arena and peer_base");
    // bf16 x keeps the exact table in the fp16 table mode, as sqllm_lutgemv_fused_dt does
    const int bits = items[0].a.bits, mode = opt->lut_mode == SQLLM_LUT_FP16_PAIR && !bf ? 1 : 0;
    int kmax = 0;
    for (int i = 0; i < n_items; ++i) {
        const sqllm_seq_item &it = items[i];
        const sqllm_lutgemv_args &a = it.a;
        const int rc = check_common(&a);
        if (rc) return rc;
        if (a.bits != bits) return fail(SQLLM_EINVAL, "sequence: item %d has bits=%d, item 0 has %d (one sequence, one width)", i, a.bits, bits);
        if (a.out_features < STRIP) return fail(SQLLM_EINVAL, "sequence: item %d: out_features=%d < %d", i, a.out_features, STRIP);
        if (a.out_features > MAX_N_FUSED) return fail(SQLLM_EINVAL, "sequence: item %d: out_features=%d exceeds %d", i, a.out_features, MAX_N_FUSED);
        if (a.full_rows && a.topX > MAX_TOPX_FUSED) return fail(SQLLM_EINVAL, "sequence: topX <= %d", MAX_TOPX_FUSED);
        const int members = it.members > 0 ? it.members : 1;
        if (a.out_features % members || (a.out_features / members) % 4) return fail(SQLLM_EINVAL, "sequence: item %d: %d columns are not %d members of a multiple of 4", i, a.out_features, members);
        if (world == 1 && seq_item_len(it) != (size_t)a.out_features) return fail(SQLLM_EINVAL, "sequence: item %d: members * out_features_full must equal out_features on one GPU", i);
        if (world > 1 && seq_item_len(it) < (size_t)world * a.out_features) return fail(SQLLM_EINVAL, "sequence: item %d: full length %zu < world * shard columns", i, seq_item_len(it));
        if (world > 1 && it.y) return fail(SQLLM_EINVAL, "sequence: item %d: plain y copies exist on one GPU only (use exports)", i);
        if (seq_item_len(it) % 4) return fail(SQLLM_EINVAL, "sequence: item %d: output length must be a multiple of 4", i);
        if (it.x_from >= i || it.x_from < -1) return fail(SQLLM_EINVAL, "sequence: item %d: x_from=%d must name an earlier item (or -1)", i, it.x_from);
        if (it.x_from < 0) {
            if (!it.x_ext || (reinterpret_cast<uintptr_t>(it.x_ext) & 15)) return fail(SQLLM_EINVAL, "sequence: item %d: x_ext must be a 16-byte aligned %s vector", i, tn);
        } else {
            if (it.x_offset < 0 || it.x_offset % 4 || (size_t)it.x_offset + a.in_features > seq_item_len(items[it.x_from]))
                return fail(SQLLM_EINVAL, "sequence: item %d reads [%d, %d) of item %d's %zu outputs", i, it.x_offset, it.x_offset + a.in_features, it.x_from, seq_item_len(items[it.x_from]));
        }
        if ((reinterpret_cast<uintptr_t>(it.y) & 1) || (reinterpret_cast<uintptr_t>(it.bias) & 3)) return fail(SQLLM_EINVAL, "sequence: item %d: misaligned y / bias", i);
        kmax = std::max(kmax, a.in_features);
    }
    for (int e = 0; e < opt->n_export; ++e) {
        if (!opt->export_items || !opt->export_dst) return fail(SQLLM_EINVAL, "sequence: export arrays missing");
        const int it = opt->export_items[e];
        if (it < 0 || it >= n_items || !opt->export_dst[e] || (reinterpret_cast<uintptr_t>(opt->export_dst[e]) & 7))
            return fail(SQLLM_EINVAL, "sequence: export %d: bad item %d or destination (8-byte aligned %s vector)", e, it, tn);
    }
    const KSeqInfo ki = kseq_lookup(bits, mode, world > 1, bf);
    int sm = 0;
    unsigned raw = 0;
    const int rc = dev_setup({{ki.fn, 227 * 1024}}, &sm, &raw);
    if (rc) return rc;
    const unsigned base = (raw + 127u) & ~127u;
    const int xbytes = (kmax * 2 + 127) & ~127;  // every item's x is staged in the 16-bit dtype in one buffer, and ntb strip-sum rows follow it
    // no cap from the chunk: the weight stream runs on across items
    const int nst = v2::Carve(base, xbytes, ki.ntb * STRIP * 4, ki.tab, ki.ntb, ki.stage, 0).depth(raw, 227 * 1024, ki.stage, v2::MAXD);
    if (nst < 0) return fail(SQLLM_EINVAL, "sequence: in_features=%d does not fit the shared-memory carve-up of this table mode", kmax);
    if (nst < 2) return fail(SQLLM_EINVAL, "sequence: in_features=%d leaves no room for a weight ring in shared memory", kmax);
    const int smem = (int)(v2::Carve(base, xbytes, ki.ntb * STRIP * 4, ki.tab, ki.ntb, ki.stage, nst).end - raw);

    sqllm_sequence *s = new sqllm_sequence();
    s->n = n_items; s->bits = bits; s->mode = mode; s->world = world; s->rank = rank; s->grid = sm; s->smem = smem; s->fn = ki.fn;
    // workspace: [0,4) token counter, [64,68) error word, per parity {flags [64 + MAX_STRIPS] ints, accumulator [MAX_N_FUSED] floats} (only
    // used by CTAs that own more than 8 strips), then EVERY item's own mailboxes: outlier row sums [N], partial strip sums [grid][64],
    // dense-row parts [topX][MAX_GRID_V2].  Mailboxes are not shared between items: an item may read only a slice of its predecessor's
    // output, so "x of item g+1 is complete" does not mean that every strip owner of item g has already taken its words.
    const size_t cnt_bytes = (size_t)(64 + MAX_STRIPS) * 4, acc_bytes = (size_t)MAX_N_FUSED * 4;
    const size_t par_off = 256, par_bytes = (cnt_bytes + acc_bytes + 255) / 256 * 256;
    std::vector<size_t> cbox_off(n_items), hbox_off(n_items), dbox_off(n_items);
    size_t ws_bytes = par_off + 2 * par_bytes;
    for (int i = 0; i < n_items; ++i) {
        const bool hyb = items[i].a.full_rows && items[i].a.topX > 0;
        cbox_off[i] = ws_bytes; ws_bytes += ((size_t)items[i].a.out_features * 8 + 255) / 256 * 256;
        hbox_off[i] = ws_bytes; ws_bytes += (size_t)MAX_GRID_V2 * 64 * 8;
        dbox_off[i] = ws_bytes; ws_bytes += hyb ? (size_t)items[i].a.topX * MAX_GRID_V2 * 8 : 0;
    }
    if (cudaMalloc(&s->d_ws, ws_bytes) != cudaSuccess || cudaMemset(s->d_ws, 0, ws_bytes) != cudaSuccess)
        return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: workspace allocation failed"));
    unsigned char *ws = static_cast<unsigned char *>(s->d_ws);
    const size_t arena_need = sqllm_sequence_arena_bytes(items, n_items);
    if (opt->arena) {
        if (opt->arena_bytes < arena_need || (reinterpret_cast<uintptr_t>(opt->arena) & 127))
            return seq_fail_free(s, fail(SQLLM_EINVAL, "sequence: arena of %zu bytes (128-byte aligned) needed, got %zu", arena_need, opt->arena_bytes));
        s->d_arena = opt->arena;
    } else {
        if (cudaMalloc(&s->d_arena, arena_need) != cudaSuccess || cudaMemset(s->d_arena, 0, arena_need) != cudaSuccess)
            return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: arena allocation failed"));
        s->own_arena = true;
    }
    std::vector<seq::SeqDesc> descs(n_items);
    std::vector<size_t> yoff(n_items);
    size_t off = 0;
    for (int i = 0; i < n_items; ++i) {
        yoff[i] = off;
        off += (seq_item_len(items[i]) * 4 + 127) / 128 * 128;
    }
    for (int i = 0; i < n_items; ++i) {
        const sqllm_seq_item &it = items[i];
        const sqllm_lutgemv_args &a = it.a;
        seq::SeqDesc &d = descs[i];
        memset(&d, 0, sizeof(d));
        v2::P2 &p = d.p;
        int G = 0;
        int rc = plan_layer(a, sm, p, G);
        if (rc) return seq_fail_free(s, rc);
        if (G > MAX_GRID_V2) return seq_fail_free(s, fail(SQLLM_EINVAL, "sequence: grid of %d CTAs exceeds the mailbox area", G));
        p.nstage = nst; p.smem_raw = raw;
        p.y_is_half = 1;
        p.bias = it.bias;
        p.out = it.y;
        p.x = it.x_from < 0 ? it.x_ext : nullptr;
        unsigned char *par = ws + par_off + (size_t)(i & 1) * par_bytes;
        p.ws_cnt = reinterpret_cast<int *>(par);
        p.ws_acc = reinterpret_cast<float *>(par + cnt_bytes);
        p.ws_hbox = reinterpret_cast<unsigned long long *>(ws + hbox_off[i]);
        p.ws_cbox = reinterpret_cast<unsigned long long *>(ws + cbox_off[i]);
        p.ws_dbox = reinterpret_cast<unsigned long long *>(ws + dbox_off[i]);
        p.xw_world = world > 1 ? world : 0; p.xw_rank = rank;
        p.xw_members = it.members > 0 ? it.members : 1;
        p.xw_nfull = it.out_features_full > 0 ? it.out_features_full : p.N / p.xw_members;
        p.trace = opt->trace ? reinterpret_cast<unsigned long long *>(opt->trace) + (size_t)i * 1024 * 32 : nullptr;
        d.x_tag = it.x_from < 0 ? nullptr : reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[it.x_from]) + it.x_offset;
        d.y_off = yoff[i];
        if ((rc = tensor_maps(a, d.tm_big, d.tm_small))) return seq_fail_free(s, rc);
    }
    std::vector<seq::SeqExport> ex(std::max(1, opt->n_export));
    for (int e = 0; e < opt->n_export; ++e) {
        const int it = opt->export_items[e];
        ex[e].src = reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[it]);
        ex[e].dst = opt->export_dst[e];
        ex[e].n = (int)seq_item_len(items[it]);
    }
    if (cudaMalloc(&s->d_descs, descs.size() * sizeof(seq::SeqDesc)) != cudaSuccess ||
        cudaMemcpy(s->d_descs, descs.data(), descs.size() * sizeof(seq::SeqDesc), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMalloc(&s->d_exports, ex.size() * sizeof(seq::SeqExport)) != cudaSuccess ||
        cudaMemcpy(s->d_exports, ex.data(), ex.size() * sizeof(seq::SeqExport), cudaMemcpyHostToDevice) != cudaSuccess)
        return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: descriptor upload failed: %s", cudaGetErrorString(cudaGetLastError())));
    seq::SeqCfg &c = s->cfg;
    memset(&c, 0, sizeof(c));
    c.descs = static_cast<const seq::SeqDesc *>(s->d_descs);
    c.ngemv = n_items;
    c.epoch = reinterpret_cast<const unsigned *>(ws);
    c.err = reinterpret_cast<int *>(ws + 64);
    c.smem_raw = raw; c.xbytes = xbytes; c.nstage = nst;
    c.world = world; c.rank = rank;
    c.peer_base = reinterpret_cast<const unsigned long long *>(opt->peer_base);
    c.arena_base = reinterpret_cast<unsigned long long>(s->d_arena);
    c.exports = static_cast<const seq::SeqExport *>(s->d_exports);
    c.nexport = opt->n_export;
    *out = s;
    return SQLLM_OK;
}

extern "C" int sqllm_sequence_run(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    seq::seq_bump_epoch<<<1, 1, 0, st>>>(reinterpret_cast<unsigned *>(s->d_ws));
    const cudaError_t e = launch_ex(s->fn, s->grid, v2::THREADS2, s->smem, st, COOPERATIVE, s->cfg);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "sequence launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

extern "C" int sqllm_sequence_error(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    int h = 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (cudaMemcpyAsync(&h, static_cast<unsigned char *>(s->d_ws) + 64, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return fail(SQLLM_ECUDA, "sequence: reading the error word failed: %s", cudaGetErrorString(cudaGetLastError()));
    return h != 0;
}

extern "C" int sqllm_sequence_reset_error(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    if (cudaMemsetAsync(static_cast<unsigned char *>(s->d_ws) + 64, 0, 4, static_cast<cudaStream_t>(stream)) != cudaSuccess)
        return fail(SQLLM_ECUDA, "sequence: clearing the error word failed: %s", cudaGetErrorString(cudaGetLastError()));
    return SQLLM_OK;
}

extern "C" void sqllm_sequence_destroy(sqllm_sequence *s) {
    if (!s) return;
    cudaFree(s->d_descs);
    cudaFree(s->d_exports);
    cudaFree(s->d_ws);
    if (s->own_arena) cudaFree(s->d_arena);
    delete s;
}

namespace {

// ---- batched symbols: tile kernel + outlier kernels (lutgemm_batched.cuh) ----------------------------------------------
int launch_batched(const sqllm_lutgemv_args *a, cudaStream_t st) {
    using namespace batched;
    const auto kern = a->bits == 4 ? lutgemm_batched_kernel<4> : lutgemm_batched_kernel<3>;
    const int rc = dev_setup({{kern, 227 * 1024}});
    if (rc) return rc;
    const int K = a->in_features, N = a->out_features, B = a->batch;
    const int XU = a->bits == 4 ? 8 : 32, tab = a->bits == 4 ? CB<4>::TAB : CB<3>::TAB;
    PB p;
    p.qw = reinterpret_cast<const uint32_t *>(a->qweight); p.lut = a->lookup_table; p.x = a->vec; p.mul = a->mul;
    p.K = K; p.N = N; p.B = B; p.R = K / XU;
    // K-slabs: the BT x rows of a slab sit in shared memory next to the table and the partial sums; <= 2048 inputs per slab keeps a
    // CTA under 90 KB, i.e. two CTAs (16 warps) per SM
    int slabs = (K + 2047) / 2048;
    p.ks = 2 * ((p.R + 2 * slabs - 1) / (2 * slabs));
    slabs = (p.R + p.ks - 1) / p.ks;
    const int kslab = p.ks * XU;
    const size_t smem = (size_t)2 * tab + (size_t)BT * (kslab * 4 + 16) + (size_t)BW * BT * STRIP * 4;
    if (smem > 227 * 1024) return fail(SQLLM_EINVAL, "batched tile needs %zu B of shared memory", smem);
    const int strips = (N + STRIP - 1) / STRIP, btiles = (B + BT - 1) / BT;
    if (btiles > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", B, 65535 * BT);
    const dim3 grid(strips, slabs, btiles);
    kern<<<grid, BTHREADS, smem, st>>>(p);
    if (a->rows) {
        const dim3 blk(32, 8), g((N + 7) / 8, std::min((B + 31) / 32, 64));
        csr_batched_kernel<<<g, blk, 0, st>>>(a->rows, a->cols, a->vals, a->vec, a->mul, K, N, B);
    }
    if (a->full_rows && a->topX > 0) {
        if (a->topX > 256) return fail(SQLLM_EINVAL, "batched path supports topX <= 256");
        const int per = 256 / a->topX;
        dense_rows_batched_kernel<<<B, per * a->topX, 0, st>>>(a->full_rows, a->full_row_indices, a->topX, a->vec, a->mul, K, N, B);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "batched launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

// ---- a few fp16 / bf16 rows (lutgemv_rows.cuh): plan + launch ------------------------------------------------------------------
// Slabs per strip S (the cluster size) from K, N and the SM count only - never from M, so that a row's result does not depend on
// M: the smallest S in {1, 2, 4, 8} that gives at least two CTAs per SM and a slab of at most SLAB_GOAL inputs, with no more
// slabs than units.  Rows per CTA RB from M: 2, 4 or 8 (a row computes the same bits whatever RB is).
struct RowsPlan { int S, ks, kpad, RB, smem; };
int rows_plan(int bits, int K, int N, int M, int sm, RowsPlan &pl) {
    using namespace rows;
    const int XU = bits == 4 ? 8 : 32, R = K / XU, strips = (N + STRIP - 1) / STRIP;
    int S = 1;
    while (S < MAX_SLABS && 2 * S <= R && ((long long)strips * S < 2LL * sm || (long long)(R + S - 1) / S * XU > SLAB_GOAL)) S *= 2;
    pl.S = S;
    pl.ks = (R + S - 1) / S;
    pl.kpad = (pl.ks + (pl.ks & 1)) * XU;
    pl.RB = M <= 2 ? 2 : M <= 4 ? 4 : 8;
#define RS(B, RBV) SR<B, RBV>::total(pl.kpad)
    pl.smem = bits == 4 ? (pl.RB == 2 ? RS(4, 2) : pl.RB == 4 ? RS(4, 4) : RS(4, 8)) : (pl.RB == 2 ? RS(3, 2) : pl.RB == 4 ? RS(3, 4) : RS(3, 8));
#undef RS
    if (pl.smem > 227 * 1024) return fail(SQLLM_EINVAL, "in_features=%d needs %d B of shared memory per CTA (> 227 KB)", K, pl.smem);
    return SQLLM_OK;
}

typedef void (*KRows)(const rows::PR);
template <typename XT>
KRows krows_lookup_t(int bits, int RB) {
    using namespace rows;
    if (bits == 4) return RB == 2 ? lutgemv_rows_kernel<4, 2, XT> : RB == 4 ? lutgemv_rows_kernel<4, 4, XT> : lutgemv_rows_kernel<4, 8, XT>;
    return RB == 2 ? lutgemv_rows_kernel<3, 2, XT> : RB == 4 ? lutgemv_rows_kernel<3, 4, XT> : lutgemv_rows_kernel<3, 8, XT>;
}
KRows krows_lookup(int bits, int RB, bool bf16) { return bf16 ? krows_lookup_t<__nv_bfloat16>(bits, RB) : krows_lookup_t<__half>(bits, RB); }

// ---- input gradient (lutgemm_t.cuh): plan + launch --------------------------------------------------------------------------
// Strip splits S (the cluster size) from K, N and the SM count only - never from M, so that a row's result does not depend on M:
// the smallest S in {1, 2, 4, 8} that gives at least two CTAs per SM, with at least two strips per CTA.  Rows per CTA RB from M:
// 1, 2, 4 or 8 (a row computes the same bits whatever RB is).
struct TPlan { int S, RB, smem; };
void t_plan(int K, int N, int M, int sm, TPlan &pl) {
    using namespace bwd;
    const int slabs = (K + KS - 1) / KS, strips = (N + STRIP - 1) / STRIP;
    int S = 1;
    while (S < MAX_SPLIT && 4 * S <= strips && (long long)slabs * S < 2LL * sm) S *= 2;
    pl.S = S;
    pl.RB = M <= 1 ? 1 : M <= 2 ? 2 : M <= 4 ? 4 : 8;
    pl.smem = pl.RB == 1 ? ST<1>::TOTAL : pl.RB == 2 ? ST<2>::TOTAL : pl.RB == 4 ? ST<4>::TOTAL : ST<8>::TOTAL;
}

typedef void (*KT)(const bwd::PT);
KT kt_lookup(int bits, int RB) {
    using namespace bwd;
    if (bits == 4) return RB == 1 ? lutgemm_t_kernel<4, 1> : RB == 2 ? lutgemm_t_kernel<4, 2> : RB == 4 ? lutgemm_t_kernel<4, 4> : lutgemm_t_kernel<4, 8>;
    return RB == 1 ? lutgemm_t_kernel<3, 1> : RB == 2 ? lutgemm_t_kernel<3, 2> : RB == 4 ? lutgemm_t_kernel<3, 4> : lutgemm_t_kernel<3, 8>;
}

// ---- codebook gradient (lut_grad.cuh, lut_grad_tc.cuh): plan -------------------------------------------------------------
// K splits S (the cluster size) from K, N and the SM count only: the smallest S in {1, 2, 4, 8} that gives at least one CTA per
// SM, with at least two k-tiles per CTA.
int lg_split(int K, int N, int sm) {
    using namespace lg;
    const int ktiles = (K + TK - 1) / TK, ctiles = (N + TC - 1) / TC;
    int S = 1;
    while (S < MAX_SPLIT && 4 * S <= ktiles && (long long)ctiles * S < sm) S *= 2;
    return S;
}

// ---- fused GEMV: v2, or v1 in the deterministic mode; with an exchange descriptor (v2 only) the result goes to every rank's
// arena instead of y ---------------------------------------------------------------------------------------------------------------
// x_dt / y_dt: SQLLM_DT_* codes, a pair sqllm_lutgemv_fused_dt accepts
int lutgemv_fused(const sqllm_lutgemv_args *a, const void *x, int x_dt, void *y, int y_dt, const float *bias,
                  void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, cudaStream_t st) {
    int rc = check_common(a);
    if (rc) return rc;
    if (!x || (!xc && !y)) return fail(SQLLM_EINVAL, xc ? "x / exchange descriptor must not be null" : "x / y must not be null");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(bias) & 15))
        return fail(SQLLM_EINVAL, xc ? "bias must be 16-byte aligned" : "y and bias must be 16-byte aligned");
    const int det = det_mode();
    if (xc) {
        if (det == 1) return fail(SQLLM_EINVAL, "the exchange path needs the default (non-deterministic) fused mode");
        if (xc->world < 1 || xc->world > 64 || xc->rank < 0 || xc->rank >= xc->world) return fail(SQLLM_EINVAL, "bad world / rank (%d / %d)", xc->world, xc->rank);
        if (xc->members < 1 || a->out_features % xc->members) return fail(SQLLM_EINVAL, "out_features=%d is not %d equal members", a->out_features, xc->members);
        const int w = a->out_features / xc->members;
        if (w % 4) return fail(SQLLM_EINVAL, "shard width %d must be a multiple of 4", w);
        if (xc->out_features_full < xc->world * w) return fail(SQLLM_EINVAL, "out_features_full=%d < world * shard width = %d", xc->out_features_full, xc->world * w);
        if (!xc->peer_base) return fail(SQLLM_EINVAL, "peer_base must not be null");
        if ((xc->out_offset & 15) || (xc->flag_offset & 7) || (xc->state_offset & 7) || (xc->error_offset & 3)) return fail(SQLLM_EINVAL, "misaligned arena offsets");
        const int yb = y_dt == SQLLM_DT_F32 ? 4 : 2;
        if ((xc->out_features_full * yb) % 16 || (w * yb) % 8) return fail(SQLLM_EINVAL, "vector sizes must keep 8/16-byte store alignment");
    }
    const bool hyb = a->full_rows && a->topX > 0;
    if (hyb && a->topX > MAX_TOPX_FUSED) return fail(SQLLM_EINVAL, "fused path supports topX <= %d", MAX_TOPX_FUSED);
    unsigned char *ws = static_cast<unsigned char *>(workspace);
    if (det == 0) {
        if (!workspace || workspace_bytes < WS_HEADER) return fail(SQLLM_EWORKSPACE, "workspace too small: need %zu bytes, got %zu", (size_t)WS_HEADER, workspace_bytes);
        v2::P2 q;
        memset(&q, 0, sizeof(q));
        q.ws_cnt = reinterpret_cast<int *>(ws);
        q.ws_acc = reinterpret_cast<float *>(ws + WS_ACC_OFF);
        q.ws_hbox = reinterpret_cast<unsigned long long *>(ws + WS_HBOX_OFF);
        q.ws_cbox = reinterpret_cast<unsigned long long *>(ws + WS_CBOX_OFF);
        q.ws_dbox = reinterpret_cast<unsigned long long *>(ws + WS_DBOX_OFF);
        q.x = x; q.out = y; q.y_is_half = y_dt != SQLLM_DT_F32; q.bias = bias;
        if (xc) {
            q.xw_world = xc->world; q.xw_rank = xc->rank; q.xw_members = xc->members; q.xw_nfull = xc->out_features_full;
            q.xw_base = reinterpret_cast<const unsigned long long *>(xc->peer_base);
            q.xw_out_off = xc->out_offset; q.xw_flag_off = xc->flag_offset; q.xw_state_off = xc->state_offset; q.xw_err_off = xc->error_offset;
        }
        // layers narrower than one strip keep the exact codebook in the fp16 table mode: their results do not depend on the mode;
        // bf16 x always does (the pair table multiplies fp16 by fp16)
        const int variant = x_dt == SQLLM_DT_F16 ? (lut_mode() == 1 && a->out_features >= STRIP ? 2 : 1) : x_dt == SQLLM_DT_BF16 ? 3 : 0;
        return launch2(a, variant, true, q, st);
    }
    Plan pl;
    rc = make_plan(a->bits, a->in_features, a->out_features, hyb ? a->topX : 0, a->rows != nullptr, STAGE, pl);
    if (rc) return rc;
    if (!workspace || workspace_bytes < pl.ws_bytes)
        return fail(SQLLM_EWORKSPACE, "workspace too small: need %zu bytes, got %zu", pl.ws_bytes, workspace_bytes);
    Params p;
    memset(&p, 0, sizeof(p));
    p.ws_cnt = reinterpret_cast<int *>(ws + pl.ws_cnt_off);
    p.ws_hyb = reinterpret_cast<float *>(ws + pl.ws_hyb_off);
    p.ws_part = reinterpret_cast<float *>(ws + pl.ws_part_off);
    p.ws_csr = reinterpret_cast<float *>(ws + pl.ws_csr_off);
    p.x = x; p.x_dt = x_dt; p.out = y; p.y_dt = y_dt; p.bias = bias;
    return launch(a, pl, p, st);
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int sqllm_abi_version(void) { return SQLLM_ABI_VERSION; }
void sqllm_set_deterministic(int on) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    g_det = on ? 1 : 0;
}
void sqllm_set_lut_mode(int mode) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    g_lut_mode = mode == SQLLM_LUT_FP16_PAIR ? 1 : 0;
}
int sqllm_get_lut_mode(void) { return lut_mode(); }
int sqllm_workspace_error(const void *workspace, void *stream) {
    if (!workspace) return fail(SQLLM_EINVAL, "null workspace");
    int flag = 0;
    if (cudaMemcpyAsync(&flag, static_cast<const unsigned char *>(workspace) + 64, 4, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)) != cudaSuccess ||
        cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess)
        return fail(SQLLM_ECUDA, "cannot read the workspace error word: %s", cudaGetErrorString(cudaGetLastError()));
    return flag ? 1 : 0;
}

// debug hook (not in the public header): successive launches write their timeline at buf, buf+stride, ...
void sqllm_debug_set_trace(unsigned long long *buf, size_t stride_words) { g_trace = buf; g_trace_stride = stride_words; }
int sqllm_debug_last_grid(void) { return g_last_grid; }
const char *sqllm_last_error(void) { return g_err; }

int sqllm_device_sm_count(void) {
    int sm = 0;
    return dev_setup({}, &sm) ? 0 : sm;
}

size_t sqllm_workspace_bytes(int bits, int in_features, int out_features, int topX) {
    Plan pl;
    if (bits != 3 && bits != 4) return 0;
    if (in_features <= 0 || in_features % 64 || out_features <= 0) return 0;
    // CSR staging changes the shared-memory footprint, hence occupancy, grid and chunk: take the max of both plans.  The
    // deterministic mode gets exactly what its kernel needs.  The default mode plans with the CSR cols / vals alone in the staging
    // buffer: less shared memory, at least as many CTAs and strip partials, so a workspace sized in either mode serves both.
    const int stage = det_mode() == 1 ? STAGE : CSR_CH * 8;
    size_t b = 0;
    for (int csr = 0; csr < 2; ++csr)
        if (make_plan(bits, in_features, out_features, topX, csr != 0, stage, pl) == SQLLM_OK && pl.ws_bytes > b) b = pl.ws_bytes;
    return b;
}

int sqllm_lutgemv(const sqllm_lutgemv_args *a, void *stream) {
    int rc = check_common(a);
    if (rc) return rc;
    if (!a->vec || !a->mul) return fail(SQLLM_EINVAL, "vec / mul must not be null");
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch must be >= 1");
    if (reinterpret_cast<uintptr_t>(a->vec) & 15) return fail(SQLLM_EINVAL, "vec must be 16-byte aligned");
    if (a->batch >= 2) return launch_batched(a, static_cast<cudaStream_t>(stream));
    v2::P2 q;
    memset(&q, 0, sizeof(q));
    q.x = a->vec;
    q.out = a->mul;
    return launch2(a, 0, false, q, static_cast<cudaStream_t>(stream));
}

int sqllm_lutgemv_fused(const sqllm_lutgemv_args *a, const void *x, int x_is_half, void *y, int y_is_half,
                        const float *bias, void *workspace, size_t workspace_bytes, void *stream) {
    return sqllm_lutgemv_fused_dt(a, x, x_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias,
                                  workspace, workspace_bytes, stream);
}

int sqllm_lutgemv_fused_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *workspace, size_t workspace_bytes, void *stream) {
    if (!fused_dt_pair(x_dtype, y_dtype)) return fused_dt_fail(x_dtype, y_dtype);
    return lutgemv_fused(a, x, x_dtype, y, y_dtype, bias, workspace, workspace_bytes, nullptr, static_cast<cudaStream_t>(stream));
}

int sqllm_lutgemv_fused_exchange(const sqllm_lutgemv_args *a, const void *x, int x_is_half, int y_is_half, const float *bias,
                                 void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, void *stream) {
    return sqllm_lutgemv_fused_exchange_dt(a, x, x_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias,
                                           workspace, workspace_bytes, xc, stream);
}

int sqllm_lutgemv_fused_exchange_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, int y_dtype, const float *bias,
                                    void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, void *stream) {
    if (!fused_dt_pair(x_dtype, y_dtype)) return fused_dt_fail(x_dtype, y_dtype);
    if (!xc) {
        const int rc = check_common(a);
        return rc ? rc : fail(SQLLM_EINVAL, "x / exchange descriptor must not be null");
    }
    return lutgemv_fused(a, x, x_dtype, nullptr, y_dtype, bias, workspace, workspace_bytes, xc, static_cast<cudaStream_t>(stream));
}

int sqllm_lutgemm_fused(const sqllm_lutgemv_args *a, const void *x, void *y, int y_is_half, const float *bias, void *stream) {
    return sqllm_lutgemm_fused_dt(a, x, SQLLM_DT_F16, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias, stream);
}

// sqllm_lutgemm_fused_dt (f32 = false) and sqllm_lutgemm_fused_f32 (f32 = true: x and y fp32, the dtype codes are not looked at):
// the argument checks, in this order and all before any device access, then the launch
static int lutgemm_tc_launch(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                             void *stream, bool f32) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->out_features + tc::BN - 1) / tc::BN > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * tc::BN);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x) must be >= 1 (got %d)", a->batch);
    if (!x || !y) return fail(SQLLM_EINVAL, "x / y must not be null");
    if (!f32) {
        if (x_dtype != SQLLM_DT_F16 && x_dtype != SQLLM_DT_BF16) return fail(SQLLM_EINVAL, "x_dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", x_dtype);
        if (y_dtype != SQLLM_DT_F32 && y_dtype != x_dtype) return fail(SQLLM_EINVAL, "y_dtype=%d must be SQLLM_DT_F32 or x's dtype (%d)", y_dtype, x_dtype);
    }
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3) || (reinterpret_cast<uintptr_t>(bias) & 3))
        return fail(SQLLM_EINVAL, "qweight, lookup_table and bias must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(y) & 15) return fail(SQLLM_EINVAL, "y must be 16-byte aligned");
    if (f32) { x_dtype = SQLLM_DT_F32; y_dtype = SQLLM_DT_F32; }
    const bool bf = x_dtype == SQLLM_DT_BF16;
    const auto kern = f32 ? (a->bits == 4 ? tc::lutgemm_tc_kernel<4, true, true> : tc::lutgemm_tc_kernel<3, true, true>)
                    : a->bits == 4 ? (bf ? tc::lutgemm_tc_kernel<4, true> : tc::lutgemm_tc_kernel<4, false>)
                                   : (bf ? tc::lutgemm_tc_kernel<3, true> : tc::lutgemm_tc_kernel<3, false>);
    const int smem = f32 ? tc::L<3, 3>::SMEM : bf ? tc::L<3>::SMEM : tc::L<2>::SMEM;
    if ((rc = dev_setup({{kern, smem}}))) return rc;
    tc::PT p;
    set_layer(p, *a);
    p.x = static_cast<const unsigned short *>(x); p.y = y; p.y_16 = y_dtype != SQLLM_DT_F32; p.bias = bias;
    p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
    const dim3 grid((a->batch + tc::BM - 1) / tc::BM, (a->out_features + tc::BN - 1) / tc::BN);
    kern<<<grid, tc::THREADS, smem, static_cast<cudaStream_t>(stream)>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_fused launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_lutgemm_fused_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *stream) {
    return lutgemm_tc_launch(a, x, x_dtype, y, y_dtype, bias, stream, false);
}

int sqllm_lutgemm_fused_f32(const sqllm_lutgemv_args *a, const float *x, float *y, const float *bias, void *stream) {
    return lutgemm_tc_launch(a, x, SQLLM_DT_F32, y, SQLLM_DT_F32, bias, stream, true);
}

int sqllm_lutgemv_rows(const sqllm_lutgemv_args *a, const void *x, void *y, int y_is_half, const float *bias, void *stream) {
    return sqllm_lutgemv_rows_dt(a, x, SQLLM_DT_F16, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias, stream);
}

int sqllm_lutgemv_rows_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias, void *stream) {
    int rc = check_layer(a, 32, 4);
    if (rc) return rc;
    if ((x_dtype != SQLLM_DT_F16 && x_dtype != SQLLM_DT_BF16) || (y_dtype != SQLLM_DT_F32 && y_dtype != x_dtype))
        return fail(SQLLM_EINVAL, "x_dtype=%d, y_dtype=%d: x must be SQLLM_DT_F16 or SQLLM_DT_BF16, y SQLLM_DT_F32 or x's dtype", x_dtype, y_dtype);
    if (a->in_features > SQLLM_ROWS_MAX_IN) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d: the slab of x a CTA stages would not fit its shared memory", a->in_features, SQLLM_ROWS_MAX_IN);
    if ((a->out_features + STRIP - 1) / STRIP > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * STRIP);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x) must be >= 1 (got %d)", a->batch);
    if (!x || !y) return fail(SQLLM_EINVAL, "x / y must not be null");
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3) || (reinterpret_cast<uintptr_t>(bias) & 3))
        return fail(SQLLM_EINVAL, "qweight, lookup_table and bias must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(y) & 15) return fail(SQLLM_EINVAL, "y must be 16-byte aligned");
    int sm = 0;
    if ((rc = dev_setup({}, &sm))) return rc;
    RowsPlan pl;
    if ((rc = rows_plan(a->bits, a->in_features, a->out_features, a->batch, sm, pl))) return rc;
    const KRows kern = krows_lookup(a->bits, pl.RB, x_dtype == SQLLM_DT_BF16);
    if ((rc = dev_setup({{kern, 227 * 1024}}))) return rc;
    const int groups = (a->batch + pl.RB - 1) / pl.RB;
    if (groups > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", a->batch, 65535 * pl.RB);
    rows::PR p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.x = x; p.y = y; p.y_16 = y_dtype != SQLLM_DT_F32; p.bias = bias;
    p.K = a->in_features; p.N = a->out_features; p.M = a->batch; p.R = a->bits == 4 ? p.K / 8 : p.K / 32;
    p.ks = pl.ks; p.kpad = pl.kpad;
    p.qw_al16 = (reinterpret_cast<uintptr_t>(a->qweight) & 15) == 0;
    // the S CTAs of a strip's cluster split its K
    const cudaError_t e = launch_ex(kern, dim3(pl.S, (a->out_features + STRIP - 1) / STRIP, groups), rows::RTHREADS, pl.smem,
                                    static_cast<cudaStream_t>(stream), cluster_of(pl.S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemv_rows launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_lutgemm_t(const sqllm_lutgemv_args *a, const void *dy, int dy_dtype, void *dx, int dx_dtype, int path, void *stream) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->in_features + bwd::KS - 1) / bwd::KS > 65535) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d", a->in_features, 65535 * bwd::KS);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of dy) must be >= 1 (got %d)", a->batch);
    if (!dy || !dx) return fail(SQLLM_EINVAL, "dy / dx must not be null");
    if (!dt_valid(dy_dtype)) return fail(SQLLM_EINVAL, "dy_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", dy_dtype);
    if (dx_dtype != SQLLM_DT_F32 && dx_dtype != dy_dtype) return fail(SQLLM_EINVAL, "dx_dtype=%d must be SQLLM_DT_F32 or dy's dtype (%d)", dx_dtype, dy_dtype);
    if (path < 0 || path > 2) return fail(SQLLM_EINVAL, "path=%d must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)", path);
    if (path == 1 && dy_dtype == SQLLM_DT_F32) return fail(SQLLM_EINVAL, "path=1 (tensor cores) takes fp16 or bf16 dy, not fp32");
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3))
        return fail(SQLLM_EINVAL, "qweight and lookup_table must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(dy) & (dy_dtype == SQLLM_DT_F32 ? 3 : 1)) return fail(SQLLM_EINVAL, "dy must be aligned to its element size");
    if (reinterpret_cast<uintptr_t>(dx) & 15) return fail(SQLLM_EINVAL, "dx must be 16-byte aligned");
    if (path == 0) path = dy_dtype != SQLLM_DT_F32 && a->batch >= SQLLM_BWD_TC_MIN_ROWS ? 1 : 2;
    if (path == 1) {
        const bool bf = dy_dtype == SQLLM_DT_BF16;
        const auto kern = a->bits == 4 ? (bf ? tct::lutgemm_tc_t_kernel<4, true> : tct::lutgemm_tc_t_kernel<4, false>)
                                       : (bf ? tct::lutgemm_tc_t_kernel<3, true> : tct::lutgemm_tc_t_kernel<3, false>);
        const int smem = bf ? tct::L<3>::SMEM : tct::L<2>::SMEM;
        if ((rc = dev_setup({{kern, smem}}))) return rc;
        tct::PT p;
        memset(&p, 0, sizeof(p));
        set_layer(p, *a);
        p.dy = dy; p.dx = dx; p.dx_dt = dx_dtype;
        p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
        p.dy_al16 = (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && a->out_features % 8 == 0;
        const dim3 grid((a->batch + tc::BM - 1) / tc::BM, (a->in_features + tct::BK - 1) / tct::BK);
        kern<<<grid, tct::THREADS, smem, static_cast<cudaStream_t>(stream)>>>(p);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_t (tensor cores) launch failed: %s", cudaGetErrorString(e));
        return SQLLM_OK;
    }
    int sm = 0;
    if ((rc = dev_setup({}, &sm))) return rc;
    TPlan pl;
    t_plan(a->in_features, a->out_features, a->batch, sm, pl);
    const KT kern = kt_lookup(a->bits, pl.RB);
    if ((rc = dev_setup({{kern, pl.smem}}))) return rc;
    const int groups = (a->batch + pl.RB - 1) / pl.RB;
    if (groups > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", a->batch, 65535 * pl.RB);
    bwd::PT p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.dy = dy; p.dx = dx; p.dy_dt = dy_dtype; p.dx_dt = dx_dtype;
    p.K = a->in_features; p.N = a->out_features; p.M = a->batch;
    p.strips = (a->out_features + STRIP - 1) / STRIP;
    p.qw_al16 = (reinterpret_cast<uintptr_t>(a->qweight) & 15) == 0 && a->out_features % 4 == 0;
    const cudaError_t e = launch_ex(kern, dim3(pl.S, (a->in_features + bwd::KS - 1) / bwd::KS, groups), bwd::TTHREADS, pl.smem,
                                    static_cast<cudaStream_t>(stream), cluster_of(pl.S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_t launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_lut_grad(const sqllm_lutgemv_args *a, const void *x, int x_dtype, const void *dy, int dy_dtype, float *dlut, float *dvals,
                   float *dfull_rows, int path, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    if (a->bits != 3 && a->bits != 4) return fail(SQLLM_EINVAL, "bits must be 3 or 4 (got %d)", a->bits);
    if (a->in_features <= 0 || a->in_features % 32) return fail(SQLLM_EINVAL, "in_features=%d must be a positive multiple of 32", a->in_features);
    if (a->out_features <= 0) return fail(SQLLM_EINVAL, "out_features=%d must be positive", a->out_features);
    if ((a->out_features + lg::TC - 1) / lg::TC > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * lg::TC);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x and dy) must be >= 1 (got %d)", a->batch);
    if (!a->qweight) return fail(SQLLM_EINVAL, "qweight must not be null");
    if (!x || !dy) return fail(SQLLM_EINVAL, "x / dy must not be null");
    if (!dt_valid(x_dtype)) return fail(SQLLM_EINVAL, "x_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", x_dtype);
    if (!dt_valid(dy_dtype)) return fail(SQLLM_EINVAL, "dy_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", dy_dtype);
    if (path < 0 || path > 2) return fail(SQLLM_EINVAL, "path=%d must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)", path);
    const bool tc_dtypes = x_dtype == dy_dtype && x_dtype != SQLLM_DT_F32;
    if (path == 1 && !tc_dtypes)
        return fail(SQLLM_EINVAL, "path=1 (tensor cores) takes x and dy both fp16 or both bf16 (got x_dtype=%d, dy_dtype=%d)", x_dtype, dy_dtype);
    if (!dlut && !dvals && !dfull_rows) return fail(SQLLM_EINVAL, "no output requested: dlut, dvals and dfull_rows are all null");
    if (dvals && (!a->rows || !a->cols)) return fail(SQLLM_EINVAL, "dvals needs the CSR arrays (rows, cols)");
    if (a->topX < 0) return fail(SQLLM_EINVAL, "topX < 0");
    if (dfull_rows && (!a->full_row_indices || a->topX < 1)) return fail(SQLLM_EINVAL, "dfull_rows needs the dense rows (full_row_indices, topX >= 1)");
    if (reinterpret_cast<uintptr_t>(a->qweight) & 3) return fail(SQLLM_EINVAL, "qweight must be 4-byte aligned");
    if ((reinterpret_cast<uintptr_t>(x) & (x_dtype == SQLLM_DT_F32 ? 3 : 1)) || (reinterpret_cast<uintptr_t>(dy) & (dy_dtype == SQLLM_DT_F32 ? 3 : 1)))
        return fail(SQLLM_EINVAL, "x and dy must be aligned to their element size");
    if ((reinterpret_cast<uintptr_t>(dlut) & 3) || (reinterpret_cast<uintptr_t>(dvals) & 3) || (reinterpret_cast<uintptr_t>(dfull_rows) & 3))
        return fail(SQLLM_EINVAL, "dlut, dvals and dfull_rows must be 4-byte aligned");
    if (path == 0) path = tc_dtypes && a->batch >= SQLLM_LUT_GRAD_TC_MIN_ROWS ? 1 : 2;

    lg::PG p;
    memset(&p, 0, sizeof(p));
    p.qw = reinterpret_cast<const uint32_t *>(a->qweight);
    p.x = x; p.dy = dy; p.x_dt = x_dtype; p.dy_dt = dy_dtype;
    p.rows = dvals ? a->rows : nullptr; p.cols = dvals ? a->cols : nullptr;
    p.fri = dfull_rows ? a->full_row_indices : nullptr; p.topX = dfull_rows ? a->topX : 0;
    p.dlut = dlut; p.dvals = dvals; p.dfull = dfull_rows;
    p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
    p.ktiles = (a->in_features + lg::TK - 1) / lg::TK;
    p.x_al16 = (reinterpret_cast<uintptr_t>(x) & 15) == 0;  // in_features % 32 == 0: every row is then 16-byte aligned
    p.dy_al16 = (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && a->out_features % 8 == 0;
    const bool bf = dy_dtype == SQLLM_DT_BF16;
    void (*kern)(const lg::PG);
    int smem;
    if (path == 1) {
        kern = bf ? (a->bits == 4 ? lgt::lut_grad_tc_kernel<4, true> : lgt::lut_grad_tc_kernel<3, true>)
                  : (a->bits == 4 ? lgt::lut_grad_tc_kernel<4, false> : lgt::lut_grad_tc_kernel<3, false>);
        smem = lgt::SMEM;
    } else {
        kern = a->bits == 4 ? lg::lut_grad_kernel<4> : lg::lut_grad_kernel<3>;
        smem = lg::SMEM;
    }
    int sm = 0;
    const int rc = dev_setup({{kern, smem}}, &sm);
    if (rc) return rc;
    const int S = lg_split(a->in_features, a->out_features, sm);
    const cudaError_t e = launch_ex(kern, dim3(S, (a->out_features + lg::TC - 1) / lg::TC), lg::THREADS, smem,
                                    static_cast<cudaStream_t>(stream), cluster_of(S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lut_grad launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_dequantize(const sqllm_lutgemv_args *a, int col0, int ncols, void *w, int w_dtype, void *stream) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->in_features + dq::BK - 1) / dq::BK > 65535) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d", a->in_features, 65535 * dq::BK);
    if (col0 < 0 || ncols < 1 || col0 > a->out_features - ncols)
        return fail(SQLLM_EINVAL, "column range col0=%d, ncols=%d must be non-empty and lie in [0, out_features=%d)", col0, ncols, a->out_features);
    if (!w) return fail(SQLLM_EINVAL, "w must not be null");
    if (!dt_valid(w_dtype)) return fail(SQLLM_EINVAL, "w_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", w_dtype);
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3))
        return fail(SQLLM_EINVAL, "qweight and lookup_table must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(w) & 15) return fail(SQLLM_EINVAL, "w must be 16-byte aligned");
    void (*kern)(const dq::PD);
    if (w_dtype == SQLLM_DT_F32) kern = a->bits == 4 ? dq::dequant_kernel<4, float> : dq::dequant_kernel<3, float>;
    else if (w_dtype == SQLLM_DT_F16) kern = a->bits == 4 ? dq::dequant_kernel<4, __half> : dq::dequant_kernel<3, __half>;
    else kern = a->bits == 4 ? dq::dequant_kernel<4, __nv_bfloat16> : dq::dequant_kernel<3, __nv_bfloat16>;
    if ((rc = dev_setup({{kern, dq::SMEM}}))) return rc;
    dq::PD p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.K = a->in_features; p.N = a->out_features; p.c0 = col0; p.n = ncols; p.w = w;
    const dim3 grid((ncols + dq::BN - 1) / dq::BN, (a->in_features + dq::BK - 1) / dq::BK);
    kern<<<grid, dq::THREADS, dq::SMEM, static_cast<cudaStream_t>(stream)>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "dequantize launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_fisher_accumulate(const void *x, const void *dy, int dtype, int rows, int seq_len, int in_features, int out_features,
                            float *fisher, void *stream) {
    if (dtype != SQLLM_DT_F16 && dtype != SQLLM_DT_BF16)
        return fail(SQLLM_EINVAL, "fisher_accumulate: dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", dtype);
    if (rows < 1) return fail(SQLLM_EINVAL, "fisher_accumulate: rows=%d must be >= 1", rows);
    if (seq_len < 1) return fail(SQLLM_EINVAL, "fisher_accumulate: seq_len=%d must be >= 1", seq_len);
    if (rows % seq_len) return fail(SQLLM_EINVAL, "fisher_accumulate: rows=%d must be a multiple of seq_len=%d", rows, seq_len);
    if (in_features < 1 || in_features % 8)
        return fail(SQLLM_EINVAL, "fisher_accumulate: in_features=%d must be a positive multiple of 8", in_features);
    if (out_features < 1 || out_features % 8)
        return fail(SQLLM_EINVAL, "fisher_accumulate: out_features=%d must be a positive multiple of 8", out_features);
    if ((out_features + fis::TN - 1) / fis::TN > 65535)
        return fail(SQLLM_EINVAL, "fisher_accumulate: out_features=%d exceeds %d", out_features, 65535 * fis::TN);
    if (!x || !dy || !fisher) return fail(SQLLM_EINVAL, "fisher_accumulate: x / dy / fisher must not be null");
    if (((uintptr_t)x | (uintptr_t)dy | (uintptr_t)fisher) & 15)
        return fail(SQLLM_EINVAL, "fisher_accumulate: x / dy / fisher must be 16-byte aligned");
    void (*kern)(const fis::PF) = dtype == SQLLM_DT_BF16 ? fis::fisher_kernel<true> : fis::fisher_kernel<false>;
    const int rc = dev_setup({{kern, fis::SMEM}});
    if (rc) return rc;
    fis::PF p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.dy = dy; p.f = fisher;
    p.rows = rows; p.T = seq_len; p.K = in_features; p.N = out_features;
    const dim3 grid((in_features + fis::TK - 1) / fis::TK, (out_features + fis::TN - 1) / fis::TN);
    // a cluster of one, not PDL: the kernel does not wait on the grid dependency, it reads x, dy and F as the previous kernel left them
    const cudaError_t e = launch_ex(kern, grid, fis::THREADS, fis::SMEM, static_cast<cudaStream_t>(stream), cluster_of(1), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "fisher_accumulate launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_unpack_indices(int bits, const int32_t *qweight, int in_features, int out_features, uint8_t *idx, void *stream) {
    if ((bits != 3 && bits != 4) || !qweight || !idx || in_features % 32 || in_features <= 0 || out_features <= 0)
        return fail(SQLLM_EINVAL, "bad arguments to sqllm_unpack_indices");
    unpack_kernel<<<1024, 256, 0, static_cast<cudaStream_t>(stream)>>>(bits, reinterpret_cast<const uint32_t *>(qweight),
                                                                       in_features, out_features, idx);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "unpack launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

// ---- weighted 1-D k-means and the GPU pack (kmeans1d.cuh) ----------------------------------------------------------------
namespace {
constexpr size_t KM_BUDGET = (size_t)512 << 20;  // workspace rows are chunked to about this many bytes

size_t km_align(size_t b) { return (b + 255) & ~(size_t)255; }

size_t km_row_bytes(int n, int k) {
    const size_t n1 = (size_t)n + 1;
    return 2 * sizeof(float) * n + (3 + 2) * sizeof(double) * n1 + (size_t)(k - 1) * sizeof(uint16_t) * n1;
}

int km_chunk(int rows, int n, int k) { return (int)std::max<size_t>(1, std::min<size_t>(rows, KM_BUDGET / km_row_bytes(n, k))); }

struct KmLayout {
    size_t offs, keys, vals, pref, d, opt, temp, temp_bytes, total;
};

int km_check(int rows, int n, int k) {
    if (rows < 1) return fail(SQLLM_EINVAL, "kmeans1d: rows=%d must be >= 1", rows);
    if (k < 2 || k > km::MAX_K) return fail(SQLLM_EINVAL, "kmeans1d: k=%d must be in [2, %d]", k, km::MAX_K);
    if (n < k || n > km::MAX_N) return fail(SQLLM_EINVAL, "kmeans1d: n=%d must be in [k=%d, %d]", n, k, km::MAX_N);
    return SQLLM_OK;
}

int km_layout(int rows, int n, int k, KmLayout &L) {
    const int C = km_chunk(rows, n, k);
    const size_t n1 = (size_t)n + 1, items = (size_t)C * n;
    size_t temp = 0;
    const cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(nullptr, temp, (const float *)nullptr, (float *)nullptr,
                                                                   (const float *)nullptr, (float *)nullptr, (int)items, C,
                                                                   (const int *)nullptr, (const int *)nullptr);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d: sort workspace query failed: %s", cudaGetErrorString(e));
    size_t o = 0;
    L.offs = o; o += km_align(sizeof(int) * (C + 1));
    L.keys = o; o += km_align(sizeof(float) * items);
    L.vals = o; o += km_align(sizeof(float) * items);
    L.pref = o; o += km_align(3 * sizeof(double) * n1 * C);
    L.d = o; o += km_align(2 * sizeof(double) * n1 * C);
    L.opt = o; o += km_align((size_t)(k - 1) * sizeof(uint16_t) * n1 * C);
    L.temp = o; L.temp_bytes = temp; o += km_align(temp);
    L.total = o;
    return SQLLM_OK;
}
}  // namespace

int sqllm_kmeans1d_workspace_bytes(int rows, int n, int k, size_t *bytes) {
    if (!bytes) return fail(SQLLM_EINVAL, "kmeans1d_workspace_bytes: bytes must not be null");
    int rc = km_check(rows, n, k);
    if (rc) return rc;
    KmLayout L;
    if ((rc = km_layout(rows, n, k, L))) return rc;
    *bytes = L.total;
    return SQLLM_OK;
}

int sqllm_kmeans1d(const float *w, const float *s, int rows, int n, int k, float *centroids, uint8_t *labels, void *workspace,
                   size_t workspace_bytes, void *stream) {
    int rc = km_check(rows, n, k);
    if (rc) return rc;
    if (!w || !s || !centroids || !labels) return fail(SQLLM_EINVAL, "kmeans1d: w / s / centroids / labels must not be null");
    if (((uintptr_t)w | (uintptr_t)s | (uintptr_t)centroids) & 3) return fail(SQLLM_EINVAL, "kmeans1d: w / s / centroids must be 4-byte aligned");
    if (!workspace) return fail(SQLLM_EWORKSPACE, "kmeans1d: workspace must not be null");
    if ((uintptr_t)workspace & 255) return fail(SQLLM_EINVAL, "kmeans1d: workspace must be 256-byte aligned");
    KmLayout L;
    if ((rc = km_layout(rows, n, k, L))) return rc;
    if (workspace_bytes < L.total)
        return fail(SQLLM_EWORKSPACE, "kmeans1d: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    char *ws = static_cast<char *>(workspace);
    int *offs = reinterpret_cast<int *>(ws + L.offs);
    float *keys = reinterpret_cast<float *>(ws + L.keys), *vals = reinterpret_cast<float *>(ws + L.vals);
    const int C = km_chunk(rows, n, k);
    km::segment_offsets_kernel<<<(C + 256) / 256, 256, 0, st>>>(offs, C, n);
    for (int r0 = 0; r0 < rows; r0 += C) {
        const int c = std::min(C, rows - r0);
        const size_t at = (size_t)r0 * n;
        size_t temp = L.temp_bytes;
        cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(ws + L.temp, temp, w + at, keys, s + at, vals, c * n, c, offs,
                                                                 offs + 1, 0, 32, st);
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d: segmented sort failed: %s", cudaGetErrorString(e));
        km::kmeans1d_kernel<<<c, km::THREADS, 0, st>>>(keys, vals, w + at, n, k, reinterpret_cast<double *>(ws + L.pref),
                                                       reinterpret_cast<double *>(ws + L.d), reinterpret_cast<uint16_t *>(ws + L.opt),
                                                       centroids + (size_t)r0 * k, labels + at);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d launch failed: %s", cudaGetErrorString(e));
    }
    return SQLLM_OK;
}

int sqllm_pack_indices(int bits, const uint8_t *labels, int in_features, int out_features, int32_t *qweight, void *stream) {
    if (bits != 3 && bits != 4) return fail(SQLLM_EINVAL, "pack_indices: bits=%d must be 3 or 4", bits);
    if (in_features <= 0 || in_features % 32)
        return fail(SQLLM_EINVAL, "pack_indices: in_features=%d must be a positive multiple of 32", in_features);
    if (out_features <= 0) return fail(SQLLM_EINVAL, "pack_indices: out_features=%d must be >= 1", out_features);
    if (!labels || !qweight) return fail(SQLLM_EINVAL, "pack_indices: labels / qweight must not be null");
    if ((uintptr_t)qweight & 3) return fail(SQLLM_EINVAL, "pack_indices: qweight must be 4-byte aligned");
    const size_t work = (size_t)in_features / 32 * out_features;
    const int grid = (int)std::min<size_t>(4096, (work + 255) / 256);
    km::pack_indices_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(bits, labels, in_features, out_features,
                                                                                 reinterpret_cast<uint32_t *>(qweight));
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "pack_indices launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

// ---- the reference's 12 launchers -----------------------------------------------------------------
static int run12(int bits, const float *vec, const int32_t *mat, float *mul, const float *lut, int height, int width,
                 int batch, int vec_height, const int32_t *rows, const int32_t *cols, const float *vals, int num_rows,
                 const float *full_rows, const int32_t *fri, int fr_height, int fr_width, void *stream) {
    sqllm_lutgemv_args a;
    memset(&a, 0, sizeof(a));
    a.bits = bits;
    if (height <= 0 || height % bits) return fail(SQLLM_EINVAL, "height=%d is not a multiple of bits=%d", height, bits);
    a.in_features = height / bits * 32;
    a.out_features = width;
    a.batch = batch;
    if (vec_height >= 0 && vec_height != a.in_features)
        return fail(SQLLM_EINVAL, "vec has %d features, packed matrix implies %d", vec_height, a.in_features);
    if (rows && num_rows != width) return fail(SQLLM_EINVAL, "num_rows=%d must equal the matrix width %d", num_rows, width);
    if (full_rows && fr_height != a.in_features)
        return fail(SQLLM_EINVAL, "full_rows has %d rows, expected in_features=%d", fr_height, a.in_features);
    a.qweight = mat; a.lookup_table = lut; a.vec = vec; a.mul = mul;
    a.rows = rows; a.cols = cols; a.vals = vals;
    a.full_rows = full_rows; a.full_row_indices = fri; a.topX = full_rows ? fr_width : 0;
    return sqllm_lutgemv(&a, stream);
}

int sqllm_vecquant3matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul, const float *lut, int height,
                                         int width, void *stream) {
    return run12(3, vec, mat, mul, lut, height, width, 1, -1, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul, const float *lut, int height,
                                         int width, void *stream) {
    return run12(4, vec, mat, mul, lut, height, width, 1, -1, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul, const float *lut,
                                                 int height, int width, int batch, int vec_height, void *stream) {
    return run12(3, vec, mat, mul, lut, height, width, batch, vec_height, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul, const float *lut,
                                                 int height, int width, int batch, int vec_height, void *stream) {
    return run12(4, vec, mat, mul, lut, height, width, batch, vec_height, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat, const float *vec,
                                              float *mul, int num_rows, const int32_t *mat3, const float *lut, int height,
                                              int width, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat, const float *vec,
                                              float *mul, int num_rows, const int32_t *mat4, const float *lut, int height,
                                              int width, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows, const int32_t *mat3,
                                                      const float *lut, int height, int width, int batch, int vec_height,
                                                      void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows, const int32_t *mat4,
                                                      const float *lut, int height, int width, int batch, int vec_height,
                                                      void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows, const int32_t *fri,
                                                     float *mul, int num_rows, const int32_t *mat3, const float *lut,
                                                     int height, int width, int fr_height, int fr_width, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows, const int32_t *fri,
                                                     float *mul, int num_rows, const int32_t *mat4, const float *lut,
                                                     int height, int width, int fr_height, int fr_width, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                             const float *vec, const float *full_rows, const int32_t *fri,
                                                             float *mul, int num_rows, const int32_t *mat3, const float *lut,
                                                             int height, int width, int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                             const float *vec, const float *full_rows, const int32_t *fri,
                                                             float *mul, int num_rows, const int32_t *mat4, const float *lut,
                                                             int height, int width, int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}

}  // extern "C"
