// common.cuh - what every kernel of the library shares: the fused-path limits and the layout of the fused workspace header, the PTX
// wrappers (shared-memory loads, cp.async, mbarrier, TMA, PDL, named barriers, cluster rank), fp32 pair math, the 16-bit conversions,
// the 3-bit field decode of the exact-table GEMVs (v1 and v2) and the TRACE time stamps of -DSQLLM_TRACE builds.
#pragma once
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint, no -lcuda)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "sqllm_b200.h"

namespace {

constexpr int STRIP = 64;                 // output columns per strip (16 lanes x 4 columns)
constexpr int MAX_TOPX_FUSED = SQLLM_FUSED_MAX_TOPX;
constexpr int MAX_STRIPS = 16320;         // per-strip tickets in the workspace header (out_features <= 1,044,480)
constexpr int MAX_N_FUSED = SQLLM_FUSED_MAX_OUT;  // fused path: the scratch accumulator lives at a fixed place in the workspace
constexpr size_t WS_ACC_OFF = 65536;       // [64 KB, 64 KB + 4*MAX_N_FUSED): fp32 accumulator (zero between launches)
constexpr int MAX_GRID_V2 = 256;           // v2 runs one CTA per SM
constexpr size_t WS_HBOX_OFF = WS_ACC_OFF + (size_t)MAX_N_FUSED * 4;       // v2 mailboxes: [MAX_GRID_V2][64] x 8 bytes (partial strip sums)
constexpr size_t WS_CBOX_OFF = WS_HBOX_OFF + (size_t)MAX_GRID_V2 * 64 * 8;  // ... and [MAX_N_FUSED] x 8 bytes (outlier row sums); zero between launches
constexpr size_t WS_DBOX_OFF = WS_CBOX_OFF + (size_t)MAX_N_FUSED * 8;          // ... and [MAX_TOPX_FUSED][MAX_GRID_V2] x 8 bytes (dense-row parts, one per contributing CTA)
constexpr size_t WS_HEADER = WS_DBOX_OFF + (size_t)MAX_TOPX_FUSED * MAX_GRID_V2 * 8;  // tickets + accumulator + mailboxes: never shared with data of any shape

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

// thread-block clusters: the multi-row GEMV, the transposed LUT-GEMM and the codebook gradient split K (or N) over a cluster
namespace rows {
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ float4 ld_cluster_v4(uint32_t local, uint32_t rank) {  // the same shared address in CTA `rank` of the cluster
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local), "r"(rank));
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
}  // namespace rows

}  // namespace
