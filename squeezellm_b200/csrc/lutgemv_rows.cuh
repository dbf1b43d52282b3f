// lutgemv_rows.cuh - the multi-row LUT-GEMV behind sqllm_lutgemv_rows_dt: a few fp16 or bf16 rows (decode of several sequences,
// speculative-decoding verification, short prompts) in ONE launch.  It shares the table layout, decode and row FMAs
// (batched::unit_fma) of lutgemm_batched.cuh.
//
//   y[m][c] = sum_k W[k][c] x[m][k] + CSR + dense rows (+ bias),  fp16 or bf16 x [M][K] (XT), y fp32 or x's type, exact fp32
//   codebook, fp32 sums.
//
// Tiling: a CTA owns one 64-column strip, one K-slab and one group of RB rows; grid (S, strips, ceil(M / RB)), launched as clusters of
// (S, 1, 1): the S CTAs of a cluster split the strip's K.  S comes from K, N and the SM count only (rows_plan), never from M, and
// every row runs the same instructions whatever RB is, so a row's result does not depend on M or on the other rows.
//   * x: the CTA stages its slab of its rows, converted to fp32 (exact for both types), rows padded to an even number of units with
//     zeros.  Nothing after the staging depends on x's type.
//   * weights: each lane reads its 16 bytes per unit row straight from global memory, one position ahead (as lutgemm_batched_kernel),
//     decodes its 4 columns x one unit once and runs them against all RB rows.
//   * outliers, folded per slab: the CSR entries of the strip's 64 channels whose column lies in the slab (gathered from the staged
//     x), and the dense rows whose channel lies in the strip, over the slab.  No limit on topX or on the entries of a CSR row;
//     duplicate dense-row channels add up, channels outside [0, N) and CSR columns outside [0, K) are ignored.
//   * reduction: every CTA leaves partial[RB][64] in its shared memory; after a cluster barrier the leader (rank 0) reads the
//     peers' partials over DSMEM in rank order, adds the bias, converts and stores y once; a second cluster barrier keeps the
//     peers' shared memory alive until then.  No workspace, no atomics, no spin-waits: bit-reproducible, safe on several streams,
//     CUDA-graph capturable.
#pragma once
#include "common.cuh"
#include "lutgemm_batched.cuh"

namespace {

namespace rows {

constexpr int RW = 8;                 // warps per CTA
constexpr int RTHREADS = RW * 32;
constexpr int CSR_SPLIT = RTHREADS / STRIP;  // threads that walk one channel's CSR entries (interleaved), summed in a fixed order
constexpr int SLAB_GOAL = 2048;       // inputs per slab the plan aims below (x of 8 rows: 64 KB, two CTAs per SM)
constexpr int MAX_SLABS = 8;          // S <= 8: portable cluster size

struct PR {
    const uint32_t *qw;
    const float *lut;
    const void *x;      // [M][K], fp16 or bf16 (the kernel's XT)
    void *y;            // [M][N], fp32 or XT
    const float *bias;  // may be null
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX;
    int K, N, M, R;     // R = units per strip
    int ks;             // units per slab
    int kpad;           // floats per staged x row: ks rounded up to an even number of units
    int y_16;           // y is XT, not fp32
    int qw_al16;        // qweight is 16-byte aligned: 16-byte weight loads
};

// shared-memory carve-up behind the table (which is aligned to its own size), in bytes; host and device use the same numbers
template <int BITS, int RB>
struct SR {
    using C = batched::CB<BITS>;
    __host__ __device__ static int xpitch(int kpad) { return kpad * 4 + 16; }  // +16: the RB rows a lane reads start in different banks
    __host__ __device__ static int off_part(int kpad) { return C::TAB + RB * xpitch(kpad); }              // [RW][RB][STRIP]
    __host__ __device__ static int off_csum(int kpad) { return off_part(kpad) + RW * RB * STRIP * 4; }   // [CSR_SPLIT][RB][STRIP]
    __host__ __device__ static int off_partial(int kpad) { return off_csum(kpad) + CSR_SPLIT * RB * STRIP * 4; }  // [RB][STRIP]
    __host__ __device__ static int off_red(int kpad) { return off_partial(kpad) + RB * STRIP * 4; }      // [RW][RB]
    // + C::TAB of slack: the table is aligned up from wherever dynamic shared memory starts
    __host__ __device__ static int total(int kpad) { return C::TAB + off_red(kpad) + RW * RB * 4; }
};

template <int BITS, int RB, typename XT>
__global__ void __launch_bounds__(RTHREADS, 2) lutgemv_rows_kernel(const PR p) {
    using C = batched::CB<BITS>;
    using L = SR<BITS, RB>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t tab = (raw + (uint32_t)C::TAB - 1u) & ~((uint32_t)C::TAB - 1u);
    unsigned char *sm = smem_raw + (tab - raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, i16 = lane & 15, jsel = lane >> 4;
    const uint32_t rank = cluster_rank();
    const int S = (int)gridDim.x;  // = cluster size
    const int strip = blockIdx.y, b0 = blockIdx.z * RB;
    const int u_lo = (int)rank * p.ks, nu = max(0, min(p.R, u_lo + p.ks) - u_lo);
    const int k_lo = u_lo * C::XU, kn = nu * C::XU;  // this slab: inputs [k_lo, k_lo + kn)
    const uint32_t xpitch = (uint32_t)L::xpitch(p.kpad), xs = tab + C::TAB;
    const int xrow = (int)xpitch / 4;  // floats per staged x row
    const float *xsf = reinterpret_cast<const float *>(sm + C::TAB);
    float *part = reinterpret_cast<float *>(sm + L::off_part(p.kpad));
    float *csum = reinterpret_cast<float *>(sm + L::off_csum(p.kpad));
    float *partial = reinterpret_cast<float *>(sm + L::off_partial(p.kpad));
    float *red = reinterpret_cast<float *>(sm + L::off_red(p.kpad));

    // ---- table (exact fp32, [value][slot], slot ((c & 3) << 4) | (c >> 2)) and the x rows of this slab, fp32 ----
    for (int it = tid; it < STRIP * C::L; it += RTHREADS) {
        const int c = it / C::L, v = it - c * C::L;
        const int col = strip * STRIP + c;
        reinterpret_cast<float *>(sm)[v * STRIP + (((c & 3) << 4) | (c >> 2))] = col < p.N ? __ldg(p.lut + (size_t)col * C::L + v) : 0.f;
    }
    {
        const int n8 = p.kpad / 8;  // pieces of 8 inputs per row; pieces past the slab (or rows past M) are zero
        for (int e = tid; e < RB * n8; e += RTHREADS) {
            const int b = e / n8, q = e - b * n8;
            float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
            if (b0 + b < p.M && 8 * q < kn) {
                const uint4 h = __ldg(reinterpret_cast<const uint4 *>(static_cast<const XT *>(p.x) + (size_t)(b0 + b) * p.K + k_lo + 8 * q));
                const float2 f0 = x16x2_to_f32x2<XT>(h.x), f1 = x16x2_to_f32x2<XT>(h.y);
                const float2 f2 = x16x2_to_f32x2<XT>(h.z), f3 = x16x2_to_f32x2<XT>(h.w);
                lo = make_float4(f0.x, f0.y, f1.x, f1.y);
                hi = make_float4(f2.x, f2.y, f3.x, f3.y);
            }
            float4 *dst = reinterpret_cast<float4 *>(sm + C::TAB + b * xpitch + 32 * q);
            dst[0] = lo;
            dst[1] = hi;
        }
    }
    __syncthreads();

    // ---- LUT-GEMM over the slab: warp w takes unit pairs 2w + jsel, step 2*RW; words are prefetched one position ahead ----
    float acc[RB][4];
#pragma unroll
    for (int b = 0; b < RB; ++b)
#pragma unroll
        for (int t = 0; t < 4; ++t) acc[b][t] = 0.f;
    uint32_t l[4];
    const uint32_t tb_hi = BITS == 4 ? (tab & 0xFFFF0000u) : tab;
#pragma unroll
    for (int t = 0; t < 4; ++t) l[t] = tb_hi | (uint32_t)((((t ^ jsel) << 4) | i16) << 2);
    const uint32_t segc = ((tab >> 8) & 0xF0u) * 0x01010101u;
    const int col0 = strip * STRIP + 4 * i16;
    const bool cvalid = col0 < p.N;
    auto load_unit = [&](int uu, uint4 (&w)[C::ROWS]) {
        const uint32_t *src = p.qw + (size_t)((u_lo + uu) * C::ROWS) * p.N + col0;
        const bool ok = uu < nu && cvalid;
#pragma unroll
        for (int r = 0; r < C::ROWS; ++r) {
            const uint32_t *s = src + (size_t)r * p.N;
            w[r] = !ok ? make_uint4(0u, 0u, 0u, 0u)
                       : p.qw_al16 ? ldg_stream(s) : make_uint4(__ldg(s), __ldg(s + 1), __ldg(s + 2), __ldg(s + 3));
        }
    };
    int u = 2 * warp + jsel;
    uint4 cur[C::ROWS], nxt[C::ROWS];
    load_unit(u, cur);
    // warp-uniform bound; with an odd unit count the last pair's second unit reads zero words against the zero x padding
    for (; u - jsel < nu; u += 2 * RW) {
        load_unit(u + 2 * RW, nxt);
        batched::unit_fma<BITS, RB>(acc, cur, jsel, l, segc, xs + (uint32_t)(u * C::XU * 4), xpitch);
#pragma unroll
        for (int r = 0; r < C::ROWS; ++r) cur[r] = nxt[r];
    }
    // fold the two half-warps (lane (i, j=1) holds column t^1 in slot t): one partial row per warp
#pragma unroll
    for (int b = 0; b < RB; ++b) {
        const float v0 = __shfl_xor_sync(0xffffffffu, acc[b][1], 16), v1 = __shfl_xor_sync(0xffffffffu, acc[b][0], 16);
        const float v2 = __shfl_xor_sync(0xffffffffu, acc[b][3], 16), v3 = __shfl_xor_sync(0xffffffffu, acc[b][2], 16);
        if (jsel == 0)
            *reinterpret_cast<float4 *>(part + ((warp * RB + b) * STRIP + 4 * i16)) = make_float4(acc[b][0] + v0, acc[b][1] + v1, acc[b][2] + v2, acc[b][3] + v3);
    }

    // ---- CSR entries of the strip's channels with their column in this slab: CSR_SPLIT threads per channel, interleaved ----
    if (p.rows) {
        const int c = tid & (STRIP - 1), q = tid / STRIP;
        const int col = strip * STRIP + c;
        float a[RB];
#pragma unroll
        for (int b = 0; b < RB; ++b) a[b] = 0.f;
        if (col < p.N) {
            const int e1 = __ldg(p.rows + col + 1);
#pragma unroll 4
            for (int e = __ldg(p.rows + col) + q; e < e1; e += CSR_SPLIT) {
                const int k = __ldg(p.cols + e) - k_lo;
                if ((unsigned)k < (unsigned)kn) {
                    const float v = __ldg(p.vals + e);
#pragma unroll
                    for (int b = 0; b < RB; ++b) a[b] = fmaf(v, xsf[b * xrow + k], a[b]);
                }
            }
        }
#pragma unroll
        for (int b = 0; b < RB; ++b) csum[(q * RB + b) * STRIP + c] = a[b];
    }
    __syncthreads();
    for (int e = tid; e < RB * STRIP; e += RTHREADS) {
        const int b = e / STRIP, c = e - b * STRIP;
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < RW; ++w) tot += part[(w * RB + b) * STRIP + c];
        if (p.rows) {
            float o = csum[b * STRIP + c];
#pragma unroll
            for (int q = 1; q < CSR_SPLIT; ++q) o += csum[(q * RB + b) * STRIP + c];
            tot += o;
        }
        partial[e] = tot;
    }

    // ---- dense rows whose channel lies in this strip, over the slab, in index order (duplicates add up) ----
    if (p.topX > 0) {
        __syncthreads();
        for (int j = 0; j < p.topX; ++j) {
            const int cj = __ldg(p.fri + j) - strip * STRIP;
            if ((unsigned)cj >= (unsigned)STRIP || strip * STRIP + cj >= p.N) continue;  // CTA-uniform
            float a[RB];
#pragma unroll
            for (int b = 0; b < RB; ++b) a[b] = 0.f;
#pragma unroll 4
            for (int k = tid; k < kn; k += RTHREADS) {
                const float f = __ldg(p.full_rows + (size_t)(k_lo + k) * p.topX + j);
#pragma unroll
                for (int b = 0; b < RB; ++b) a[b] = fmaf(f, xsf[b * xrow + k], a[b]);
            }
#pragma unroll
            for (int b = 0; b < RB; ++b) {
                const float s = warp_sum(a[b]);
                if (lane == 0) red[warp * RB + b] = s;
            }
            __syncthreads();
            if (tid < RB) {
                float s = red[tid];
#pragma unroll
                for (int w = 1; w < RW; ++w) s += red[w * RB + tid];
                partial[tid * STRIP + cj] += s;
            }
            __syncthreads();
        }
    }

    // ---- cluster reduction: the leader sums the S partials in rank order, adds the bias and stores y once ----
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
    if (rank == 0) {
        for (int e = tid; e < RB * (STRIP / 4); e += RTHREADS) {
            const int b = e / (STRIP / 4), c = 4 * (e - b * (STRIP / 4));
            const int row = b0 + b, col = strip * STRIP + c;
            if (row >= p.M || col >= p.N) continue;
            const uint32_t la = smem_u32(partial + b * STRIP + c);
            float4 s = ld_cluster_v4(la, 0);
            for (int r = 1; r < S; ++r) {
                const float4 t = ld_cluster_v4(la, (uint32_t)r);
                s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
            }
            if (p.bias) {
                s.x += __ldg(p.bias + col); s.y += __ldg(p.bias + col + 1); s.z += __ldg(p.bias + col + 2); s.w += __ldg(p.bias + col + 3);
            }
            const size_t o = (size_t)row * p.N + col;
            if (p.y_16) {
                uint2 v;
                if constexpr (std::is_same<XT, __nv_bfloat16>::value) {
                    const __nv_bfloat162 h01 = __floats2bfloat162_rn(s.x, s.y), h23 = __floats2bfloat162_rn(s.z, s.w);
                    v.x = *reinterpret_cast<const uint32_t *>(&h01);
                    v.y = *reinterpret_cast<const uint32_t *>(&h23);
                } else {
                    const __half2 h01 = __floats2half2_rn(s.x, s.y), h23 = __floats2half2_rn(s.z, s.w);
                    v.x = *reinterpret_cast<const uint32_t *>(&h01);
                    v.y = *reinterpret_cast<const uint32_t *>(&h23);
                }
                *reinterpret_cast<uint2 *>(static_cast<XT *>(p.y) + o) = v;
            } else {
                *reinterpret_cast<float4 *>(static_cast<float *>(p.y) + o) = s;
            }
        }
    }
    asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;" ::: "memory");
}

}  // namespace rows

}  // namespace
