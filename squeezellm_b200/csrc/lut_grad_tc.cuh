// lut_grad_tc.cuh - the tile of G = x^T . dy on the tensor cores (wgmma) for sqllm_lut_grad when x and dy are both fp16 or both
// bf16.  Included by lutgemv_kernels.cu inside its anonymous namespace, after lut_grad.cuh (plan, epilogue, cluster reduction)
// and lutgemm_tc_t.cuh (MN-major descriptor).
//
// Per k-tile the CTA walks M in chunks of 64 rows, double-buffered with cp.async:
//   * x [64 m x 128 k] is the A operand and dy [64 m x 128 c] the B operand, both stored as they lie in memory - contiguous along
//     k and c, the MMA's M and N - in the 128-byte-swizzled MN-major layout (rows of 64 values, 8-row groups 1024 bytes apart,
//     the next 64 values 8 KB further) and read with imm-trans-a = imm-trans-b = 1.  Rows past M and values past K / N are
//     zero-filled; operands whose rows are not 16-byte multiples are staged with 2-byte loads.
//   * warpgroup g issues wgmma m64n128k16 for the inputs [64 g, 64 g + 64) of the tile: four k-steps (16 rows each) per chunk.
// Both operands are 16-bit values, so every product is exact in fp32: one MMA pass per chunk, no split.  Each chunk's MMAs start
// from zero and the chunk's result is added into a running fp32 sum with FADD (the promotion of lutgemm_tc.cuh): the tensor core's
// own accumulation never sees more than 64 products per output.
#pragma once

namespace lgt {

using lg::TK;
using lg::TC;
using lg::THREADS;
using lg::GST;
constexpr int MC = 64;                        // rows per chunk
constexpr int OP_BYTES = MC * 128 * 2;        // one operand chunk: 16 KB, two 8 KB atoms of 64 values
constexpr int XS = 0, DS = 2 * OP_BYTES, GSO = 4 * OP_BYTES, BINS = GSO + lg::G_BYTES;
constexpr int SMEM = BINS + lg::BIN_BYTES + 1024;  // + alignment of the swizzled tiles to 1024 bytes

// d[64] (+)= A[64 x 16] . B[16 x 128]; A and B MN-major (imm-trans-a = imm-trans-b = 1)
template <bool BF>
__device__ __forceinline__ void wgmma_tt(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
#define SQ_WGMMA_TT(TY)                                                                                                                 \
    asm volatile(                                                                                                                      \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                                   \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                                  \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "    \
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, " \
        "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n}\n"                              \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),      \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),        \
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),        \
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),        \
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])         \
        : "l"(da), "l"(db), "r"(scale_d))
    if constexpr (BF) SQ_WGMMA_TT("bf16");
    else SQ_WGMMA_TT("f16");
#undef SQ_WGMMA_TT
}

// 64 rows x 128 16-bit values of a row-major matrix (leading dimension ld, src at the chunk's first row and the tile's first value)
// into the MN-major layout at dst: row r < r_lim and value c < c_lim, else zero
__device__ __forceinline__ void stage(uint32_t dst, const unsigned short *src, int ld, int r_lim, int c_lim, bool al16) {
#pragma unroll
    for (int u = 0; u < MC * 16 / THREADS; ++u) {
        const int t = threadIdx.x + u * THREADS, r = t >> 4, ch = t & 15, c = 8 * ch;
        const uint32_t d = dst + (uint32_t)((ch >> 3) * 8192 + r * 128 + (((ch & 7) ^ (r & 7)) << 4));
        const bool ok = r < r_lim && c < c_lim;
        if (al16) {
            cp_async16_clip(d, ok ? src + (size_t)r * ld + c : src, ok ? 2 * min(8, c_lim - c) : 0);
        } else {
            uint32_t v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const unsigned short *s = src + (size_t)r * ld + c + 2 * e;
                const uint32_t lo = (ok && c + 2 * e < c_lim) ? (uint32_t)__ldg(s) : 0u;
                const uint32_t hi = (ok && c + 2 * e + 1 < c_lim) ? (uint32_t)__ldg(s + 1) : 0u;
                v[e] = lo | (hi << 16);
            }
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(d), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
        }
    }
}

template <int BITS, bool BF>
__global__ void __launch_bounds__(THREADS, 1) lut_grad_tc_kernel(const lg::PG p) {
    constexpr int L = 1 << BITS;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t sb = (raw + 1023u) & ~1023u;
    unsigned char *sm = smem_raw + (sb - raw);
    float *gs = reinterpret_cast<float *>(sm + GSO);
    float *bins = reinterpret_cast<float *>(sm + BINS);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = warp >> 2, wi = warp & 3;  // warpgroup: inputs [64 g, 64 g + 64) of the tile
    const uint32_t rank = rows::cluster_rank();
    const int S = (int)gridDim.x;  // = cluster size
    const int n0 = blockIdx.y * TC;
    int t_lo, t_hi;
    lg::slab(p.ktiles, (int)rank, S, t_lo, t_hi);
    for (int e = tid; e < L * TC; e += THREADS) bins[e] = 0.f;

    const unsigned short *x = static_cast<const unsigned short *>(p.x), *dy = static_cast<const unsigned short *>(p.dy);
    const int nch = (p.M + MC - 1) / MC;
    auto load = [&](int i, int b, int k0) {
        const int m0 = i * MC;
        stage(sb + XS + b * OP_BYTES, x + (size_t)m0 * p.K + k0, p.K, p.M - m0, p.K - k0, p.x_al16);
        stage(sb + DS + b * OP_BYTES, dy + (size_t)m0 * p.N + n0, p.N, p.M - m0, p.N - n0, p.dy_al16);
        cp_async_commit();
    };

    for (int t = t_lo; t < t_hi; ++t) {
        const int k0 = t * TK;
        load(0, 0, k0);
        cp_async_wait_all();
        tc::fence_proxy_async();
        __syncthreads();
        float acc[64], sum[64];
#pragma unroll
        for (int r = 0; r < 64; ++r) { acc[r] = 0.f; sum[r] = 0.f; }
        for (int i = 0; i < nch; ++i) {
            const int b = i & 1;
            const uint32_t xa = sb + XS + b * OP_BYTES + g * 8192, db = sb + DS + b * OP_BYTES;
            tc::wgmma_fence();
#pragma unroll
            for (int s = 0; s < MC / 16; ++s) wgmma_tt<BF>(acc, tct::mn_desc(xa + 2048 * s), tct::mn_desc(db + 2048 * s), s > 0);
            tc::wgmma_commit();
            if (i + 1 < nch) load(i + 1, b ^ 1, k0);
            tc::wgmma_wait_all();
#pragma unroll
            for (int r = 0; r < 64; ++r) {
                asm volatile("" : "+f"(acc[r])::"memory");
                sum[r] += acc[r];
            }
            cp_async_wait_all();
            tc::fence_proxy_async();
            __syncthreads();
        }
        // stage the tile of G: fragment (n, i, j) of lane l in warp wi of group g is input 64 g + 16 wi + l/4 + 8 i, channel
        // 8 n + 2 (l % 4) + j
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float *row = gs + (64 * g + 16 * wi + (lane >> 2) + 8 * i) * GST + 2 * (lane & 3);
#pragma unroll
            for (int n = 0; n < TC / 8; ++n) *reinterpret_cast<float2 *>(row + 8 * n) = make_float2(sum[4 * n + 2 * i], sum[4 * n + 2 * i + 1]);
        }
        __syncthreads();
        lg::tile_epilogue<BITS>(p, gs, bins, k0, n0, rank == 0 && t == t_lo);
        __syncthreads();
    }
    lg::reduce_bins<BITS>(p, bins, n0, rank, S);
}

}  // namespace lgt
