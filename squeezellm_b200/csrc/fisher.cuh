// fisher.cuh - the diagonal of the empirical Fisher information of a linear layer on the tensor cores (wgmma), behind
// sqllm_fisher_accumulate.  It uses the MN-major staging (lgt::stage) and wgmma (lgt::wgmma_tt) of lut_grad_tc.cuh
// and the descriptor of lutgemm_tc_t.cuh (tct::mn_desc).
//
//   F[n][k] += sum_s g_s[n][k]^2,   g_s = dy_s^T x_s   (sample s: rows [s T, s T + T) of x [rows, K] and dy [rows, N])
//
// A CTA owns one 128 (n) x 128 (k) tile of F and walks the samples in ascending order, each in chunks of 64 rows that never cross
// the sample's end (rows past it are zero-filled), NST chunks in flight with cp.async:
//   * dy [64 rows x 128 n] is the A operand and x [64 rows x 128 k] the B operand, both as they lie in memory - contiguous along n
//     and k, the MMA's M and N - in lgt::stage's 128-byte-swizzled MN-major layout, read with imm-trans-a = imm-trans-b = 1;
//   * warpgroup g issues wgmma m64n128k16 for the channels [64 g, 64 g + 64) of the tile: four k-steps (16 rows each) per chunk.
// 16-bit products are exact in fp32.  Each chunk's MMAs start from zero and the chunk's result is added into the sample's running
// fp32 sum with FADD (the promotion of lutgemm_tc.cuh): the tensor core's own accumulation never sees more than 64 products.  At
// the sample's last chunk each thread squares its 64 sums into its 64 F slots (one FFMA each, in registers) and clears the sums.
// After the last sample the tile is added to F in global memory: every element read once and written once, by one thread, in a
// fixed order.  The tile is 128 x 128 because the promotion costs a second accumulator: acc, sum and the F tile are 3 x 64
// registers per thread, which leaves room for addressing under the 255-register limit of one 256-thread CTA per SM.
#pragma once
#include "common.cuh"
#include "lut_grad_tc.cuh"
#include "lutgemm_tc.cuh"
#include "lutgemm_tc_t.cuh"

namespace {

namespace fis {

constexpr int TN = 128, TK = 128;                  // F tile: 128 output channels x 128 inputs
constexpr int THREADS = lgt::THREADS;              // two warpgroups (lgt::stage spreads a chunk over this many threads)
constexpr int MC = lgt::MC;                        // rows per chunk
constexpr int NST = 4;                             // chunks in flight
constexpr int STAGE_BYTES = 2 * lgt::OP_BYTES;     // dy chunk, then x chunk: 32 KB
constexpr int SMEM = NST * STAGE_BYTES + 1024;     // + alignment of the swizzled tiles to 1024 bytes

struct PF {
    const void *x, *dy;  // [rows][K], [rows][N]: fp16 or bf16, rows 16-byte aligned
    float *f;            // [N][K]
    int rows, T, K, N;
};

template <bool BF>
__global__ void __launch_bounds__(THREADS, 1) fisher_kernel(const PF p) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = warp >> 2, wi = warp & 3;  // warpgroup: channels [64 g, 64 g + 64) of the tile
    const int k0 = blockIdx.x * TK, n0 = blockIdx.y * TN;
    const unsigned short *x = static_cast<const unsigned short *>(p.x), *dy = static_cast<const unsigned short *>(p.dy);
    const int cps = (p.T + MC - 1) / MC;  // chunks per sample
    const int nch = p.rows / p.T * cps;

    auto load = [&](int i) {  // chunk i into stage i % NST; one commit group per call, empty past the last chunk
        if (i < nch) {
            const int s = i / cps, c = i - s * cps;
            const size_t m0 = (size_t)s * p.T + (size_t)c * MC;
            const uint32_t b = sb + (uint32_t)((i % NST) * STAGE_BYTES);
            lgt::stage(b, dy + m0 * p.N + n0, p.N, p.T - c * MC, p.N - n0, true);
            lgt::stage(b + lgt::OP_BYTES, x + m0 * p.K + k0, p.K, p.T - c * MC, p.K - k0, true);
        }
        cp_async_commit();
    };

    float acc[64], sum[64], f[64];
#pragma unroll
    for (int r = 0; r < 64; ++r) { acc[r] = 0.f; sum[r] = 0.f; f[r] = 0.f; }
#pragma unroll
    for (int j = 0; j < NST - 1; ++j) load(j);
    int c = 0;  // chunk of the current sample
    for (int i = 0; i < nch; ++i) {
        cp_async_wait_pending<NST - 2>();  // this thread's copies of chunk i have landed
        tc::fence_proxy_async();
        __syncthreads();                   // ... and every thread's; every warpgroup is done with chunk i - 1's stage
        load(i + NST - 1);                 // into that stage
        const uint32_t b = sb + (uint32_t)((i % NST) * STAGE_BYTES);
        tc::wgmma_fence();
#pragma unroll
        for (int s = 0; s < MC / 16; ++s)
            lgt::wgmma_tt<BF>(acc, tct::mn_desc(b + g * 8192 + 2048 * s), tct::mn_desc(b + lgt::OP_BYTES + 2048 * s), s > 0);
        tc::wgmma_commit();
        tc::wgmma_wait_all();
#pragma unroll
        for (int r = 0; r < 64; ++r) {
            asm volatile("" : "+f"(acc[r])::"memory");
            sum[r] += acc[r];
        }
        if (++c == cps) {  // the sample's last chunk: F += g_s^2
            c = 0;
#pragma unroll
            for (int r = 0; r < 64; ++r) {
                f[r] = fmaf(sum[r], sum[r], f[r]);
                sum[r] = 0.f;
            }
        }
    }
    cp_async_wait_all();

    // fragment (n, i, j) of lane l in warp wi of group g is channel n0 + 64 g + 16 wi + l/4 + 8 i, input k0 + 8 n + 2 (l % 4) + j
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = n0 + 64 * g + 16 * wi + (lane >> 2) + 8 * i;
        if (row >= p.N) continue;
        float *dst = p.f + (size_t)row * p.K + k0 + 2 * (lane & 3);
#pragma unroll
        for (int n = 0; n < TK / 8; ++n) {
            if (k0 + 8 * n + 2 * (lane & 3) >= p.K) continue;  // K is even: the pair is in range or out of it
            float2 v = *reinterpret_cast<const float2 *>(dst + 8 * n);
            v.x += f[4 * n + 2 * i];
            v.y += f[4 * n + 2 * i + 1];
            *reinterpret_cast<float2 *>(dst + 8 * n) = v;
        }
    }
}

}  // namespace fis

}  // namespace
