// lutgemm_tc_t.cuh - the transposed LUT-GEMM on the tensor cores (wgmma), behind sqllm_lutgemm_t's tensor-core path: the input
// gradient of QuantLinearLUT for fp16 or bf16 dy.  Included by lutgemv_kernels.cu inside its anonymous namespace, after
// lutgemm_tc.cuh, whose operand layout, wgmma descriptors and 3-bit index helpers it shares.
//
//   dx[M, K] = dy[M, N] . W^T,   W = LUT + CSR + dense rows          (one launch, every output written once, no atomics)
//
// A CTA owns one 128 (m) x 128 (k) tile of dx (grid.x = M-tiles, so the CTAs that run together share one k-range's weights in L2)
// and walks N, the reduction axis, in chunks of 64 columns.  Per chunk, all 256 threads first build the operands in shared memory:
//   * dy tile [128 m x 64 c], 16-byte cp.async into the 128-byte-swizzled K-major layout (the forward's x layout; rows past M and
//     columns past N are zero-filled; a dy whose rows are not 16-byte multiples is staged with 2-byte loads);
//   * the chunk's codebook rows, fp32 [value][column];
//   * B tiles: thread (c, q) owns column c of the chunk and the 32 inputs [32 q, 32 q + 32) of the tile.  It decodes its indices
//     (coalesced across the warp's lanes: adjacent columns), adds the CSR entries of column c whose input lies in its range and
//     the dense rows on column c, and stores its 32 values contiguously along k: row c of the MN-major B operand, which the MMA
//     reads with imm-trans-b = 1.
// Exactness (every product exact, fp32 accumulation):
//   * fp16 dy: a power-of-two scale S_i per chunk from the CTA-wide max |w| of the folded chunk (one reduction, one barrier); every
//     weight is split into hi = fp16(w / S_i) and lo = fp16(w / S_i - hi), two MMA passes into the chunk's accumulator, then
//     sum = fma(acc, S_i, sum) (S_i is a power of two: exact).  hi + lo carry about 22 significant bits of w / S_i.  Known limit:
//     a weight more than about 2^20 below the largest weight of its chunk falls into fp16's subnormal range in lo and is kept to
//     about 2^-40 of that largest weight (absolute, not relative).
//   * bf16 dy: w is split into three bf16 parts (tc::split3_bf16x2, all 24 significant bits); bf16 has fp32's exponent range, so
//     no scale.
// CSR columns outside [0, K) and dense-row channels outside [0, N) are ignored; duplicate entries add up.  No limit on topX or on the
// entries per CSR row (each thread scans its column's CSR row in full: rows need not be ascending).
#pragma once

namespace tct {

using tc::BM;
constexpr int BK = 128, BNC = 64;   // dx tile 128 x 128, 64 columns of N per chunk
constexpr int THREADS = 256;        // two warpgroups
constexpr int AS = 0, A_BYTES = BM * BNC * 2;           // dy tile, 16 KB
constexpr int B0 = AS + 2 * A_BYTES, B_BYTES = BNC * BK * 2;  // one B part, 16 KB: two 8 KB atoms of 64 k
template <int NPART>
struct L {
    static constexpr int LUTO = B0 + 2 * NPART * B_BYTES;  // fp32 [2][16][BNC]
    static constexpr int RED = LUTO + 2 * 16 * BNC * 4;   // fp32 [2][8]
    static constexpr int SMEM = RED + 64 + 1024;          // + alignment of the swizzled tiles to 1024 bytes
};

struct PT {
    const uint32_t *qw;
    const float *lut;
    const void *dy;      // [M][N] fp16 / bf16
    void *dx;            // [M][K]
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX, M, K, N, dx_dt, dy_al16;
};

// MN-major operand, 128-byte swizzle: rows of 64 elements (128 bytes) along MN, 8-row groups 1024 bytes apart (SBO), the next 64
// MN elements 8 KB further (LBO)
__device__ __forceinline__ uint64_t mn_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// d[64] (+)= A[64 x 16] . B[16 x 128]; A K-major, B MN-major (imm-trans-b = 1)
template <bool BF>
__device__ __forceinline__ void wgmma_t(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
#define SQ_WGMMA_T(TY)                                                                                                                  \
    asm volatile(                                                                                                                      \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                                   \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                                  \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "    \
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, " \
        "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 1;\n}\n"                              \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),      \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),        \
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),        \
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),        \
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])         \
        : "l"(da), "l"(db), "r"(scale_d))
    if constexpr (BF) SQ_WGMMA_T("bf16");
    else SQ_WGMMA_T("f16");
#undef SQ_WGMMA_T
}

// 3-bit: weights of inputs J.. of a 32-input group from its three words, through a [value][BNC] fp32 codebook column at lb
template <int J>
__device__ __forceinline__ void dec3(float (&w)[32], const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t lb) {
    w[J] = lds_f32(lb + (tc::idx3<J>(w0, w1, w2) << 8));
    if constexpr (J + 1 < 32) dec3<J + 1>(w, w0, w1, w2, lb);
}

template <int BITS, bool BF>
__global__ void __launch_bounds__(THREADS, 1) lutgemm_tc_t_kernel(const PT p) {
    constexpr int LV = 1 << BITS;
    constexpr int WROWS = BITS == 4 ? 4 : 3;  // packed words per (column, 32 k)
    constexpr int NPART = BF ? 3 : 2;
    using G = L<NPART>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t sb = (raw + 1023u) & ~1023u;
    unsigned char *sm = smem_raw + (sb - raw);
    float *red_s = reinterpret_cast<float *>(sm + G::RED);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = tid & (BNC - 1), q = tid >> 6;  // decode role: chunk column, 32-input quarter of the tile
    const int m0 = blockIdx.x * BM, k0 = blockIdx.y * BK;
    const int K = p.K, N = p.N;
    const int kb = k0 + 32 * q;
    const bool kvalid = kb < K;
    const int nch = (N + BNC - 1) / BNC;

    uint32_t wq[WROWS];
    auto load_words = [&](int i) {
        const int col = i * BNC + c;
        const int r0 = BITS == 4 ? kb / 8 : 3 * (kb / 32);
#pragma unroll
        for (int r = 0; r < WROWS; ++r) wq[r] = (i < nch && kvalid && col < N) ? __ldg(p.qw + (size_t)(r0 + r) * N + col) : 0u;
    };

    // operands of chunk i into buffer b; returns the chunk's scale (1 for bf16)
    auto stage = [&](int i, int b) -> float {
        const int n0 = i * BNC, col = n0 + c;
        const bool cvalid = kvalid && col < N;
        // dy tile
        const uint32_t as = sb + AS + b * A_BYTES;
        if (p.dy_al16) {
#pragma unroll
            for (int t = 0; t < BM * BNC / 8 / THREADS; ++t) {
                const int idx = tid + t * THREADS, r = idx >> 3, ch = idx & 7;
                const int gr = m0 + r, gc = n0 + ch * 8;
                const bool ok = gr < p.M && gc < N;
                const unsigned short *src = static_cast<const unsigned short *>(p.dy) + (ok ? (size_t)gr * N + gc : 0);
                cp_async16_clip(as + r * 128 + ((ch ^ (r & 7)) << 4), src, ok ? 2 * min(8, N - gc) : 0);
            }
            cp_async_commit();
        } else {
            for (int idx = tid; idx < BM * BNC / 8; idx += THREADS) {
                const int r = idx >> 3, ch = idx & 7, gr = m0 + r, gc = n0 + ch * 8;
                uint32_t v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const unsigned short *s = static_cast<const unsigned short *>(p.dy) + (size_t)gr * N + gc + 2 * e;
                    const uint32_t lo = (gr < p.M && gc + 2 * e < N) ? (uint32_t)__ldg(s) : 0u;
                    const uint32_t hi = (gr < p.M && gc + 2 * e + 1 < N) ? (uint32_t)__ldg(s + 1) : 0u;
                    v[e] = lo | (hi << 16);
                }
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(as + r * 128 + ((ch ^ (r & 7)) << 4)), "r"(v[0]), "r"(v[1]),
                             "r"(v[2]), "r"(v[3]) : "memory");
            }
        }
        // codebook of the chunk's columns: [value][column]
        float *lut_s = reinterpret_cast<float *>(sm + G::LUTO) + b * 16 * BNC;
        for (int e = tid; e < BNC * LV; e += THREADS) {
            const int cc = e / LV, v = e % LV;
            lut_s[v * BNC + cc] = n0 + cc < N ? __ldg(p.lut + (size_t)(n0 + cc) * LV + v) : 0.f;
        }
        __syncthreads();
        // decode this thread's 32 weights of column c; the next chunk's words are requested first
        float w[32];
        const uint32_t lb = sb + G::LUTO + (uint32_t)(b * 16 * BNC * 4 + c * 4);
        if constexpr (BITS == 4) {
            const uint32_t q0 = wq[0], q1 = wq[1], q2 = wq[2], q3 = wq[3];
            load_words(i + 1);
            const uint32_t qq[4] = {q0, q1, q2, q3};
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int n = 0; n < 8; ++n) w[8 * r + n] = lds_f32(lb + (((qq[r] >> (4 * n)) & 15u) << 8));
        } else {
            const uint32_t q0 = wq[0], q1 = wq[1], q2 = wq[2];
            load_words(i + 1);
            dec3<0>(w, q0, q1, q2, lb);
        }
        if (cvalid) {
            if (p.rows) {
                const int e1 = __ldg(p.rows + col + 1);
                for (int e = __ldg(p.rows + col); e < e1; ++e) {  // storage order; any column order
                    const int kk = __ldg(p.cols + e) - kb;
                    if (kk >= 0 && kk < 32 && kb + kk < K) tc::add_at(w, kk, __ldg(p.vals + e));
                }
            }
            for (int j = 0; j < p.topX; ++j) {
                if (__ldg(p.fri + j) != col) continue;
                const float *fr = p.full_rows + (size_t)kb * p.topX + j;
#pragma unroll
                for (int kk = 0; kk < 32; ++kk) w[kk] += __ldg(fr + (size_t)kk * p.topX);
            }
        } else {
#pragma unroll
            for (int kk = 0; kk < 32; ++kk) w[kk] = 0.f;
        }
        // split and store: row c of each part's MN-major tile, inputs 32 q .. 32 q + 31 (atom q / 2, chunks 4 (q % 2) .. + 3)
        float scale = 1.f;
        const uint32_t rowoff = (uint32_t)((q >> 1) * 8192 + c * 128);
        if constexpr (!BF) {
            float mx = 0.f;
#pragma unroll
            for (int kk = 0; kk < 32; ++kk) mx = fmaxf(mx, fabsf(w[kk]));
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
            if (lane == 0) red_s[b * 8 + warp] = mx;
            __syncthreads();
            mx = red_s[b * 8];
#pragma unroll
            for (int v = 1; v < 8; ++v) mx = fmaxf(mx, red_s[b * 8 + v]);
            int ex = 15;
            if (mx > 0.f && mx <= 3.0e38f) { frexpf(mx, &ex); ex = max(ex, -100); }  // mx < 2^ex
            const float inv = ldexpf(1.f, 15 - ex);
            scale = ldexpf(1.f, ex - 15);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                uint32_t hv[4], lv[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float a0 = w[8 * t + 2 * u] * inv, a1 = w[8 * t + 2 * u + 1] * inv;
                    const __half h0 = __float2half_rn(a0), h1 = __float2half_rn(a1);
                    const __half l0 = __float2half_rn(a0 - __half2float(h0)), l1 = __float2half_rn(a1 - __half2float(h1));
                    hv[u] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                    lv[u] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                }
                const uint32_t off = rowoff + ((((uint32_t)(4 * (q & 1) + t)) ^ (uint32_t)(c & 7)) << 4);
                const uint32_t bh = sb + B0 + (uint32_t)((b * NPART + 0) * B_BYTES), bl = sb + B0 + (uint32_t)((b * NPART + 1) * B_BYTES);
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bh + off), "r"(hv[0]), "r"(hv[1]), "r"(hv[2]), "r"(hv[3]) : "memory");
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bl + off), "r"(lv[0]), "r"(lv[1]), "r"(lv[2]), "r"(lv[3]) : "memory");
            }
        } else {
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                uint32_t pv[3][4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    uint32_t h[3];
                    tc::split3_bf16x2(w[8 * t + 2 * u], w[8 * t + 2 * u + 1], h);
#pragma unroll
                    for (int pp = 0; pp < 3; ++pp) pv[pp][u] = h[pp];
                }
                const uint32_t off = rowoff + ((((uint32_t)(4 * (q & 1) + t)) ^ (uint32_t)(c & 7)) << 4);
#pragma unroll
                for (int pp = 0; pp < 3; ++pp) {
                    const uint32_t bp = sb + B0 + (uint32_t)((b * NPART + pp) * B_BYTES);
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bp + off), "r"(pv[pp][0]), "r"(pv[pp][1]), "r"(pv[pp][2]), "r"(pv[pp][3]) : "memory");
                }
            }
        }
        return scale;
    };

    load_words(0);
    float s_cur = stage(0, 0), s_nxt = 1.f;
    cp_async_wait_all();
    tc::fence_proxy_async();
    __syncthreads();

    const int g = warp >> 2;  // warpgroup: rows [64 g, 64 g + 64) of the tile
    float acc[64], sum[64];
#pragma unroll
    for (int r = 0; r < 64; ++r) { acc[r] = 0.f; sum[r] = 0.f; }
    for (int i = 0; i < nch; ++i) {
        const int b = i & 1;
        const uint32_t xa = sb + AS + b * A_BYTES + g * 64 * 128;
        tc::wgmma_fence();
        // smallest part first: the tensor core's fp32 accumulation rounds each k-step's sum to the accumulator's magnitude, so the
        // small parts go in while the accumulator is still small
#pragma unroll
        for (int pp = NPART - 1; pp >= 0; --pp) {
            const uint32_t bp = sb + B0 + (uint32_t)((b * NPART + pp) * B_BYTES);
#pragma unroll
            for (int s = 0; s < BNC / 16; ++s) wgmma_t<BF>(acc, tc::sw128_desc(xa + 32 * s), mn_desc(bp + 2048 * s), pp < NPART - 1 || s > 0);
        }
        tc::wgmma_commit();
        if (i + 1 < nch) s_nxt = stage(i + 1, b ^ 1);
        tc::wgmma_wait_all();
#pragma unroll
        for (int r = 0; r < 64; ++r) {
            asm volatile("" : "+f"(acc[r])::"memory");
            sum[r] = fmaf(acc[r], s_cur, sum[r]);
        }
        s_cur = s_nxt;
        cp_async_wait_all();
        tc::fence_proxy_async();
        __syncthreads();
    }

    // ---- epilogue: fragment (n, i, j) of lane l in warp wi of the group: row 16 wi + l/4 + 8 i, input 8 n + 2 (l % 4) + j ----
    const int wi = warp & 3;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = m0 + 64 * g + 16 * wi + (lane >> 2) + 8 * i;
        if (row >= p.M) continue;
#pragma unroll
        for (int n = 0; n < BK / 8; ++n) {
            const int gk = k0 + 8 * n + 2 * (lane & 3);
            if (gk >= K) continue;  // K % 32 == 0: both inputs of the pair are in range or neither
            const float v0 = sum[4 * n + 2 * i], v1 = sum[4 * n + 2 * i + 1];
            const size_t o = (size_t)row * K + gk;
            if (p.dx_dt == SQLLM_DT_F32) *reinterpret_cast<float2 *>(static_cast<float *>(p.dx) + o) = make_float2(v0, v1);
            else if (p.dx_dt == SQLLM_DT_F16) *reinterpret_cast<__half2 *>(static_cast<__half *>(p.dx) + o) = __floats2half2_rn(v0, v1);
            else *reinterpret_cast<__nv_bfloat162 *>(static_cast<__nv_bfloat16 *>(p.dx) + o) = __floats2bfloat162_rn(v0, v1);
        }
    }
}

}  // namespace tct
