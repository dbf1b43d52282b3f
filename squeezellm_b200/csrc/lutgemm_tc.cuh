// lutgemm_tc.cuh - tensor-core (wgmma) LUT-GEMM for M >= 1 rows of fp16 or bf16 activations (sqllm_lutgemm_fused_dt) or fp32 ones
// (sqllm_lutgemm_fused_f32).  Included by lutgemv_kernels.cu inside its anonymous namespace.
//
// fp32 x (F32X) is not exact in a 16-bit operand: it is split like the weights into three bf16 parts (split3_bf16x2), loaded into
// registers at the start of each chunk's build (the loads fly while the weights are decoded) and stored as three x tiles of the
// same swizzled layout; the MMAs take the six part products whose orders sum to at most 2 (x_l.w_h, x_m.w_m, x_h.w_l, x_m.w_h,
// x_h.w_m, x_h.w_h: smallest first, 24 k16 steps per chunk, 384 products per accumulator before the promotion).  The dropped
// x_m.w_l + x_l.w_m + x_l.w_l are below 2^-23 |x w| per product.  fp32 x always writes fp32 y.
//
//   y[M, N] = bias + x . W_lut + x . S_csr + x . W_dense            (one launch, every output written once, no atomics)
//
// A CTA owns one 128 x 128 output tile (grid.x = M-tiles, so the CTAs that run together share one N-tile's weights in L2) and walks
// K in chunks of 64.  Per chunk, all 256 threads first build the operands in shared memory:
//   * x tile [128 rows x 64 k] fp16 / bf16, 16-byte cp.async into the 128-byte-swizzled K-major layout wgmma reads (rows past M
//     and k past K are zero-filled);
//   * B tiles: thread (c, h) owns column c of the tile and k-half h of the chunk.  It decodes its 32 indices through the tile's
//     codebook (fp32, staged [value][column]: conflict-free), adds the CSR outliers and dense rows of its column that fall in its
//     k range (the outlier fold: no x gather, no extra MMA), scales by the column's power-of-two 1/s_c and splits every weight
//     exactly into parts of x's type: fp16 x: hi = fp16(w/s_c) and lo = fp16(w/s_c - hi); bf16 x: hi, mid and lo (split3_bf16x2).
//     One column's 64 k of one part are one swizzled 128-byte row.
// Then each of the two warpgroups issues wgmma m64n128k16 -> f32 for its 64 rows, four k-steps per part, into the same
// accumulator: fp16 x the steps of hi, then those of lo; bf16 x lo, mid, then hi (smallest part first: the tensor core rounds
// each k-step's sum to the accumulator's magnitude, so the small parts go in while the accumulator is still small).  x is exact
// in its own type, hi + lo carry about 22 significant bits of w / s_c and hi + mid + lo all 24, so every product is exact and
// the error is that of the fp32 accumulation.  The chunk's accumulator starts from zero and is added into a running fp32 sum
// with FADD once the chunk's MMAs have completed (promotion: the tensor core's own fp32 accumulation never sees more than one
// chunk's products per output, 128 for fp16 x and 192 for bf16 x).  Two buffers: the operands of chunk i+1 are built while the
// MMAs of chunk i run.
// Epilogue: y = sum * s_c + bias, x's type or fp32, ragged M and N tails masked.
//
// s_c = 2^(e - 15) with 2^e > |lut_c|max + (CSR values of row c) + sum over the dense rows of column c of their max |value|, so
// every folded weight / s_c stays below 2^15 (finite in fp16) and lo stays a normal fp16 number for every weight within 2^-17 of
// that bound.  bf16 has fp32's exponent range and needs no scale; it is kept (a power of two: exact) so both types share the
// code.  The dense-row maxima are found at tile start by the whole CTA, one dense row at a time.
//
// CSR rows are walked with a cursor that needs ascending column indices; tile start checks each row, and a row that is not
// ascending is filtered in full at every chunk instead (slow, still exact).  Column indices outside [0, K) and dense-row indices
// outside [0, N) are ignored.  No limit on topX or on the number of outliers.
#pragma once

namespace tc {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int THREADS = 256;  // two warpgroups
constexpr int XS = 0, XS_BYTES = BM * BK * 2;  // x part q of buffer b at XS + (XPART b + q) XS_BYTES
constexpr int B_BYTES = BN * BK * 2;
template <int NPART, int XPART = 1>  // weight parts: 2 (fp16 x: hi, lo) or 3 (bf16 / fp32 x: hi, mid, lo); x parts: 3 for fp32 x
struct L {
    static constexpr int B0 = XS + 2 * XPART * XS_BYTES;    // weight part pp of buffer b at B0 + (2 pp + b) B_BYTES
    static constexpr int LUT = B0 + 2 * NPART * B_BYTES;    // fp32 [16][BN]
    static constexpr int SCALE = LUT + 16 * BN * 4;         // fp32 [BN] s_c
    static constexpr int DSUM = SCALE + BN * 4;             // fp32 [BN] sum of the column's dense-row maxima
    static constexpr int DCNT = DSUM + BN * 4;              // int [BN] dense rows on the column
    static constexpr int DFIRST = DCNT + BN * 4;            // int [BN] first of them
    static constexpr int RED = DFIRST + BN * 4;             // fp32 [8] block reduction
    static constexpr int SMEM = RED + 64 + 1024;            // + alignment of the swizzled tiles to 1024 bytes
};

struct PT {
    const uint32_t *qw;
    const float *lut;
    const unsigned short *x;  // [M][K] fp16 / bf16
    void *y;                  // [M][N]
    const float *bias;
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX, M, K, N, y_16;  // y_16: y in x's type, else fp32
};

__device__ __forceinline__ uint64_t sw128_desc(uint32_t saddr) {  // K-major operand, 128-byte swizzle, 8-row groups 1024 bytes apart
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// d[64] (+)= A[64 x 16] . B[16 x 128]; A and B K-major in shared memory, fp16 (BF = false) or bf16 (BF = true)
template <bool BF>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
#define SQ_WGMMA_K(TY)                                                                                                                  \
    asm volatile(                                                                                                                      \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                                   \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                                  \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "    \
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, " \
        "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"                              \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),      \
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),        \
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),        \
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),        \
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),        \
          "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),        \
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])         \
        : "l"(da), "l"(db), "r"(scale_d))
    if constexpr (BF) SQ_WGMMA_K("bf16");
    else SQ_WGMMA_K("f16");
#undef SQ_WGMMA_K
}

// Two fp32 values each split exactly into three bf16 parts: hi = bf16(w), mid = bf16(w - hi), lo = bf16(w - hi - mid).  Every
// subtraction is exact and hi + mid + lo == w down to bf16's subnormal range.  pv[pp] packs part pp of w0 (low half) and w1.
__device__ __forceinline__ void split3_bf16x2(const float w0, const float w1, uint32_t (&pv)[3]) {
    uint32_t h[3][2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        float r = s ? w1 : w0;
#pragma unroll
        for (int pp = 0; pp < 3; ++pp) {
            const __nv_bfloat16 x = __float2bfloat16_rn(r);
            h[pp][s] = (uint32_t)__bfloat16_as_ushort(x);
            r -= __bfloat162float(x);  // exact
        }
    }
#pragma unroll
    for (int pp = 0; pp < 3; ++pp) pv[pp] = h[pp][0] | (h[pp][1] << 16);
}

// 3-bit index J (0..31) of a 32-input group from its three words (squeezellm/quant.py:177-203 layout)
template <int J>
__device__ __forceinline__ uint32_t idx3(const uint32_t w0, const uint32_t w1, const uint32_t w2) {
    if constexpr (J < 10) return (w0 >> (3 * J)) & 7u;
    else if constexpr (J == 10) return (w0 >> 30) | ((w1 & 1u) << 2);
    else if constexpr (J < 21) return (w1 >> (3 * (J - 11) + 1)) & 7u;
    else if constexpr (J == 21) return (w1 >> 31) | ((w2 & 3u) << 1);
    else return (w2 >> (3 * (J - 22) + 2)) & 7u;
}
template <int J>
__device__ __forceinline__ void dec3(float (&w)[32], const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t lb) {
    w[J] = lds_f32(lb + (idx3<J>(w0, w1, w2) << 9));
    if constexpr (J + 1 < 32) dec3<J + 1>(w, w0, w1, w2, lb);
}
// the 32 weights of a 4-bit group from its four words (8 nibbles each, lowest first)
__device__ __forceinline__ void dec4(float (&w)[32], const uint32_t (&q)[4], const uint32_t lb) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int n = 0; n < 8; ++n) w[8 * r + n] = lds_f32(lb + (((q[r] >> (4 * n)) & 15u) << 9));
}

__device__ __forceinline__ void add_at(float (&w)[32], const int kk, const float v) {  // w[kk] += v, kk in [0, 32), registers only
#pragma unroll
    for (int j = 0; j < 32; ++j)
        if (j == kk) w[j] += v;
}

// BF: bf16 x (three weight parts), else fp16 x (two).  F32X (with BF): fp32 x, split into three bf16 parts like the weights.
template <int BITS, bool BF, bool F32X = false>
__global__ void __launch_bounds__(THREADS, 1) lutgemm_tc_kernel(const PT p) {
    static_assert(BF || !F32X, "fp32 x takes the bf16 operands");
    constexpr int LV = 1 << BITS;
    constexpr int WROWS = BITS == 4 ? 4 : 3;  // packed words per (column, 32 k)
    constexpr int NPART = BF ? 3 : 2;
    constexpr int XPART = F32X ? 3 : 1;
    using G = L<NPART, XPART>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t sb = (raw + 1023u) & ~1023u;
    unsigned char *sm = smem_raw + (sb - raw);
    float *scale_s = reinterpret_cast<float *>(sm + G::SCALE);
    float *dsum_s = reinterpret_cast<float *>(sm + G::DSUM);
    int *dcnt_s = reinterpret_cast<int *>(sm + G::DCNT);
    int *dfirst_s = reinterpret_cast<int *>(sm + G::DFIRST);
    float *red_s = reinterpret_cast<float *>(sm + G::RED);
    const auto bpart = [&](int pp, int b) { return sb + (uint32_t)(G::B0 + (2 * pp + b) * B_BYTES); };  // part pp of buffer b
    const auto xpart = [&](int q, int b) { return sb + (uint32_t)(XS + (XPART * b + q) * XS_BYTES); };  // x part q of buffer b

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int c = tid & (BN - 1), h = tid >> 7;  // decode role: tile column, k-half of the chunk
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int col = n0 + c;
    const bool cvalid = col < p.N;
    const int K = p.K, N = p.N;

    // ---- tile start: codebook, dense-row bookkeeping, per-column scale and outlier cursor ----
    for (int e = tid; e < BN * LV; e += THREADS) {
        const int cc = e / LV, v = e % LV;
        const float val = n0 + cc < N ? __ldg(p.lut + (size_t)(n0 + cc) * LV + v) : 0.f;
        reinterpret_cast<float *>(sm + G::LUT)[v * BN + cc] = val;
    }
    if (tid < BN) { dsum_s[tid] = 0.f; dcnt_s[tid] = 0; dfirst_s[tid] = 0; }
    __syncthreads();
    if (p.full_rows && p.topX > 0) {
        const int nend = min(N, n0 + BN);
        for (int j = 0; j < p.topX; ++j) {  // uniform loop: the branch below is taken by the whole CTA or by none of it
            const int f = __ldg(p.fri + j);
            if (f < n0 || f >= nend) continue;
            float m = 0.f;
            for (int k = tid; k < K; k += THREADS) m = fmaxf(m, fabsf(__ldg(p.full_rows + (size_t)k * p.topX + j)));
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
            if (lane == 0) red_s[warp] = m;
            __syncthreads();
            if (tid == 0) {
                float mm = red_s[0];
                for (int w = 1; w < THREADS / 32; ++w) mm = fmaxf(mm, red_s[w]);
                dsum_s[f - n0] += mm;
                if (dcnt_s[f - n0]++ == 0) dfirst_s[f - n0] = j;
            }
            __syncthreads();
        }
    }
    const uint32_t lb = sb + G::LUT + c * 4;
    int e_cur = 0, e_end = 0;
    bool sorted = true;
    float inv_s;
    {
        float bnd = 0.f;
#pragma unroll
        for (int v = 0; v < LV; ++v) bnd = fmaxf(bnd, fabsf(lds_f32(lb + v * BN * 4)));
        if (p.rows && cvalid) {
            e_cur = __ldg(p.rows + col); e_end = __ldg(p.rows + col + 1);
            float smax = 0.f, ssum = 0.f;
            bool distinct = true;
            int prev = (int)0x80000000;
            for (int e = e_cur; e < e_end; ++e) {
                const int k = __ldg(p.cols + e);
                const float a = fabsf(__ldg(p.vals + e));
                sorted = sorted && k >= prev;
                distinct = distinct && k != prev;
                prev = k;
                smax = fmaxf(smax, a); ssum += a;
            }
            bnd += (sorted && distinct) ? smax : ssum;  // several entries on one k add up
        }
        bnd += dsum_s[c];
        int ex = 15;
        if (bnd > 0.f && bnd <= 3.0e38f) { frexpf(bnd, &ex); ex = max(ex, -100); }  // bnd < 2^ex
        inv_s = ldexpf(1.f, 15 - ex);
        if (h == 0) scale_s[c] = ldexpf(1.f, ex - 15);
    }
    const int d_cnt = dcnt_s[c], d_first = dfirst_s[c];

    const int nch = (K + BK - 1) / BK;
    uint32_t wq[WROWS];
    auto load_words = [&](int i) {
        const int kb = i * BK + 32 * h;
        const int r0 = BITS == 4 ? kb / 8 : 3 * (kb / 32);
#pragma unroll
        for (int r = 0; r < WROWS; ++r) wq[r] = (i < nch && kb < K && cvalid) ? __ldg(p.qw + (size_t)(r0 + r) * N + col) : 0u;
    };

    // operands of chunk i into buffer b: x by cp.async (fp32 x: loaded into registers here, split and stored after the weights),
    // this thread's 32 weights of column c decoded, folded, split and stored
    constexpr int XV = BM * BK / 4 / THREADS;  // fp32 x: float4 loads per thread and chunk
    auto stage = [&](int i, int b) {
        const int k0 = i * BK;
        float4 xv[F32X ? XV : 1];
        if constexpr (F32X) {  // the loads are in flight while the weights are decoded
            const float *xf = reinterpret_cast<const float *>(p.x);
#pragma unroll
            for (int q = 0; q < XV; ++q) {
                const int idx = tid + q * THREADS, r = idx >> 4, c4 = idx & 15;
                const int gr = m0 + r, gk = k0 + 4 * c4;
                xv[q] = gr < p.M && gk < K ? __ldg(reinterpret_cast<const float4 *>(xf + (size_t)gr * K + gk)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
            const uint32_t xs = sb + XS + b * XS_BYTES;
#pragma unroll
            for (int q = 0; q < BM * BK / 8 / THREADS; ++q) {
                const int idx = tid + q * THREADS, r = idx >> 3, ch = idx & 7;
                const int gr = m0 + r, gk = k0 + ch * 8;
                const bool ok = gr < p.M && gk < K;
                cp_async16_clip(xs + r * 128 + ((ch ^ (r & 7)) << 4), ok ? p.x + (size_t)gr * K + gk : p.x, ok ? 16 : 0);
            }
            cp_async_commit();
        }

        const int kb = k0 + 32 * h;
        float w[32];  // the next chunk's words are requested before this chunk's are decoded
        if constexpr (BITS == 4) {
            const uint32_t q0 = wq[0], q1 = wq[1], q2 = wq[2], q3 = wq[3];
            load_words(i + 1);
            const uint32_t q[4] = {q0, q1, q2, q3};
            dec4(w, q, lb);
        } else {
            const uint32_t q0 = wq[0], q1 = wq[1], q2 = wq[2];
            load_words(i + 1);
            dec3<0>(w, q0, q1, q2, lb);
        }
        if (kb < K && cvalid) {
            if (sorted) {
                for (; e_cur < e_end; ++e_cur) {
                    const int kk = __ldg(p.cols + e_cur) - kb;
                    if (kk >= 32) break;
                    if (kk >= 0) add_at(w, kk, __ldg(p.vals + e_cur));
                }
            } else {
                for (int e = e_cur; e < e_end; ++e) {
                    const int kk = __ldg(p.cols + e) - kb;
                    if (kk >= 0 && kk < 32) add_at(w, kk, __ldg(p.vals + e));
                }
            }
            for (int j = d_first, found = 0; found < d_cnt; ++j) {
                if (__ldg(p.fri + j) != col) continue;
                ++found;
                const float *fr = p.full_rows + (size_t)kb * p.topX + j;
#pragma unroll
                for (int kk = 0; kk < 32; ++kk) w[kk] += __ldg(fr + (size_t)kk * p.topX);
            }
        }
        const uint32_t rowoff = c * 128;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if constexpr (BF) {
                uint32_t pv[3][4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    uint32_t t[3];
                    split3_bf16x2(w[8 * q + 2 * u] * inv_s, w[8 * q + 2 * u + 1] * inv_s, t);
#pragma unroll
                    for (int pp = 0; pp < 3; ++pp) pv[pp][u] = t[pp];
                }
                const uint32_t off = rowoff + ((((uint32_t)(4 * h + q)) ^ (uint32_t)(c & 7)) << 4);
#pragma unroll
                for (int pp = 0; pp < 3; ++pp)
                    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bpart(pp, b) + off), "r"(pv[pp][0]), "r"(pv[pp][1]), "r"(pv[pp][2]), "r"(pv[pp][3]) : "memory");
            } else {
                uint32_t hv[4], lv[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float a0 = w[8 * q + 2 * u] * inv_s, a1 = w[8 * q + 2 * u + 1] * inv_s;
                    const __half h0 = __float2half_rn(a0), h1 = __float2half_rn(a1);
                    const __half l0 = __float2half_rn(a0 - __half2float(h0)), l1 = __float2half_rn(a1 - __half2float(h1));
                    hv[u] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                    lv[u] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                }
                const uint32_t off = rowoff + ((((uint32_t)(4 * h + q)) ^ (uint32_t)(c & 7)) << 4);
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bpart(0, b) + off), "r"(hv[0]), "r"(hv[1]), "r"(hv[2]), "r"(hv[3]) : "memory");
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(bpart(1, b) + off), "r"(lv[0]), "r"(lv[1]), "r"(lv[2]), "r"(lv[3]) : "memory");
            }
        }
        if constexpr (F32X) {  // x = hi + mid + lo exactly (split3_bf16x2), part q into its own tile: k 4 c4 .. 4 c4 + 3 of row r
#pragma unroll
            for (int q = 0; q < XV; ++q) {
                const int idx = tid + q * THREADS, r = idx >> 4, c4 = idx & 15;
                uint32_t t01[3], t23[3];
                split3_bf16x2(xv[q].x, xv[q].y, t01);
                split3_bf16x2(xv[q].z, xv[q].w, t23);
                const uint32_t off = r * 128 + ((((uint32_t)(c4 >> 1)) ^ (uint32_t)(r & 7)) << 4) + (c4 & 1) * 8;
#pragma unroll
                for (int pp = 0; pp < 3; ++pp)
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(xpart(pp, b) + off), "r"(t01[pp]), "r"(t23[pp]) : "memory");
            }
        }
    };

    load_words(0);
    stage(0, 0);
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();

    const int g = warp >> 2;  // warpgroup: rows [64 g, 64 g + 64) of the tile
    float acc[64], sum[64];
#pragma unroll
    for (int r = 0; r < 64; ++r) { acc[r] = 0.f; sum[r] = 0.f; }
    for (int i = 0; i < nch; ++i) {
        const int b = i & 1;
        const uint32_t xa = sb + XS + b * XS_BYTES + g * 64 * 128;
        wgmma_fence();
        if constexpr (F32X) {  // the six x part . w part products of part orders summing to <= 2, smallest first
            constexpr int PX[6] = {2, 1, 0, 1, 0, 0}, PW[6] = {0, 1, 2, 0, 1, 0};  // 0 hi, 1 mid, 2 lo
#pragma unroll
            for (int t = 0; t < 6; ++t)
#pragma unroll
                for (int s = 0; s < BK / 16; ++s)
                    wgmma_m64n128k16<true>(acc, sw128_desc(xpart(PX[t], b) + g * 64 * 128 + 32 * s), sw128_desc(bpart(PW[t], b) + 32 * s),
                                           t > 0 || s > 0);
        } else if constexpr (BF) {  // lo, mid, hi: smallest part first
#pragma unroll
            for (int pp = NPART - 1; pp >= 0; --pp)
#pragma unroll
                for (int s = 0; s < BK / 16; ++s)
                    wgmma_m64n128k16<true>(acc, sw128_desc(xa + 32 * s), sw128_desc(bpart(pp, b) + 32 * s), pp < NPART - 1 || s > 0);
        } else {  // hi, then lo
            const uint32_t bh = bpart(0, b), bl = bpart(1, b);
#pragma unroll
            for (int s = 0; s < BK / 16; ++s) wgmma_m64n128k16<false>(acc, sw128_desc(xa + 32 * s), sw128_desc(bh + 32 * s), s > 0);
#pragma unroll
            for (int s = 0; s < BK / 16; ++s) wgmma_m64n128k16<false>(acc, sw128_desc(xa + 32 * s), sw128_desc(bl + 32 * s), 1);
        }
        wgmma_commit();
        if (i + 1 < nch) stage(i + 1, b ^ 1);
        wgmma_wait_all();
#pragma unroll
        for (int r = 0; r < 64; ++r) {
            asm volatile("" : "+f"(acc[r])::"memory");
            sum[r] += acc[r];
        }
        cp_async_wait_all();
        fence_proxy_async();
        __syncthreads();
    }

    // ---- epilogue: fragment (n, i, j) of lane l in warp wi of the group: row 16 wi + l/4 + 8 i, column 8 n + 2 (l % 4) + j ----
    const int wi = warp & 3;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = m0 + 64 * g + 16 * wi + (lane >> 2) + 8 * i;
        if (row >= p.M) continue;
#pragma unroll
        for (int n = 0; n < BN / 8; ++n) {
            const int cl = 8 * n + 2 * (lane & 3), gc = n0 + cl;
            if (gc >= N) continue;
            float v0 = sum[4 * n + 2 * i] * scale_s[cl], v1 = sum[4 * n + 2 * i + 1] * scale_s[cl + 1];
            if (p.bias) { v0 += __ldg(p.bias + gc); if (gc + 1 < N) v1 += __ldg(p.bias + gc + 1); }
            const size_t o = (size_t)row * N + gc;
            if (!F32X && p.y_16) {
                if constexpr (BF) {
                    __nv_bfloat16 *y = reinterpret_cast<__nv_bfloat16 *>(p.y);
                    if (gc + 1 < N && !(N & 1)) *reinterpret_cast<__nv_bfloat162 *>(y + o) = __floats2bfloat162_rn(v0, v1);
                    else { y[o] = __float2bfloat16_rn(v0); if (gc + 1 < N) y[o + 1] = __float2bfloat16_rn(v1); }
                } else {
                    __half *y = reinterpret_cast<__half *>(p.y);
                    if (gc + 1 < N && !(N & 1)) *reinterpret_cast<__half2 *>(y + o) = __floats2half2_rn(v0, v1);
                    else { y[o] = __float2half_rn(v0); if (gc + 1 < N) y[o + 1] = __float2half_rn(v1); }
                }
            } else {
                float *y = reinterpret_cast<float *>(p.y);
                if (gc + 1 < N && !(N & 1)) *reinterpret_cast<float2 *>(y + o) = make_float2(v0, v1);
                else { y[o] = v0; if (gc + 1 < N) y[o + 1] = v1; }
            }
        }
    }
}

}  // namespace tc
