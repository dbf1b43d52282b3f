// lutgemm_t.cuh - the transposed LUT-GEMM behind sqllm_lutgemm_t: the input gradient of QuantLinearLUT on the CUDA cores.
// Included by lutgemv_kernels.cu inside its anonymous namespace, after lutgemv_rows.cuh (cluster helpers).
//
//   dx[m][k] = sum_c dy[m][c] W[k][c],   W[k][c] = LUT[c][idx(k,c)] + CSR(c,k) + sum_j full_rows[k][j] [fri[j] == c]
//
// fp16 / bf16 / fp32 dy [M][N], dx fp32 or dy's dtype [M][K]; exact fp32 codebook, fp32 sums.  The bias plays no part.
//
// Tiling: a CTA owns one slab of KS = 128 inputs, one group of RB rows of dy and one range of 64-column strips; grid
// (S, slabs, ceil(M / RB)), launched as clusters of (S, 1, 1): the S CTAs of a cluster split the strips of N, the reduction axis.
// S comes from K, N and the SM count only, never from M, and every row runs the same instructions whatever RB is, so a row's
// result does not depend on M or on the other rows.
//   * items: the slab is 16 items of 8 inputs, one per half-warp (4-bit: one packed word row; 3-bit: a quarter of a 32-input
//     group, decoded from the group's three word rows).  Lane i of a half-warp owns columns 4i..4i+3 of every strip, as in the
//     forward kernels, so a warp's weight loads are coalesced along the columns.
//   * per strip: the strip's codebook ([value][slot] fp32, the forward's conflict-free layout) and its RB x 64 values of dy (as
//     fp32) are staged in shared memory, double-buffered with one barrier per strip.  Each lane decodes its 4 columns x 8 inputs
//     and adds, per row and input, the 4 products of the strip into its running sum (acc[RB][8]: inputs along registers).
//   * after the last strip the 16 lanes of a half-warp hold partial sums of the same 8 inputs over different columns: a fixed
//     xor tree adds them up.
//   * CSR outliers, filtered per slab: warp w walks the CSR rows of channels w, w+8, ... of the cluster rank's range, 32 entries
//     at a time, keeps those whose column lies in the slab and adds val * dy[m][c] into its own [RB][KS] copy in shared memory,
//     one entry at a time in storage order; the 8 copies are added in warp order.  Filtering per slab needs no transposed copy
//     of the CSR arrays (the C ABI takes the forward's CSR as it is) and no sorting, and has no limit on the entries per row.
//   * dense rows: thread k of the slab adds full_rows[k][j] * dy[m][fri[j]] for every j whose channel lies in the rank's range,
//     in index order (duplicates add up).
//   * reduction: every CTA leaves partial[RB][KS]; after a cluster barrier the leader reads the peers' partials over DSMEM in
//     rank order, converts and stores dx once; a second cluster barrier keeps the peers' shared memory alive until then.  No
//     workspace, no atomics: bit-reproducible, safe on several streams, CUDA-graph capturable.
// CSR columns outside [0, K) and dense-row channels outside [0, N) are ignored.
#pragma once

namespace bwd {

constexpr int TW = 8;                 // warps per CTA
constexpr int TTHREADS = TW * 32;
constexpr int KS = 128;               // inputs per slab: 16 items of 8
constexpr int MAX_SPLIT = 8;          // S <= 8: portable cluster size
constexpr int TABB = 16 * STRIP * 4;  // one codebook buffer (4-bit; 3-bit uses half)

struct PT {
    const uint32_t *qw;
    const float *lut;
    const void *dy;     // [M][N]
    void *dx;           // [M][K]
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX;
    int K, N, M;
    int strips;
    int dy_dt, dx_dt;   // SQLLM_DT_*
    int qw_al16;        // qweight 16-byte aligned and N % 4 == 0: 16-byte weight loads
};

// shared-memory carve-up in bytes; host and device use the same numbers
template <int RB>
struct ST {
    static constexpr int TAB = 0;                           // [2][16][STRIP] fp32 codebooks
    static constexpr int DY = 2 * TABB;                     // [2][RB][STRIP] fp32
    static constexpr int CSR = DY + 2 * RB * STRIP * 4;     // [TW][RB][KS] fp32
    static constexpr int PART = CSR + TW * RB * KS * 4;     // [RB][KS] fp32
    static constexpr int TOTAL = PART + RB * KS * 4;
};

__device__ __forceinline__ float ld_dy(const void *p, int dt, size_t i) {
    if (dt == SQLLM_DT_F32) return __ldg(static_cast<const float *>(p) + i);
    if (dt == SQLLM_DT_F16) return __half2float(__ldg(static_cast<const __half *>(p) + i));
    return __bfloat162float(__ldg(static_cast<const __nv_bfloat16 *>(p) + i));
}

template <int BITS, int RB>
__global__ void __launch_bounds__(TTHREADS, 2) lutgemm_t_kernel(const PT p) {
    constexpr int L = 1 << BITS;
    constexpr int ROWS = BITS == 4 ? 1 : 3;  // packed word rows per item
    using G = ST<RB>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t sb = smem_u32(smem_raw);
    float *dys = reinterpret_cast<float *>(smem_raw + G::DY);
    float *csr = reinterpret_cast<float *>(smem_raw + G::CSR);
    float *part = reinterpret_cast<float *>(smem_raw + G::PART);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, i16 = lane & 15, jsel = lane >> 4;
    const uint32_t rank = rows::cluster_rank();
    const int S = (int)gridDim.x;  // = cluster size
    const int k_lo = blockIdx.y * KS, b0 = blockIdx.z * RB;
    const int s_lo = (int)((long long)p.strips * rank / S), s_hi = (int)((long long)p.strips * (rank + 1) / S);
    const int c_lo = s_lo * STRIP, c_hi = min(p.N, s_hi * STRIP);  // this rank's channels
    const int it = 2 * warp + jsel, kit = k_lo + 8 * it;            // this half-warp's item: inputs [kit, kit + 8)
    const bool kvalid = kit < p.K;
    const int r0 = BITS == 4 ? kit / 8 : 3 * (kit / 32), quarter = (kit / 8) & 3;

    if (p.rows)
        for (int e = tid; e < TW * RB * KS; e += TTHREADS) csr[e] = 0.f;

    // ---- strip staging: codebook (one float4 of one column per thread) and dy (fp32), via registers ----
    constexpr int DYN = (RB * STRIP + TTHREADS - 1) / TTHREADS;
    float4 lv = make_float4(0.f, 0.f, 0.f, 0.f);
    float dv[DYN];
    auto fetch = [&](int s) {
        if (tid < STRIP * L / 4) {
            const int c = tid / (L / 4), q = tid % (L / 4), col = s * STRIP + c;
            const float *src = p.lut + (size_t)col * L + 4 * q;  // 4-byte loads: the table need only be 4-byte aligned
            lv = col < p.N ? make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < DYN; ++i) {
            const int e = tid + i * TTHREADS, b = e / STRIP, col = s * STRIP + (e % STRIP);
            dv[i] = (e < RB * STRIP && b0 + b < p.M && col < p.N) ? ld_dy(p.dy, p.dy_dt, (size_t)(b0 + b) * p.N + col) : 0.f;
        }
    };
    auto store = [&](int buf) {
        if (tid < STRIP * L / 4) {
            const int c = tid / (L / 4), q = tid % (L / 4);
            float *t = reinterpret_cast<float *>(smem_raw + G::TAB + buf * TABB) + (4 * q) * STRIP + (((c & 3) << 4) | (c >> 2));
            t[0] = lv.x; t[STRIP] = lv.y; t[2 * STRIP] = lv.z; t[3 * STRIP] = lv.w;
        }
#pragma unroll
        for (int i = 0; i < DYN; ++i) {
            const int e = tid + i * TTHREADS;
            if (e < RB * STRIP) dys[buf * RB * STRIP + e] = dv[i];
        }
    };
    auto load_words = [&](int s, uint4 (&w)[ROWS]) {
        const int col0 = s * STRIP + 4 * i16;
        const bool ok = s < s_hi && kvalid && col0 < p.N;
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
            const uint32_t *src = p.qw + (size_t)(r0 + r) * p.N + col0;
            if (!ok) w[r] = make_uint4(0u, 0u, 0u, 0u);
            else if (p.qw_al16) w[r] = BITS == 4 ? ldg_stream(src) : __ldg(reinterpret_cast<const uint4 *>(src));
            else w[r] = make_uint4(__ldg(src), col0 + 1 < p.N ? __ldg(src + 1) : 0u, col0 + 2 < p.N ? __ldg(src + 2) : 0u,
                                   col0 + 3 < p.N ? __ldg(src + 3) : 0u);
        }
    };

    float acc[RB][8];
#pragma unroll
    for (int b = 0; b < RB; ++b)
#pragma unroll
        for (int n = 0; n < 8; ++n) acc[b][n] = 0.f;
    uint32_t lt[4];  // table address of the lane's column t ^ jsel (half-warp 1 walks its columns in the order 1, 0, 3, 2)
#pragma unroll
    for (int t = 0; t < 4; ++t) lt[t] = sb + G::TAB + (uint32_t)((((t ^ jsel) << 4) | i16) << 2);

    uint4 cur[ROWS], nxt[ROWS];
    if (s_lo < s_hi) {
        fetch(s_lo);
        store(0);
        load_words(s_lo, cur);
    }
    __syncthreads();
    for (int s = s_lo, buf = 0; s < s_hi; ++s, buf ^= 1) {
        if (s + 1 < s_hi) fetch(s + 1);
        load_words(s + 1, nxt);
        // decode: wv[t][n] = W[kit + n][column 4 i16 + (t ^ jsel)]
        float wv[4][8];
        const uint32_t tb = (uint32_t)(buf * TABB);
        if constexpr (BITS == 4) {
            const uint4 q = cur[0];
            const uint32_t w[4] = {jsel ? q.y : q.x, jsel ? q.x : q.y, jsel ? q.w : q.z, jsel ? q.z : q.w};
#pragma unroll
            for (int t = 0; t < 4; ++t)
#pragma unroll
                for (int n = 0; n < 8; ++n) wv[t][n] = lds_f32(lt[t] + tb + (((w[t] >> (4 * n)) & 15u) << 8));
        } else {
            const uint32_t a[4] = {jsel ? cur[0].y : cur[0].x, jsel ? cur[0].x : cur[0].y, jsel ? cur[0].w : cur[0].z, jsel ? cur[0].z : cur[0].w};
            const uint32_t b[4] = {jsel ? cur[1].y : cur[1].x, jsel ? cur[1].x : cur[1].y, jsel ? cur[1].w : cur[1].z, jsel ? cur[1].z : cur[1].w};
            const uint32_t c[4] = {jsel ? cur[2].y : cur[2].x, jsel ? cur[2].x : cur[2].y, jsel ? cur[2].w : cur[2].z, jsel ? cur[2].z : cur[2].w};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                // index J of a group sits at bit 3J of the 96-bit word c:b:a; this quarter's 8 indices are bits [24 q, 24 q + 24)
                const uint32_t v = quarter == 0 ? a[t] : quarter == 1 ? __funnelshift_r(a[t], b[t], 24)
                                 : quarter == 2 ? __funnelshift_r(b[t], c[t], 16) : c[t] >> 8;
#pragma unroll
                for (int n = 0; n < 8; ++n) wv[t][n] = lds_f32(lt[t] + tb + (((v >> (3 * n)) & 7u) << 8));
            }
        }
#pragma unroll
        for (int b = 0; b < RB; ++b) {
            const float4 d4 = lds_v4(sb + G::DY + (uint32_t)(((buf * RB + b) * STRIP + 4 * i16) * 4));
            const float d0 = jsel ? d4.y : d4.x, d1 = jsel ? d4.x : d4.y, d2 = jsel ? d4.w : d4.z, d3 = jsel ? d4.z : d4.w;
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                // the strip's 4 products first, then one add into the running sum
                float d = wv[0][n] * d0;
                d = fmaf(wv[1][n], d1, d); d = fmaf(wv[2][n], d2, d); d = fmaf(wv[3][n], d3, d);
                acc[b][n] += d;
            }
        }
#pragma unroll
        for (int r = 0; r < ROWS; ++r) cur[r] = nxt[r];
        if (s + 1 < s_hi) store(buf ^ 1);
        __syncthreads();
    }

    // ---- sum over the half-warp's 16 lanes (fixed xor tree: every lane ends with the same bits), one store per value ----
#pragma unroll
    for (int b = 0; b < RB; ++b)
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            float v = acc[b][n];
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            if (((b * 8 + n) & 15) == i16) part[b * KS + 8 * it + n] = v;
        }

    // ---- CSR entries of the rank's channels whose column lies in the slab: warp w takes channels c_lo + w, + TW, ... ----
    if (p.rows) {
        float *mine = csr + warp * RB * KS;
        for (int c = c_lo + warp; c < c_hi; c += TW) {
            const int e0 = __ldg(p.rows + c), e1 = __ldg(p.rows + c + 1);
            for (int e = e0; e < e1; e += 32) {
                const int ee = e + lane;
                const int kl = ee < e1 ? __ldg(p.cols + ee) - k_lo : -1;
                const bool hit = (unsigned)kl < (unsigned)KS && k_lo + kl < p.K;
                const float v = hit ? __ldg(p.vals + ee) : 0.f;
                unsigned mask = __ballot_sync(0xffffffffu, hit);
                while (mask) {  // warp-uniform: one entry at a time, in storage order
                    const int src = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const int k = __shfl_sync(0xffffffffu, kl, src);
                    const float val = __shfl_sync(0xffffffffu, v, src);
                    if (lane < RB && b0 + lane < p.M) {
                        float *o = mine + lane * KS + k;
                        *o = fmaf(val, ld_dy(p.dy, p.dy_dt, (size_t)(b0 + lane) * p.N + c), *o);
                    }
                    __syncwarp();
                }
            }
        }
    }

    // ---- dense rows whose channel lies in the rank's range, in index order: thread k of the slab, all RB rows ----
    float dacc[RB];
#pragma unroll
    for (int b = 0; b < RB; ++b) dacc[b] = 0.f;
    if (p.topX > 0 && tid < KS && k_lo + tid < p.K) {
        const float *fr = p.full_rows + (size_t)(k_lo + tid) * p.topX;
        for (int j = 0; j < p.topX; ++j) {
            const int c = __ldg(p.fri + j);
            if (c < c_lo || c >= c_hi) continue;
            const float f = __ldg(fr + j);
#pragma unroll
            for (int b = 0; b < RB; ++b)
                if (b0 + b < p.M) dacc[b] = fmaf(f, ld_dy(p.dy, p.dy_dt, (size_t)(b0 + b) * p.N + c), dacc[b]);
        }
    }
    __syncthreads();
    if (tid < KS) {
#pragma unroll
        for (int b = 0; b < RB; ++b) {
            float t = part[b * KS + tid];
            if (p.rows) {
                float o = csr[b * KS + tid];
#pragma unroll
                for (int w = 1; w < TW; ++w) o += csr[(w * RB + b) * KS + tid];
                t += o;
            }
            part[b * KS + tid] = t + dacc[b];
        }
    }

    // ---- cluster reduction: the leader sums the S partials in rank order and stores dx once ----
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
    if (rank == 0) {
        for (int e = tid; e < RB * (KS / 4); e += TTHREADS) {
            const int b = e / (KS / 4), k4 = 4 * (e - b * (KS / 4));
            const int row = b0 + b, k = k_lo + k4;
            if (row >= p.M || k >= p.K) continue;
            const uint32_t la = smem_u32(part + b * KS + k4);
            float4 s = rows::ld_cluster_v4(la, 0);
            for (int r = 1; r < S; ++r) {
                const float4 t = rows::ld_cluster_v4(la, (uint32_t)r);
                s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
            }
            const size_t o = (size_t)row * p.K + k;
            if (p.dx_dt == SQLLM_DT_F32) {
                *reinterpret_cast<float4 *>(static_cast<float *>(p.dx) + o) = s;
            } else if (p.dx_dt == SQLLM_DT_F16) {
                const __half2 h01 = __floats2half2_rn(s.x, s.y), h23 = __floats2half2_rn(s.z, s.w);
                uint2 v;
                v.x = *reinterpret_cast<const uint32_t *>(&h01);
                v.y = *reinterpret_cast<const uint32_t *>(&h23);
                *reinterpret_cast<uint2 *>(static_cast<__half *>(p.dx) + o) = v;
            } else {
                const __nv_bfloat162 h01 = __floats2bfloat162_rn(s.x, s.y), h23 = __floats2bfloat162_rn(s.z, s.w);
                uint2 v;
                v.x = *reinterpret_cast<const uint32_t *>(&h01);
                v.y = *reinterpret_cast<const uint32_t *>(&h23);
                *reinterpret_cast<uint2 *>(static_cast<__nv_bfloat16 *>(p.dx) + o) = v;
            }
        }
    }
    asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;" ::: "memory");
}

}  // namespace bwd
