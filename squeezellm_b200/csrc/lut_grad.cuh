// lut_grad.cuh - gradients of QuantLinearLUT's continuous parameters behind sqllm_lut_grad: the per-channel codebook, the CSR
// outlier values and the dense rows, from G = x^T . dy (3-bit index helpers: lutgemm_tc.cuh).  This file holds the plan,
// the epilogue and the cluster reduction that both kernels share, and the CUDA-core kernel; lut_grad_tc.cuh the tensor-core one.
//
//   G[k][c] = sum_m x[m][k] dy[m][c]                                   (K x N, the reduction over the rows)
//   dLUT[c][v] = sum_{k : idx(k,c) = v} G[k][c]
//   dvals[e] = G[cols[e]][c]  for e in CSR row c with 0 <= cols[e] < K, else 0
//   dfull_rows[k][j] = G[k][fri[j]]  if 0 <= fri[j] < N, else 0
//
// Tiling: a CTA owns 128 channels (a column tile, grid.y) and one slab of 128-input tiles (k-tiles) of K; grid (S, column tiles),
// launched as clusters of (S, 1, 1): the S CTAs of a cluster split K.  Per k-tile the CTA forms the 128 x 128 tile of G over all
// M rows (a chunk at a time, each chunk's sum started from zero and then added into a running fp32 sum), stages it in shared
// memory and runs the epilogue:
//   * thread c < 128 decodes idx(k, c) for the tile's inputs and adds G[k][c] into bins[idx][c], in ascending k;
//   * thread 128 + c writes dvals for the entries of CSR row c whose column lies in the tile (each entry is written once, by the
//     one CTA whose k-tile holds it); rank 0 of the cluster writes 0 for the entries whose column is outside [0, K) at its first tile;
//   * all threads write dfull_rows[k][j] for the tile's inputs and every j whose channel lies in the column tile; the clusters of
//     column tile 0 write 0 for the j whose channel is outside [0, N).
// After the slab the bins ([2^bits][128] fp32) of the S CTAs are added by the leader over DSMEM in rank order and dLUT is written
// once.  No workspace, no atomics, no spin-waits: bit-reproducible, CUDA-graph capturable and safe on several streams.
#pragma once
#include "common.cuh"
#include "lutgemm_tc.cuh"

namespace {

namespace lg {

constexpr int TK = 128, TC = 128;     // G tile: 128 inputs x 128 channels
constexpr int THREADS = 256;
constexpr int GST = TC + 8;           // row stride of the staged G tile (floats): float2 fragment stores without bank conflicts
constexpr int MAX_SPLIT = 8;          // S <= 8: portable cluster size
constexpr int G_BYTES = TK * GST * 4;
constexpr int BIN_BYTES = 16 * TC * 4;

struct PG {
    const uint32_t *qw;
    const void *x, *dy;   // [M][K], [M][N]
    int x_dt, dy_dt;      // SQLLM_DT_*
    const int *rows, *cols;
    const int *fri;
    int topX;
    float *dlut, *dvals, *dfull;
    int M, K, N, ktiles;
    int x_al16, dy_al16;  // 16-byte rows: cp.async staging (tensor cores)
};

// the k-tiles [t_lo, t_hi) of cluster rank `rank` of S
__device__ __forceinline__ void slab(int ktiles, int rank, int S, int &t_lo, int &t_hi) {
    t_lo = (int)((long long)ktiles * rank / S);
    t_hi = (int)((long long)ktiles * (rank + 1) / S);
}

template <int J>
__device__ __forceinline__ void bin3(float *bins, const float *g, const uint32_t w0, const uint32_t w1, const uint32_t w2) {
    float *b = bins + tc::idx3<J>(w0, w1, w2) * TC;
    *b += g[J * GST];
    if constexpr (J + 1 < 32) bin3<J + 1>(bins, g, w0, w1, w2);
}

// the epilogue of one k-tile: gs holds G[k0 + k][n0 + c] at gs[k * GST + c]; bins[v * TC + c] of this CTA
template <int BITS>
__device__ __forceinline__ void tile_epilogue(const PG &p, const float *gs, float *bins, int k0, int n0, bool zero_csr) {
    const int tid = threadIdx.x;
    const int kn = min(TK, p.K - k0);  // inputs of the tile (a multiple of 32)
    if (tid < TC) {
        const int c = tid, col = n0 + c;
        if (p.dlut && col < p.N) {
            constexpr int WR = BITS == 4 ? 4 : 3;  // packed words per 32-input group
            const uint32_t *q = p.qw + col;
            const int ng = kn / 32;
            uint32_t w[WR], nx[WR] = {};
            auto load_group = [&](uint32_t (&d)[WR], int g32) {  // the group's words, first packed row (k0 + 32 g32) / 32 * WR
                const size_t r0 = (size_t)WR * ((k0 + 32 * g32) / 32);
#pragma unroll
                for (int r = 0; r < WR; ++r) d[r] = __ldg(q + (r0 + r) * p.N);
            };
            load_group(w, 0);
            for (int g32 = 0; g32 < ng; ++g32) {
                if (g32 + 1 < ng) load_group(nx, g32 + 1);  // the next group's words are in flight while this group is binned
                const float *g = gs + (32 * g32) * GST + c;
                if constexpr (BITS == 4) {
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int n = 0; n < 8; ++n) bins[((w[r] >> (4 * n)) & 15u) * TC + c] += g[(8 * r + n) * GST];
                } else {
                    bin3<0>(bins + c, g, w[0], w[1], w[2]);
                }
#pragma unroll
                for (int r = 0; r < WR; ++r) w[r] = nx[r];
            }
        }
    } else if (p.dvals) {
        const int c = tid - TC, col = n0 + c;
        if (col < p.N) {
            const int e1 = __ldg(p.rows + col + 1);
            for (int e = __ldg(p.rows + col); e < e1; ++e) {  // storage order; any column order
                const int k = __ldg(p.cols + e);
                if (k >= k0 && k < k0 + kn) p.dvals[e] = gs[(k - k0) * GST + c];
                else if (zero_csr && (unsigned)k >= (unsigned)p.K) p.dvals[e] = 0.f;
            }
        }
    }
    if (p.dfull) {
        const int nend = min(p.N, n0 + TC);
        for (int e = tid; e < kn * p.topX; e += THREADS) {  // j fastest: coalesced stores
            const int kk = e / p.topX, j = e - kk * p.topX;
            const int f = __ldg(p.fri + j);
            float *o = p.dfull + (size_t)(k0 + kk) * p.topX + j;
            if (f >= n0 && f < nend) *o = gs[kk * GST + (f - n0)];
            else if (n0 == 0 && (unsigned)f >= (unsigned)p.N) *o = 0.f;
        }
    }
}

__device__ __forceinline__ float ld_cluster_f32(uint32_t local, uint32_t rank) {  // the same shared address in CTA `rank` of the cluster
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local), "r"(rank));
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

// the end of a slab: the leader adds the S CTAs' bins in rank order and stores dLUT [N][2^bits] once
template <int BITS>
__device__ __forceinline__ void reduce_bins(const PG &p, const float *bins, int n0, uint32_t rank, int S) {
    constexpr int L = 1 << BITS;
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
    if (rank == 0 && p.dlut) {
        const int cn = min(TC, p.N - n0);
        for (int e = threadIdx.x; e < cn * L; e += THREADS) {  // (c, v), v fastest: coalesced stores
            const int c = e / L, v = e - c * L;
            const uint32_t la = smem_u32(bins + v * TC + c);
            float s = ld_cluster_f32(la, 0);
            for (int r = 1; r < S; ++r) s += ld_cluster_f32(la, (uint32_t)r);
            p.dlut[(size_t)(n0 + c) * L + v] = s;
        }
    }
    asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;" ::: "memory");  // the peers' bins stay alive until read
}

// ---- CUDA cores: any x / dy dtype pair, fp32 products and sums -----------------------------------------------------------
// Per chunk of MC rows, x [MC][128 k] and dy [MC][128 c] are staged in shared memory as fp32 (fetched into registers one chunk
// ahead).  Thread (tk, tn) = (tid / 16, tid % 16) owns the 8 x 8 block of G with inputs {4 tk + i, 64 + 4 tk + i} and channels
// {4 tn + j, 64 + 4 tn + j}: per row two float4 of x and two of dy from shared memory (conflict-free), 64 FMAs.
constexpr int MC = 32;
constexpr int XS = 0, DS = MC * TK * 4, GSO = DS + MC * TC * 4, BINS = GSO + G_BYTES, SMEM = BINS + BIN_BYTES;
constexpr int PER = MC * TK / THREADS;  // values of x (and of dy) per thread per chunk

// this thread's PER raw elements of a chunk of a row-major matrix [rows][ld] (rows m0.., columns c0..c0 + 127): the 32-bit words
// of fp32, the 16-bit words of fp16 / bf16, 0 outside [0, M) x [0, C).  The dtype branch is outside the loop and nothing is
// converted here, so all PER loads are in flight at once; cvt_raw converts at the shared-memory store.
__device__ __forceinline__ void ld_raw(uint32_t (&v)[PER], const void *src, int dt, int ld, int m0, int M, int c0, int C) {
    if (dt == SQLLM_DT_F32) {
        const uint32_t *s = static_cast<const uint32_t *>(src);
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int e = threadIdx.x + u * THREADS, m = m0 + e / TK, c = c0 + e % TK;
            v[u] = (m < M && c < C) ? __ldg(s + (size_t)m * ld + c) : 0u;
        }
    } else {
        const unsigned short *s = static_cast<const unsigned short *>(src);
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int e = threadIdx.x + u * THREADS, m = m0 + e / TK, c = c0 + e % TK;
            v[u] = (m < M && c < C) ? (uint32_t)__ldg(s + (size_t)m * ld + c) : 0u;
        }
    }
}
__device__ __forceinline__ float cvt_raw(uint32_t v, int dt) {
    if (dt == SQLLM_DT_F32) return __uint_as_float(v);
    if (dt == SQLLM_DT_F16) return __half2float(__ushort_as_half((unsigned short)v));
    return __uint_as_float(v << 16);  // bf16: the upper half of an fp32
}

template <int BITS>
__global__ void __launch_bounds__(THREADS, 1) lut_grad_kernel(const PG p) {
    constexpr int L = 1 << BITS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t sb = smem_u32(smem_raw);
    float *xs = reinterpret_cast<float *>(smem_raw + XS);
    float *ds = reinterpret_cast<float *>(smem_raw + DS);
    float *gs = reinterpret_cast<float *>(smem_raw + GSO);
    float *bins = reinterpret_cast<float *>(smem_raw + BINS);
    const int tid = threadIdx.x, tk = tid >> 4, tn = tid & 15;
    const uint32_t rank = rows::cluster_rank();
    const int S = (int)gridDim.x;  // = cluster size
    const int n0 = blockIdx.y * TC;
    int t_lo, t_hi;
    slab(p.ktiles, (int)rank, S, t_lo, t_hi);
    for (int e = tid; e < L * TC; e += THREADS) bins[e] = 0.f;

    const int nch = (p.M + MC - 1) / MC;
    uint32_t xv[PER], dv[PER];  // the next chunk, raw
    auto fetch = [&](int i, int k0) {
        ld_raw(xv, p.x, p.x_dt, p.K, i * MC, p.M, k0, p.K);
        ld_raw(dv, p.dy, p.dy_dt, p.N, i * MC, p.M, n0, p.N);
    };

    for (int t = t_lo; t < t_hi; ++t) {
        const int k0 = t * TK;
        float sum[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) sum[i][j] = 0.f;
        fetch(0, k0);
        for (int i = 0; i < nch; ++i) {
            __syncthreads();  // the previous chunk (or tile epilogue) is done with the staging buffers
#pragma unroll
            for (int u = 0; u < PER; ++u) {
                xs[tid + u * THREADS] = cvt_raw(xv[u], p.x_dt);
                ds[tid + u * THREADS] = cvt_raw(dv[u], p.dy_dt);
            }
            __syncthreads();
            if (i + 1 < nch) fetch(i + 1, k0);
            float acc[8][8];
#pragma unroll
            for (int a = 0; a < 8; ++a)
#pragma unroll
                for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
            const int rows_here = min(MC, p.M - i * MC);
            for (int m = 0; m < rows_here; ++m) {
                const uint32_t xr = sb + XS + (uint32_t)(m * TK * 4), dr = sb + DS + (uint32_t)(m * TC * 4);
                const float4 xa = lds_v4(xr + 16 * tk), xb = lds_v4(xr + 256 + 16 * tk);
                const float4 da = lds_v4(dr + 16 * tn), db = lds_v4(dr + 256 + 16 * tn);
                const float xk[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
                const float dc[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
#pragma unroll
                for (int a = 0; a < 8; ++a)
#pragma unroll
                    for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(xk[a], dc[b], acc[a][b]);
            }
#pragma unroll
            for (int a = 0; a < 8; ++a)
#pragma unroll
                for (int b = 0; b < 8; ++b) sum[a][b] += acc[a][b];
        }
        // stage the tile of G: input 4 tk + a (a < 4) or 64 + 4 tk + a - 4, channel likewise
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            float *row = gs + (a < 4 ? 4 * tk + a : 64 + 4 * tk + a - 4) * GST;
            *reinterpret_cast<float4 *>(row + 4 * tn) = make_float4(sum[a][0], sum[a][1], sum[a][2], sum[a][3]);
            *reinterpret_cast<float4 *>(row + 64 + 4 * tn) = make_float4(sum[a][4], sum[a][5], sum[a][6], sum[a][7]);
        }
        __syncthreads();
        tile_epilogue<BITS>(p, gs, bins, k0, n0, rank == 0 && t == t_lo);
    }
    __syncthreads();
    reduce_bins<BITS>(p, bins, n0, rank, S);
}

}  // namespace lg

}  // namespace
