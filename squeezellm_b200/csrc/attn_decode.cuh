// attn_decode.cuh - batch-1 decode attention of one layer for one token (sqllm_attn_decode): rotary on q and the new k, the append of
// k / v at slot `pos` of the KV cache, and softmax(scale q.K^T[0..pos]) V[0..pos] per query head with grouped KV heads.
//
// Shape.  One thread-block cluster of S CTAs per (KV head, chunk of up to GMAX query heads of its group); S depends on n_kv and the
// SM count only.  The positions 0..pos are dealt to the S CTAs in blocks of BLOCK_POS, a range each CTA computes from the device
// `pos`, and inside a CTA to its 8 warps, U * RPW positions per warp step.  A K / V row is D/8 lanes of 16 bytes (RPW rows per warp
// load), read straight into registers with no L1 allocation; every K / V load serves the G query heads of the CTA.  Each lane keeps an
// online softmax (m, l, acc) per head for the positions of its row slot; the partial states are combined in a fixed order: the row
// slots of a warp by an xor tree, the warps of a CTA in warp order, the CTAs of the cluster in rank order over distributed shared
// memory.  No workspace, no atomics: bit-reproducible.
//
// The CTA whose range holds `pos` takes the new k (rotated, rounded to the dtype) and v from its shared memory, where every CTA
// computes them from qkv; one CTA stores them into the cache.  So no CTA reads a cache slot another CTA of the launch writes, and no
// slot past `pos` is read.
#pragma once
#include "common.cuh"

namespace {
namespace attn {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_CLUSTER = 8;   // portable cluster size
constexpr int BLOCK_POS = 64;    // positions are dealt to the CTAs of a cluster in blocks of this many
constexpr int GMAX = 8;          // query heads per CTA: a larger group is split over several clusters, each reading the K / V again
constexpr float LOG2E = 1.4426950408889634f;

struct Params {
    const void *qkv;             // [n_heads*D | n_kv*D | n_kv*D]
    const int *pos;
    const float *cos, *sin;      // [capacity][D/2]
    void *k_cache, *v_cache;     // [n_kv][capacity][D]
    void *out;                   // [n_heads*D]
    int n_heads, n_kv, g, hchunks, capacity;
    float qscale;                // scale * log2(e): scores in base 2
};

// positions [p0, p1) of CTA `rank` of S for pos + 1 positions: blocks of BLOCK_POS, ceil(blocks / S) per CTA
__device__ __forceinline__ void cta_range(int pos, int rank, int S, int &p0, int &p1) {
    const int blocks = (pos + BLOCK_POS) / BLOCK_POS;
    const int chunk = (blocks + S - 1) / S * BLOCK_POS;
    p0 = rank * chunk;
    p1 = min(pos + 1, p0 + chunk);
}

__device__ __forceinline__ float ld_cluster_f32(const float *local, uint32_t rank) {
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(local)), "r"(rank));
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// the 8 values of a 16-byte word of T as fp32 (exact)
template <typename T>
__device__ __forceinline__ void unpack8(const uint4 w, float (&f)[8]) {
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 t = x16x2_to_f32x2<T>(u[j]);
        f[2 * j] = t.x;
        f[2 * j + 1] = t.y;
    }
}

// exp2(a - b) with exp2(-inf) = 0 whatever b is (an empty state or a masked position weighs nothing)
__device__ __forceinline__ float wexp2(float a, float b) { return a == -INFINITY ? 0.f : exp2f(a - b); }

template <typename T, int D, int G>
__global__ void __launch_bounds__(THREADS, 1) attn_decode_kernel(const Params p) {
    constexpr int LPR = D / 8;          // lanes per K / V row
    constexpr int RPW = 32 / LPR;       // rows per warp load
    constexpr int U = G >= 8 ? 2 : 4;   // warp loads of K (and of V) in flight per lane
    constexpr int STEP = U * RPW;       // positions per warp step
    __shared__ __align__(16) float qs[G][D];
    __shared__ __align__(16) T knew[D], vnew[D];
    __shared__ __align__(16) float wacc[WARPS][G][D];
    __shared__ float wm[WARPS][G], wl[WARPS][G];
    __shared__ __align__(16) float cacc[G][D];
    __shared__ float cm[G], cl[G];

    const int pos = *p.pos;
    if (pos < 0 || pos >= p.capacity) return;  // every CTA leaves before any cluster barrier
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = gridDim.x, rank = (int)rows::cluster_rank();
    const int kvh = blockIdx.y / p.hchunks, hc = blockIdx.y % p.hchunks;
    const int h0 = kvh * p.g + hc * GMAX;               // first query head of this CTA
    const int gc = min(GMAX, p.g - hc * GMAX);          // query heads of this CTA (<= G)
    const T *qkv = static_cast<const T *>(p.qkv);
    const float *cs = p.cos + (size_t)pos * (D / 2), *sn = p.sin + (size_t)pos * (D / 2);

    // rotary (rotate-half) in fp32: q of the CTA's heads, scaled to base-2 scores; the new k rounded once to T
    for (int idx = tid; idx < G * D; idx += THREADS) {
        const int h = idx / D, i = idx % D, j = i % (D / 2);
        float v = 0.f;
        if (h < gc) {
            const T *q = qkv + (size_t)(h0 + h) * D;
            const float a = to_f32(q[j]), b = to_f32(q[j + D / 2]);
            v = (i < D / 2 ? a * cs[j] - b * sn[j] : b * cs[j] + a * sn[j]) * p.qscale;
        }
        qs[h][i] = v;
    }
    if (tid < D) {
        const int i = tid, j = i % (D / 2);
        const T *k = qkv + (size_t)p.n_heads * D + (size_t)kvh * D;
        const float a = to_f32(k[j]), b = to_f32(k[j + D / 2]);
        knew[i] = f32_to<T>(i < D / 2 ? a * cs[j] - b * sn[j] : b * cs[j] + a * sn[j]);
        vnew[i] = qkv[(size_t)(p.n_heads + p.n_kv) * D + (size_t)kvh * D + i];
    }
    __syncthreads();
    const size_t slot = ((size_t)kvh * p.capacity + pos) * D;
    if (rank == 0 && hc == 0 && tid < D) {  // the append: slot `pos` of this KV head, nothing else
        static_cast<T *>(p.k_cache)[slot + tid] = knew[tid];
        static_cast<T *>(p.v_cache)[slot + tid] = vnew[tid];
    }

    const int sub = lane / LPR, e = (lane % LPR) * 8;   // row slot of the lane, first element of its 16 bytes
    float q[G][8];
#pragma unroll
    for (int h = 0; h < G; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) q[h][j] = qs[h][e + j];
    float m[G], l[G], acc[G][8];
#pragma unroll
    for (int h = 0; h < G; ++h) {
        m[h] = -INFINITY;
        l[h] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[h][j] = 0.f;
    }

    int p0, p1;
    cta_range(pos, rank, S, p0, p1);
    const T *kbase = static_cast<const T *>(p.k_cache) + (size_t)kvh * p.capacity * D + e;
    const T *vbase = static_cast<const T *>(p.v_cache) + (size_t)kvh * p.capacity * D + e;
    for (int base = p0 + warp * STEP; base < p1; base += WARPS * STEP) {
        uint4 kr[U], vr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int t = base + u * RPW + sub;
            if (t == pos) {
                kr[u] = *reinterpret_cast<const uint4 *>(&knew[e]);
                vr[u] = *reinterpret_cast<const uint4 *>(&vnew[e]);
            } else if (t < p1) {
                kr[u] = ldg_stream(kbase + (size_t)t * D);
                vr[u] = ldg_stream(vbase + (size_t)t * D);
            } else {
                kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
            }
        }
        float s[G][U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            float kf[8];
            unpack8<T>(kr[u], kf);
            const bool live = base + u * RPW + sub < p1;
#pragma unroll
            for (int h = 0; h < G; ++h) {
                float a = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) a = fmaf(q[h][j], kf[j], a);
#pragma unroll
                for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                s[h][u] = live ? a : -INFINITY;
            }
        }
        float vf[U][8];
#pragma unroll
        for (int u = 0; u < U; ++u) unpack8<T>(vr[u], vf[u]);
#pragma unroll
        for (int h = 0; h < G; ++h) {
            float mx = m[h];
#pragma unroll
            for (int u = 0; u < U; ++u) mx = fmaxf(mx, s[h][u]);
            if (mx == -INFINITY) continue;  // no live position in this lane's slot yet
            const float corr = wexp2(m[h], mx);
            l[h] *= corr;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[h][j] *= corr;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const float w = wexp2(s[h][u], mx);
                l[h] += w;
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[h][j] = fmaf(w, vf[u][j], acc[h][j]);
            }
            m[h] = mx;
        }
    }

    // the row slots of the warp: xor tree over the lanes LPR apart
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
#pragma unroll
        for (int h = 0; h < G; ++h) {
            const float mo = __shfl_xor_sync(0xffffffffu, m[h], o), lo = __shfl_xor_sync(0xffffffffu, l[h], o);
            const float mx = fmaxf(m[h], mo);
            const float a = wexp2(m[h], mx), b = wexp2(mo, mx);
            l[h] = l[h] * a + lo * b;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float ao = __shfl_xor_sync(0xffffffffu, acc[h][j], o);
                acc[h][j] = acc[h][j] * a + ao * b;
            }
            m[h] = mx;
        }
    }
    if (sub == 0) {
#pragma unroll
        for (int h = 0; h < G; ++h) {
#pragma unroll
            for (int j = 0; j < 8; ++j) wacc[warp][h][e + j] = acc[h][j];
            if (lane == 0) { wm[warp][h] = m[h]; wl[warp][h] = l[h]; }
        }
    }
    __syncthreads();
    // the warps of the CTA, in warp order
    for (int idx = tid; idx < G * D; idx += THREADS) {
        const int h = idx / D, i = idx % D;
        float mx = -INFINITY;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) mx = fmaxf(mx, wm[w][h]);
        float L = 0.f, A = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            const float c = wexp2(wm[w][h], mx);
            L += wl[w][h] * c;
            A += wacc[w][h][i] * c;
        }
        cacc[h][i] = A;
        if (i == 0) { cm[h] = mx; cl[h] = L; }
    }
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
    // the CTAs of the cluster, in rank order; CTA r finishes the outputs r, r + S*THREADS, ... of its heads
    T *out = static_cast<T *>(p.out);
    for (int idx = rank * THREADS + tid; idx < gc * D; idx += S * THREADS) {
        const int h = idx / D, i = idx % D;
        float mr[MAX_CLUSTER], mx = -INFINITY;
#pragma unroll
        for (int r = 0; r < MAX_CLUSTER; ++r) {
            if (r < S) { mr[r] = ld_cluster_f32(&cm[h], r); mx = fmaxf(mx, mr[r]); }
        }
        float L = 0.f, A = 0.f;
#pragma unroll
        for (int r = 0; r < MAX_CLUSTER; ++r) {
            if (r < S) {
                const float c = wexp2(mr[r], mx);
                L += ld_cluster_f32(&cl[h], r) * c;
                A += ld_cluster_f32(&cacc[h][i], r) * c;
            }
        }
        out[(size_t)(h0 + h) * D + i] = f32_to<T>(A / L);
    }
    asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;" ::: "memory");  // the peers' partials stay alive until read
}

}  // namespace attn
}  // namespace
