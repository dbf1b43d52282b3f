// attn_verify.cuh - decode attention of T <= 16 new tokens of one sequence at positions *pos .. *pos+T-1 (sqllm_attn_verify): the
// decode kernel (attn_decode_row.inc) generalised from query heads to (token, query head) rows, for verifying drafted tokens.
//
// Shape.  The T*g rows of one KV head's group are token-major (row r is token r / g, head r % g); one thread-block cluster of S CTAs per
// (KV head, chunk of up to GMAX rows), so every K / V row a CTA loads serves all the rows of its chunk: at g = 1 and T = 8 one chunk per
// KV head, the K / V bytes of one decode call.  The positions 0 .. pos+T-1 are dealt to the S CTAs in blocks of BLOCK_POS (cta_range),
// and inside a CTA to its warps exactly as in the decode kernel.  Row r's own causal limit pos + r/g masks only positions of the last
// T, which lie in the last block.  Every CTA computes the T rotated k' (rounded to the dtype once, rope() of attn_decode.cuh) and the
// T v into shared memory, takes positions >= pos from there and reads the cache only below pos; one CTA per KV head stores them.  So
// no CTA reads a slot written in the same launch, and no slot at or past pos + T is read.  Partial states are combined by the decode
// kernel's text (attn_combine.inc): row slots by an xor tree, warps in warp order, CTAs in rank order over distributed shared memory.
// No workspace, no atomics: bit-reproducible.  A position range outside the cache (pos < 0 or pos + T > capacity) writes nothing.
#pragma once
#include "attn_decode.cuh"

namespace {
namespace attn {

constexpr int VMAX = 16;  // tokens per call

struct VerParams {
    const void *qkv;             // [T][n_heads*D | n_kv*D | n_kv*D]
    const int *pos;              // the first token's position
    const float *cos, *sin;      // [capacity][D/2]
    void *k_cache, *v_cache;     // [n_kv][capacity][D]
    void *out;                   // [T][n_heads*D]
    int n_heads, n_kv, g, chunks, capacity, T;
    float qscale;                // scale * log2(e): scores in base 2
};

template <typename T, int D, int G>
__global__ void __launch_bounds__(THREADS, 1) attn_verify_kernel(const VerParams p) {
    constexpr int LPR = D / 8;          // lanes per K / V row
    constexpr int RPW = 32 / LPR;       // rows per warp load
    constexpr int U = G >= 8 ? 2 : 4;   // warp loads of K (and of V) in flight per lane
    constexpr int STEP = U * RPW;       // positions per warp step
    // qc holds the rotated q' until every warp has read it into registers, then the CTA's combined partial sums
    __shared__ __align__(16) float qc[G][D];
    __shared__ __align__(16) T knew[VMAX][D], vnew[VMAX][D];
    __shared__ __align__(16) float wacc[WARPS][G][D];
    __shared__ float wm[WARPS][G], wl[WARPS][G];
    __shared__ float cm[G], cl[G];

    const int pos = *p.pos;
    if (pos < 0 || pos > p.capacity - p.T) return;  // every CTA leaves before any cluster barrier
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int S = gridDim.x, rank = (int)rows::cluster_rank();
    const int kvh = blockIdx.y / p.chunks, ch = blockIdx.y % p.chunks;
    const int r0 = ch * GMAX;                           // first (token, head) row of this CTA in the group's T*g rows
    const int gc = min(GMAX, p.T * p.g - r0);           // rows of this CTA (<= G)
    T *const out = static_cast<T *>(p.out);
    const auto store_out = [&](int h, int i, float v) {  // for attn_combine.inc: row h is token t's query head `head`
        const int t = (r0 + h) / p.g, head = kvh * p.g + (r0 + h) % p.g;
        out[(size_t)t * p.n_heads * D + (size_t)head * D + i] = f32_to<T>(v);
    };
    const size_t row_elems = (size_t)(p.n_heads + 2 * p.n_kv) * D;
    const T *qkv = static_cast<const T *>(p.qkv);

    // rotary (rotate-half) in fp32 at each token's own position: q of the CTA's rows, scaled to base-2 scores; the T new k rounded
    // once to T, and the T new v
    for (int idx = tid; idx < G * D; idx += THREADS) {
        const int r = idx / D, i = idx % D, j = i % (D / 2);
        float v = 0.f;
        if (r < gc) {
            const int t = (r0 + r) / p.g, h = kvh * p.g + (r0 + r) % p.g;
            const float *cs = p.cos + (size_t)(pos + t) * (D / 2), *sn = p.sin + (size_t)(pos + t) * (D / 2);
            const T *q = qkv + t * row_elems + (size_t)h * D;
            const float a = to_f32(q[j]), b = to_f32(q[j + D / 2]);
            v = rope<D>(a, b, cs, sn, i) * p.qscale;
        }
        qc[r][i] = v;
    }
    for (int idx = tid; idx < p.T * D; idx += THREADS) {
        const int t = idx / D, i = idx % D, j = i % (D / 2);
        const float *cs = p.cos + (size_t)(pos + t) * (D / 2), *sn = p.sin + (size_t)(pos + t) * (D / 2);
        const T *k = qkv + t * row_elems + (size_t)p.n_heads * D + (size_t)kvh * D;
        const float a = to_f32(k[j]), b = to_f32(k[j + D / 2]);
        knew[t][i] = f32_to<T>(rope<D>(a, b, cs, sn, i));
        vnew[t][i] = qkv[t * row_elems + (size_t)(p.n_heads + p.n_kv) * D + (size_t)kvh * D + i];
    }
    __syncthreads();
    if (rank == 0 && ch == 0) {  // the append: slots pos .. pos+T-1 of this KV head, nothing else
        const size_t slot = ((size_t)kvh * p.capacity + pos) * D;
        for (int idx = tid; idx < p.T * D; idx += THREADS) {
            static_cast<T *>(p.k_cache)[slot + idx] = knew[idx / D][idx % D];
            static_cast<T *>(p.v_cache)[slot + idx] = vnew[idx / D][idx % D];
        }
    }

    const int sub = lane / LPR, e = (lane % LPR) * 8;   // row slot of the lane, first element of its 16 bytes
    int p0, p1;
    cta_range(pos + p.T - 1, rank, S, p0, p1);
    float q[G][8];
    int lim[G];  // the last position row h attends to, within this CTA's range; -1 for a padding row
#pragma unroll
    for (int h = 0; h < G; ++h) {
#pragma unroll
        for (int j = 0; j < 8; ++j) q[h][j] = qc[h][e + j];
        lim[h] = h < gc ? min(pos + (r0 + h) / p.g, p1 - 1) : -1;
    }
    float m[G], l[G], acc[G][8];
#pragma unroll
    for (int h = 0; h < G; ++h) {
        m[h] = -INFINITY;
        l[h] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[h][j] = 0.f;
    }

    const T *kbase = static_cast<const T *>(p.k_cache) + (size_t)kvh * p.capacity * D + e;
    const T *vbase = static_cast<const T *>(p.v_cache) + (size_t)kvh * p.capacity * D + e;
    for (int base = p0 + warp * STEP; base < p1; base += WARPS * STEP) {
        uint4 kr[U], vr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int t = base + u * RPW + sub;
            if (t >= p1) {
                kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
            } else if (t >= pos) {
                kr[u] = *reinterpret_cast<const uint4 *>(&knew[t - pos][e]);
                vr[u] = *reinterpret_cast<const uint4 *>(&vnew[t - pos][e]);
            } else {
                kr[u] = ldg_stream(kbase + (size_t)t * D);
                vr[u] = ldg_stream(vbase + (size_t)t * D);
            }
        }
        float s[G][U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            float kf[8];
            unpack8<T>(kr[u], kf);
            const int t = base + u * RPW + sub;
#pragma unroll
            for (int h = 0; h < G; ++h) {
                float a = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) a = fmaf(q[h][j], kf[j], a);
#pragma unroll
                for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
                s[h][u] = t <= lim[h] ? a : -INFINITY;
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
                // a masked position (a later token of the call) adds nothing, not even 0 * its v, which may be inf or NaN
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[h][j] = s[h][u] == -INFINITY ? acc[h][j] : fmaf(w, vf[u][j], acc[h][j]);
            }
            m[h] = mx;
        }
    }

    float (&cacc)[G][D] = qc;  // the CTA's combined sums go to qc: every warp read its q' into registers before the combine's barrier
#include "attn_combine.inc"
}

}  // namespace attn
}  // namespace
