// attn_extend.cuh - attention of one layer for a chunk of T new tokens of one sequence at positions start .. start+T-1
// (sqllm_attn_extend): the append of the chunk's rotated k and its v at slots start .. start+T-1 of the KV cache, then causal
// softmax(scale q'.K^T[0..p]) V[0..p] for every token (p = start + t) and query head, with grouped KV heads.  Two launches on one stream:
//
//   attn_append_kernel   one CTA per token: k' = rotary(k) in fp32 rounded to the dtype once - the expression of attn_decode_row.inc,
//                        so a slot holds the same bits whichever kernel wrote it - and v unchanged.
//   attn_extend_kernel   FlashAttention-2 style, K / V read from the cache only (so no CTA reads a slot written in the same launch).
//
// Shape of attn_extend_kernel.  A query tile is BM = 64 (token, query head) rows of one KV head's group, token-major (row r of the
// group's T*g rows is token r / g, head r % g), so every K / V tile serves all g heads of the group: GQA without repeating K / V.
// grid (S, tiles, n_kv), clusters of S CTAs along x; the tiles run last-first (the longest key ranges start first).  The tile's keys
// 0 .. start + t_last are dealt to the S CTAs of its cluster in blocks of BN = 64, ceil(blocks / S) per CTA.  A CTA streams its blocks
// through shared memory with cp.async, double-buffered (16-byte chunks xor-swizzled by row against ldmatrix bank conflicts); keys at
// or past the tile's limit are zero-filled, never read.  Each of the 4 warps owns 16 rows: S = Q K^T and O += P V on mma.sync m16n8k16
// with fp32 accumulation.  K and V are exact in the dtype; q' (fp32) and P (fp32) are each split into hi + lo
// parts in the dtype (q' staged in shared memory, P straight from the score registers), two MMAs per product, so the operands carry
// about 22 (fp16) or 16 (bf16) bits instead of 11 or 8.  Only blocks that cross the causal edge are masked; the softmax is online, in fp32 with exp2.  With S > 1 the CTAs' (m, l, acc) states are combined in rank order over
// distributed shared memory, as attn_decode's are.  No workspace, no atomics: bit-reproducible.
#pragma once
#include "attn_decode.cuh"

namespace {
namespace attn {

constexpr int XTHREADS = 128;      // 4 warps x 16 query rows
constexpr int BM = 64;             // (token, head) rows per query tile
constexpr int BN = 64;             // keys per K / V block
constexpr int APPEND_THREADS = 256;
constexpr float QPRE = 0.25f;      // q' is split at q'/4 (exact): |q'| <= sqrt(2) * 65504 stays finite in fp16; 4 goes into the scale
constexpr int MAX_TILES = 65535;   // gridDim.y

struct ExtParams {
    const void *qkv;             // [T][n_heads*D | n_kv*D | n_kv*D]
    const float *cos, *sin;      // [capacity][D/2]
    void *k_cache, *v_cache;     // [n_kv][capacity][D]
    void *out;                   // [T][n_heads*D]
    int n_heads, n_kv, g, capacity, start, T;
    float qscale;                // scale * log2(e) / QPRE: scores in base 2
};

// dynamic shared memory of attn_extend_kernel: K and V, two stages each (the cluster combine reuses them for [BM][D] fp32), q' hi and lo
constexpr int ext_smem_bytes(int d) { return (2 * 2 * BN + 2 * BM) * d * 2; }

template <typename T> struct Pair;
template <> struct Pair<__half> { using type = __half2; };
template <> struct Pair<__nv_bfloat16> { using type = __nv_bfloat162; };

// (a, b) rounded to T, a in the low half
template <typename T>
__device__ __forceinline__ uint32_t pack_t(float a, float b) {
    typename Pair<T>::type v;
    v.x = f32_to<T>(a);
    v.y = f32_to<T>(b);
    return *reinterpret_cast<uint32_t *>(&v);
}

// x = hi + lo + r: hi = T(x), lo = T(x - hi) for the pair (a, b)
template <typename T>
__device__ __forceinline__ void split_pair(float a, float b, uint32_t &hi, uint32_t &lo) {
    const T ha = f32_to<T>(a), hb = f32_to<T>(b);
    typename Pair<T>::type h;
    h.x = ha;
    h.y = hb;
    hi = *reinterpret_cast<uint32_t *>(&h);
    lo = pack_t<T>(a - to_f32(ha), b - to_f32(hb));
}

template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if constexpr (std::is_same<T, __half>::value) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// element offset of (row, 16-byte chunk) in a [BN][D] tile: the chunk xor-swizzled by the row's low 3 bits
template <int D>
__device__ __forceinline__ int swz(int row, int chunk) { return row * D + ((chunk ^ (row & 7)) << 3); }

// one CTA per token t: k' and v of every KV head into slot start + t
template <typename T, int D>
__global__ void __launch_bounds__(APPEND_THREADS) attn_append_kernel(const ExtParams p) {
    const int t = blockIdx.x, pos = p.start + t;
    const T *qkv = static_cast<const T *>(p.qkv) + (size_t)t * (p.n_heads + 2 * p.n_kv) * D;
    const float *cs = p.cos + (size_t)pos * (D / 2), *sn = p.sin + (size_t)pos * (D / 2);
    for (int idx = threadIdx.x; idx < p.n_kv * D; idx += APPEND_THREADS) {
        const int kvh = idx / D, i = idx % D, j = i % (D / 2);
        const T *k = qkv + (size_t)p.n_heads * D + (size_t)kvh * D;
        const float a = to_f32(k[j]), b = to_f32(k[j + D / 2]);
        const size_t slot = ((size_t)kvh * p.capacity + pos) * D + i;
        static_cast<T *>(p.k_cache)[slot] = f32_to<T>(i < D / 2 ? a * cs[j] - b * sn[j] : b * cs[j] + a * sn[j]);
        static_cast<T *>(p.v_cache)[slot] = qkv[(size_t)(p.n_heads + p.n_kv) * D + (size_t)kvh * D + i];
    }
}

template <typename T, int D>
__global__ void __launch_bounds__(XTHREADS, 1) attn_extend_kernel(const ExtParams p) {
    constexpr int KS = D / 16;        // k-steps of q.k, and 16-column pairs of the output
    constexpr int CH = D / 8;         // 16-byte chunks per K / V row
    extern __shared__ __align__(16) unsigned char xsmem[];
    T *const ks = reinterpret_cast<T *>(xsmem);   // [2][BN][D]
    T *const vs = ks + 2 * BN * D;                // [2][BN][D]
    T *const qhs = vs + 2 * BN * D;               // [BM][D]: q' hi
    T *const qls = qhs + BM * D;                  // [BM][D]: q' lo
    __shared__ float cm[BM], cl[BM];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g8 = lane >> 2, c4 = lane & 3;
    const int S = gridDim.x, rank = (int)rows::cluster_rank();
    const int tile = gridDim.y - 1 - blockIdx.y, kvh = blockIdx.z;
    const int nrows = p.T * p.g, first = tile * BM, last = min(nrows, first + BM) - 1;
    const int t_first = first / p.g, klim = p.start + last / p.g + 1;   // keys [0, klim) of this tile
    const int nb = (klim + BN - 1) / BN, chunk = (nb + S - 1) / S;
    const int kb0 = rank * chunk, kb1 = min(nb, kb0 + chunk);
    const T *kc = static_cast<const T *>(p.k_cache) + (size_t)kvh * p.capacity * D;
    const T *vc = static_cast<const T *>(p.v_cache) + (size_t)kvh * p.capacity * D;

    auto load = [&](int kb, int buf) {
        T *kd = ks + buf * BN * D, *vd = vs + buf * BN * D;
        for (int i = tid; i < BN * CH; i += XTHREADS) {
            const int r = i / CH, ch = i % CH, key = kb * BN + r, off = swz<D>(r, ch);
            if (key < klim) {
                cp_async16(smem_u32(kd + off), kc + (size_t)key * D + ch * 8);
                cp_async16(smem_u32(vd + off), vc + (size_t)key * D + ch * 8);
            } else {
                *reinterpret_cast<uint4 *>(kd + off) = make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4 *>(vd + off) = make_uint4(0, 0, 0, 0);
            }
        }
        cp_async_commit();
    };
    if (kb0 < kb1) load(kb0, 0);

    // q' of the tile's rows as hi / lo parts in shared memory (swizzled like K), read back as A fragments by ldmatrix
    for (int idx = tid; idx < BM * D; idx += XTHREADS) {
        const int r = idx / D, i = idx % D, j = i % (D / 2), rg = first + r;
        float x = 0.f;
        if (rg < nrows) {
            const int t = rg / p.g, pos = p.start + t;
            const T *q = static_cast<const T *>(p.qkv) + (size_t)t * (p.n_heads + 2 * p.n_kv) * D + (size_t)(kvh * p.g + rg % p.g) * D;
            const float a = to_f32(q[j]), b = to_f32(q[j + D / 2]), cs = p.cos[(size_t)pos * (D / 2) + j], sn = p.sin[(size_t)pos * (D / 2) + j];
            x = (i < D / 2 ? a * cs - b * sn : b * cs + a * sn) * QPRE;
        }
        const T h = f32_to<T>(x);
        qhs[swz<D>(r, i >> 3) + (i & 7)] = h;
        qls[swz<D>(r, i >> 3) + (i & 7)] = f32_to<T>(x - to_f32(h));
    }
    // the lane's two rows (g8 and g8 + 8 of its warp's 16): the last key each sees, -1 for a padding row
    int lim[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int rg = first + warp * 16 + g8 + rr * 8;
        lim[rr] = rg < nrows ? p.start + rg / p.g : -1;
    }

    float o[D / 8][4], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < D / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    const int mrow = lane & 7, mi = lane >> 3;   // ldmatrix: the row this lane addresses and its 8x8 matrix

    for (int kb = kb0; kb < kb1; ++kb) {
        const int buf = (kb - kb0) & 1;
        cp_async_wait_all();
        __syncthreads();   // block kb is in; every warp is done with the other stage
        if (kb + 1 < kb1) load(kb + 1, buf ^ 1);
        const uint32_t kbase = smem_u32(ks + buf * BN * D), vbase = smem_u32(vs + buf * BN * D);
        const uint32_t qhb = smem_u32(qhs), qlb = smem_u32(qls);

        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
        for (int kq = 0; kq < KS; ++kq) {
            uint32_t qh[4], ql[4];
            const int qoff = 2 * swz<D>(warp * 16 + (mi & 1) * 8 + mrow, kq * 2 + (mi >> 1));
            ldsm_x4(qhb + qoff, qh[0], qh[1], qh[2], qh[3]);
            ldsm_x4(qlb + qoff, ql[0], ql[1], ql[2], ql[3]);
#pragma unroll
            for (int np = 0; np < 4; ++np) {  // keys 16 np .. 16 np + 15: two n-tiles
                uint32_t b0, b1, b2, b3;
                ldsm_x4(kbase + 2 * swz<D>(np * 16 + (mi >> 1) * 8 + mrow, kq * 2 + (mi & 1)), b0, b1, b2, b3);
                mma16816<T>(s[2 * np], qh, b0, b1);
                mma16816<T>(s[2 * np], ql, b0, b1);
                mma16816<T>(s[2 * np + 1], qh, b2, b3);
                mma16816<T>(s[2 * np + 1], ql, b2, b3);
            }
        }
        const bool edge = kb * BN + BN - 1 > p.start + t_first;   // the block crosses the causal edge of some row of the tile
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kb * BN + n * 8 + 2 * c4 + (e & 1);
                s[n][e] = edge && key > lim[e >> 1] ? -INFINITY : s[n][e] * p.qscale;
            }
        }
        // online softmax per row: the max over the row's 4 lanes, the rescale, the weights
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            mx[0] = fmaxf(mx[0], fmaxf(s[n][0], s[n][1]));
            mx[1] = fmaxf(mx[1], fmaxf(s[n][2], s[n][3]));
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
            mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
            const float corr = wexp2(m[rr], mx[rr]);
            l[rr] *= corr;
#pragma unroll
            for (int n = 0; n < D / 8; ++n) {
                o[n][2 * rr] *= corr;
                o[n][2 * rr + 1] *= corr;
            }
            m[rr] = mx[rr];
        }
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                s[n][e] = wexp2(s[n][e], mx[e >> 1]);
                l[e >> 1] += s[n][e];
            }
        }
        // O += P V, P as hi / lo A fragments straight from the score accumulators
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t ph[4], pl[4];
            split_pair<T>(s[2 * kk][0], s[2 * kk][1], ph[0], pl[0]);
            split_pair<T>(s[2 * kk][2], s[2 * kk][3], ph[1], pl[1]);
            split_pair<T>(s[2 * kk + 1][0], s[2 * kk + 1][1], ph[2], pl[2]);
            split_pair<T>(s[2 * kk + 1][2], s[2 * kk + 1][3], ph[3], pl[3]);
#pragma unroll
            for (int dp = 0; dp < KS; ++dp) {  // output columns 16 dp .. 16 dp + 15: two n-tiles
                uint32_t b0, b1, b2, b3;
                ldsm_x4_t(vbase + 2 * swz<D>(kk * 16 + (mi & 1) * 8 + mrow, dp * 2 + (mi >> 1)), b0, b1, b2, b3);
                mma16816<T>(o[2 * dp], ph, b0, b1);
                mma16816<T>(o[2 * dp], pl, b0, b1);
                mma16816<T>(o[2 * dp + 1], ph, b2, b3);
                mma16816<T>(o[2 * dp + 1], pl, b2, b3);
            }
        }
    }

#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 1);
        l[rr] += __shfl_xor_sync(0xffffffffu, l[rr], 2);
    }
    const int rbase = warp * 16 + g8;   // the lane's first row in the tile
    T *const out = static_cast<T *>(p.out);
    auto out_at = [&](int r) {          // row r of the tile: its output head in out
        const int rg = first + r;
        return out + (size_t)(rg / p.g) * p.n_heads * D + (size_t)(kvh * p.g + rg % p.g) * D;
    };
    if (S == 1) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            if (lim[rr] < 0) continue;
            T *dst = out_at(rbase + rr * 8);
#pragma unroll
            for (int n = 0; n < D / 8; ++n)
                *reinterpret_cast<uint32_t *>(dst + n * 8 + 2 * c4) = pack_t<T>(o[n][2 * rr] / l[rr], o[n][2 * rr + 1] / l[rr]);
        }
        return;
    }
    // the CTAs of the cluster, in rank order: each leaves (m, l, acc) of its rows in shared memory; CTA r finishes the elements r,
    // r + S*XTHREADS, ... of the tile
    cp_async_wait_all();
    __syncthreads();
    float *const cacc = reinterpret_cast<float *>(xsmem);   // [BM][D]
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int r = rbase + rr * 8;
#pragma unroll
        for (int n = 0; n < D / 8; ++n) {
            cacc[r * D + n * 8 + 2 * c4] = o[n][2 * rr];
            cacc[r * D + n * 8 + 2 * c4 + 1] = o[n][2 * rr + 1];
        }
        if (c4 == 0) { cm[r] = m[rr]; cl[r] = l[rr]; }
    }
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
    for (int idx = rank * XTHREADS + tid; idx < BM * D; idx += S * XTHREADS) {
        const int r = idx / D, i = idx % D;
        if (first + r >= nrows) continue;
        float mr[MAX_CLUSTER], mxr = -INFINITY;
#pragma unroll
        for (int q = 0; q < MAX_CLUSTER; ++q) {
            if (q < S) { mr[q] = ld_cluster_f32(&cm[r], q); mxr = fmaxf(mxr, mr[q]); }
        }
        float L = 0.f, A = 0.f;
#pragma unroll
        for (int q = 0; q < MAX_CLUSTER; ++q) {
            if (q < S) {
                const float c = wexp2(mr[q], mxr);
                L += ld_cluster_f32(&cl[r], q) * c;
                A += ld_cluster_f32(&cacc[r * D + i], q) * c;
            }
        }
        out_at(r)[i] = f32_to<T>(A / L);
    }
    asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;" ::: "memory");  // the peers' partials stay alive until read
}

}  // namespace attn
}  // namespace
