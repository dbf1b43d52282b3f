// sample.cu - one token per row of logits behind sqllm_sample: greedy, or temperature, top-k and top-p filtering followed by a
// Gumbel-max draw from Philox4x32-10 words keyed by the row's seed and counted by its position (the contract: sqllm_b200.h).
//
// One thread-block cluster per row; its CTAs split the row in contiguous slices of quads (4 consecutive tokens share one Philox call).
// The cluster size is a function of the vocabulary alone, and every cross-CTA quantity is either an integer sum (exact in any order)
// or an argmax under a total order (ties to the lower index), so a row's token does not depend on the launch shape, the other rows
// or the SM count.  The thresholds are found by radix select on an order-preserving uint32 key of z = x / t: count histograms for
// top-k, count and fixed-point mass histograms (exp(z - z_max) in units of 2^-44, summed as uint64) for top-p.  Every pass re-reads
// the CTA's slice of the row (at most CHUNK tokens, L1/L2-resident); nothing is allocated and nothing is written but out[b].
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "host.h"

namespace cg = cooperative_groups;
using namespace sqllm;

namespace {

constexpr int THREADS = 512, WARPS = THREADS / 32;
constexpr int CHUNK = 16384;                   // tokens per CTA of a row's cluster (at most)
constexpr int MAX_CLUSTER = 8;                 // portable cluster size: 8 x 16384 covers MAX_VOCAB
constexpr int MAX_ROWS = 65535, MAX_VOCAB = 262144;
constexpr int NBIN = 2048, BPT = NBIN / THREADS;  // histogram bins (11-bit digits), bins per thread in the scans
constexpr int LEVELS = 3;                      // digits of 11, 11 and 10 bits, most significant first
__device__ __forceinline__ int digit_shift(int L) { return L == 0 ? 21 : L == 1 ? 10 : 0; }
__device__ __forceinline__ unsigned digit_mask(int L) { return L == 2 ? 0x3ffu : 0x7ffu; }
constexpr float MASS_ONE = 17592186044416.f;   // 2^44: a mass of 1 (the maximum's) in fixed point; V 2^44 < 2^63

__host__ __device__ constexpr int cluster_size(int V) { return V > (MAX_CLUSTER - 1) * CHUNK ? MAX_CLUSTER : (V + CHUNK - 1) / CHUNK; }

struct Params {
    const void *x;
    const int *pos;
    const float *temperature, *top_p;
    const int *top_k;
    const unsigned long long *seed;
    long long *out;
    long long stride;
    int V;
};

struct Smem {
    unsigned cnt[NBIN];
    unsigned long long mass[NBIN];
    float wv[WARPS];
    int wi[WARPS];
    float best_v[2];                    // this CTA's argmax of pass 1 and of the draw, read by the whole cluster
    int best_i[2];
    unsigned long long wsum[2][WARPS];  // per-warp totals of the scans (counts, masses)
    int sel;                            // the selected bin of a radix level
    unsigned sel_cnt;
    unsigned long long sel_above;       // count (top-k) or mass (top-p) above the selected bin
};

template <typename T>
__device__ __forceinline__ float ld(const T *p) { return static_cast<float>(*p); }
template <>
__device__ __forceinline__ float ld<__half>(const __half *p) { return __half2float(*p); }
template <>
__device__ __forceinline__ float ld<__nv_bfloat16>(const __nv_bfloat16 *p) { return __bfloat162float(*p); }

// order-preserving key of a non-NaN float, with -0 and +0 equal (z >= z_k compares them as equal)
__device__ __forceinline__ unsigned zkey(float z) {
    const unsigned b = z == 0.f ? 0u : __float_as_uint(z);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// torch.argmax's order: NaN above everything, then the larger value; ties to the lower index
__device__ __forceinline__ bool better(float a, int ia, float b, int ib) {
    const bool na = a != a, nb = b != b;
    if (na || nb) return na && (!nb || ia < ib);
    return a > b || (a == b && ia < ib);
}

// Philox4x32-10 (Salmon et al., SC'11): the block of counter c under key (k0, k1)
__device__ __forceinline__ uint4 philox(uint4 c, unsigned k0, unsigned k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// Gumbel noise of a word: u = ((w >> 9) + 1/2) 2^-23 is exact in fp32 and in [2^-24, 1 - 2^-24], so g is finite (|g| < 17)
__device__ __forceinline__ float gumbel(unsigned w) {
    const float u = (static_cast<float>(w >> 9) + 0.5f) * 0x1p-23f;
    return -logf(-logf(u));
}

// The argmax of (v, i) over the cluster, under `better`: block reduction, then every CTA reads the CTAs' results in rank order.
// Returns the same (v, i) in every thread of every CTA.  `slot` keeps the two reductions of a row apart (no CTA overwrites a result
// another may still read).
__device__ void cluster_argmax(cg::cluster_group &cl, Smem &s, int slot, float &v, int &i) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (better(ov, oi, v, i)) { v = ov; i = oi; }
    }
    if (lane == 0) { s.wv[warp] = v; s.wi[warp] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < WARPS; ++w)
            if (better(s.wv[w], s.wi[w], v, i)) { v = s.wv[w]; i = s.wi[w]; }
        s.best_v[slot] = v;
        s.best_i[slot] = i;
    }
    cl.sync();
    v = -INFINITY;
    i = INT_MAX;
    for (unsigned r = 0; r < cl.num_blocks(); ++r) {
        const Smem *o = cl.map_shared_rank(&s, r);
        const float ov = o->best_v[slot];
        const int oi = o->best_i[slot];
        if (better(ov, oi, v, i)) { v = ov; i = oi; }
    }
}

// Exclusive suffix sums of the cluster-wide histogram over this thread's bins BPT t .. BPT t + BPT - 1: above[j] = the sum over the
// bins above bin BPT t + j.  c[] holds the bins' totals.  Returns the grand total.  Integer sums: exact in any order.
template <typename U>
__device__ U suffix_scan(Smem &s, int which, const U (&c)[BPT], U (&above)[BPT]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    U own = 0;
#pragma unroll
    for (int j = 0; j < BPT; ++j) own += c[j];
    U incl = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const U y = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += y;
    }
    if (lane == 0) s.wsum[which][warp] = incl;
    __syncthreads();
    U acc = incl - own, total = 0;
    for (int w = 0; w < WARPS; ++w) {
        const U t = s.wsum[which][w];
        total += t;
        if (w > warp) acc += t;
    }
#pragma unroll
    for (int j = BPT - 1; j >= 0; --j) {
        above[j] = acc;
        acc += c[j];
    }
    return total;
}

template <typename T>
__global__ void __launch_bounds__(THREADS, 2) sample_kernel(const Params p) {
    __shared__ Smem s;
    cg::cluster_group cl = cg::this_cluster();
    const int b = blockIdx.y;
    const int pos = p.pos[b];
    if (pos < 0) return;  // an idle row: its whole cluster leaves before any cluster barrier
    const int V = p.V, C = (int)cl.num_blocks(), rank = (int)cl.block_rank();
    const int Q = (V + 3) >> 2, per = (Q + C - 1) / C;
    const int q0 = rank * per, q1 = min(Q, q0 + per);
    const T *x = static_cast<const T *>(p.x) + (long long)b * p.stride;
    const int tid = threadIdx.x;

    // pass 1: torch.argmax of the row
    float xm = -INFINITY;
    int im = INT_MAX;
    for (int q = q0 + tid; q < q1; q += THREADS)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = 4 * q + j;
            if (i < V) {
                const float v = ld(x + i);
                if (better(v, i, xm, im)) { xm = v; im = i; }
            }
        }
    cluster_argmax(cl, s, 0, xm, im);

    const float t = p.temperature[b];
    const float zmax = xm / t;
    int result = im;
    // greedy: t <= 0 or NaN; also a row whose z maximum is not finite (a NaN or +inf logit, no finite logit, or x / t overflowing)
    if (t > 0.f && isfinite(zmax)) {
        const int k = p.top_k[b];
        const float top_p = p.top_p[b];
        unsigned thr = 0;  // the kept tokens: zkey(z) >= thr
        if (k > 0 && k < V) {
            // top-k: the key of the k-th largest z (counted with multiplicity), or the lower bound of a bin that holds exactly the
            // tokens of rank <= k not already above it
            unsigned prefix = 0, mask = 0, rem = (unsigned)k;
            for (int L = 0; L < LEVELS; ++L) {
                const int sh = digit_shift(L);
                const unsigned dm = digit_mask(L);
                cl.sync();  // every CTA has read the previous level's histograms
                for (int d = tid; d < NBIN; d += THREADS) s.cnt[d] = 0;
                __syncthreads();
                for (int q = q0 + tid; q < q1; q += THREADS)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int i = 4 * q + j;
                        if (i < V) {
                            const unsigned key = zkey(ld(x + i) / t);
                            if ((key & mask) == prefix) atomicAdd(&s.cnt[(key >> sh) & dm], 1u);
                        }
                    }
                cl.sync();
                unsigned c[BPT], above[BPT];
#pragma unroll
                for (int j = 0; j < BPT; ++j) c[j] = 0;
                for (unsigned r = 0; r < cl.num_blocks(); ++r) {
                    const Smem *o = cl.map_shared_rank(&s, r);
#pragma unroll
                    for (int j = 0; j < BPT; ++j) c[j] += o->cnt[BPT * tid + j];
                }
                suffix_scan<unsigned>(s, 0, c, above);
#pragma unroll
                for (int j = 0; j < BPT; ++j)
                    if (above[j] < rem && rem <= above[j] + c[j]) { s.sel = BPT * tid + j; s.sel_above = above[j]; s.sel_cnt = c[j]; }
                __syncthreads();
                rem -= (unsigned)s.sel_above;
                prefix |= (unsigned)s.sel << sh;
                mask |= dm << sh;
                if (s.sel_cnt == rem) break;  // the whole bin is kept, nothing below it
            }
            thr = prefix;
        }
        if (top_p < 1.f) {
            // top-p over the tokens top-k kept: the lowest non-empty bin whose mass above, A + above, is < top_p S holds the smallest
            // kept z (the largest token of a bin has exactly that mass above it); refine inside it
            unsigned prefix = 0, mask = 0, tp = zkey(zmax);
            unsigned long long A = 0;
            double pS = 0.0;
            for (int L = 0; L < LEVELS; ++L) {
                const int sh = digit_shift(L);
                const unsigned dm = digit_mask(L);
                cl.sync();
                for (int d = tid; d < NBIN; d += THREADS) { s.cnt[d] = 0; s.mass[d] = 0; }
                if (tid == 0) s.sel = NBIN;
                __syncthreads();
                for (int q = q0 + tid; q < q1; q += THREADS)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int i = 4 * q + j;
                        if (i < V) {
                            const float z = ld(x + i) / t;
                            const unsigned key = zkey(z);
                            if (key >= thr && (key & mask) == prefix) {
                                const int d = (key >> sh) & dm;
                                atomicAdd(&s.cnt[d], 1u);
                                const unsigned long long m = __float2ull_rn(expf(z - zmax) * MASS_ONE);
                                if (m) atomicAdd(&s.mass[d], m);
                            }
                        }
                    }
                cl.sync();
                unsigned c[BPT];
                unsigned long long m[BPT], above[BPT];
#pragma unroll
                for (int j = 0; j < BPT; ++j) { c[j] = 0; m[j] = 0; }
                for (unsigned r = 0; r < cl.num_blocks(); ++r) {
                    const Smem *o = cl.map_shared_rank(&s, r);
#pragma unroll
                    for (int j = 0; j < BPT; ++j) { c[j] += o->cnt[BPT * tid + j]; m[j] += o->mass[BPT * tid + j]; }
                }
                const unsigned long long S = suffix_scan<unsigned long long>(s, 1, m, above);
                if (L == 0) pS = (double)top_p * (double)S;
#pragma unroll
                for (int j = 0; j < BPT; ++j)
                    if (c[j] && (double)(A + above[j]) < pS) atomicMin(&s.sel, BPT * tid + j);
                __syncthreads();
                const int sel = s.sel;
                if (sel == NBIN) break;  // top_p <= 0: only the maximum (tp = its key) is kept
#pragma unroll
                for (int j = 0; j < BPT; ++j)
                    if (BPT * tid + j == sel) { s.sel_above = above[j]; s.sel_cnt = c[j]; }
                __syncthreads();
                A += s.sel_above;
                prefix |= (unsigned)sel << sh;
                mask |= dm << sh;
                tp = prefix;
                if (s.sel_cnt == 1) break;  // one token: kept, and nothing below the bin is
            }
            thr = max(thr, tp);
        }
        // the draw: the kept token with the largest z + g, ties to the lower index
        const unsigned k0 = (unsigned)p.seed[b], k1 = (unsigned)(p.seed[b] >> 32);
        float sv = -INFINITY;
        int si = INT_MAX;
        for (int q = q0 + tid; q < q1; q += THREADS) {
            float z[4];
            bool keep[4], any = false;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * q + j;
                z[j] = i < V ? ld(x + i) / t : -INFINITY;
                keep[j] = i < V && zkey(z[j]) >= thr;
                any |= keep[j];
            }
            if (!any) continue;
            const uint4 w = philox(make_uint4((unsigned)q, (unsigned)pos, 0u, 0u), k0, k1);
            const unsigned ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (keep[j]) {
                    const float sc = z[j] + gumbel(ws[j]);
                    if (better(sc, 4 * q + j, sv, si)) { sv = sc; si = 4 * q + j; }
                }
        }
        cluster_argmax(cl, s, 1, sv, si);
        if (si < V) result = si;
    }
    if (rank == 0 && tid == 0) p.out[b] = result;
    cl.sync();  // the peers' results stay alive until read
}

template <typename T>
void (*kernel_of())(Params) { return sample_kernel<T>; }

int sample_launch(const sqllm_sample_args *a, void *stream) {
    if (!dt_valid(a->dtype))
        return fail(SQLLM_EINVAL, "dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", a->dtype);
    if (a->rows < 1 || a->rows > MAX_ROWS) return fail(SQLLM_EINVAL, "rows=%d must be in [1, %d]", a->rows, MAX_ROWS);
    if (a->vocab < 1 || a->vocab > MAX_VOCAB) return fail(SQLLM_EINVAL, "vocab=%d must be in [1, %d]", a->vocab, MAX_VOCAB);
    if (a->row_stride < a->vocab)
        return fail(SQLLM_EINVAL, "row_stride=%lld must be >= vocab=%d", (long long)a->row_stride, a->vocab);
    const int esize = a->dtype == SQLLM_DT_F32 ? 4 : 2;
    struct NamedPtr {
        const void *p;
        int align;
        const char *name;
    };
    for (const NamedPtr &q : {NamedPtr{a->logits, esize, "logits"}, NamedPtr{a->pos, 4, "pos"}, NamedPtr{a->temperature, 4, "temperature"},
                              NamedPtr{a->top_k, 4, "top_k"}, NamedPtr{a->top_p, 4, "top_p"}, NamedPtr{a->seed, 8, "seed"},
                              NamedPtr{a->out, 8, "out"}})
        if (!q.p || reinterpret_cast<uintptr_t>(q.p) % q.align)
            return fail(SQLLM_EINVAL, "%s must be a non-null pointer aligned to %d bytes", q.name, q.align);
    if (int rc = dev_setup({})) return rc;
    Params p;
    p.x = a->logits; p.pos = a->pos; p.temperature = a->temperature; p.top_p = a->top_p; p.top_k = a->top_k;
    p.seed = reinterpret_cast<const unsigned long long *>(a->seed); p.out = reinterpret_cast<long long *>(a->out);
    p.stride = a->row_stride; p.V = a->vocab;
    void (*fn)(Params) = a->dtype == SQLLM_DT_F32 ? kernel_of<float>() : a->dtype == SQLLM_DT_F16 ? kernel_of<__half>() : kernel_of<__nv_bfloat16>();
    const int C = cluster_size(a->vocab);
    const cudaError_t e = launch_ex(fn, dim3(C, a->rows), THREADS, 0, static_cast<cudaStream_t>(stream), cluster_of(C), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "sample launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // namespace

extern "C" {

int sqllm_sample(const sqllm_sample_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return sample_launch(a, stream);
}

}  // extern "C"
