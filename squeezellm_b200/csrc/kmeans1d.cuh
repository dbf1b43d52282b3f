// kmeans1d.cuh - exact weighted 1-D k-means per output channel (the codebook fit of SqueezeLLM's quantizer,
// reference quantization/nuq.py:50-58 + :164-176), and the GPU pack of the resulting labels into qweight.
//
// One CTA per row.  The row's (w, s) pairs arrive sorted by w (cub segmented radix sort, stable, in the host code), and
//   1. the weighted mean mu and fp64 prefix sums of s, s (w - mu), s (w - mu)^2 go to the workspace (centring limits
//      cancellation in Q - X^2 / W);
//   2. D_m(j) = min_{i<j} D_{m-1}(i) + cost(i, j) over the sorted points, cost(i, j) = Q - X^2 / W of [i, j) (0 when W = 0),
//      is solved level by level.  The leftmost argmin is monotone in j (the cost is Monge), so each level is a divide and
//      conquer over j, run breadth-first: at depth d the 2^d nodes are independent, and a node [lo, hi] scans
//      i in [opt(lo - 1), min(opt(hi + 1), mid - 1)] (the positions lo - 1 and hi + 1 were the midpoints of its ancestors).
//      The block splits into groups of THREADS / 2^d threads, one node per group; ties go to the smallest i;
//   3. thread 0 backtracks the k segments, centroid = X / W + mu rounded to fp32; a segment with W = 0 (fewer than k distinct
//      values of positive weight) takes the centroid of the nearest non-empty segment below it, else above;
//   4. every element of the original row gets label = #{j : w > fl32(0.5f (c[j-1] + c[j]))}: the nearest centroid, ties to the
//      lower index.
// Every sum has a fixed order and every argmin is a lexicographic (value, index) minimum, so a row's result depends on that row
// alone: not on the other rows, the chunking, the stream or the run.
#pragma once

namespace km {

constexpr int THREADS = 256;
constexpr int MAX_K = 16;
constexpr int MAX_N = 65535;  // opt[] is uint16

// A row whose sample weights are all zero is weighted uniformly (reference nuq.py:174-175 does the same before k-means).
struct Row {
    int n, k;
    const float *ws, *ss;  // sorted w, s  [n]
    double *pw, *px, *pq;  // prefix sums  [n + 1]
    double *d0, *d1;       // D of two consecutive levels  [n + 1]
    uint16_t *opt;         // argmin of levels 2..k  [(k - 1)][n + 1]
};

__device__ __forceinline__ double seg_cost(const Row &r, int i, double pwj, double pxj, double pqj) {
    const double W = pwj - r.pw[i];
    if (!(W > 0.0)) return 0.0;
    const double X = pxj - r.px[i];
    return fmax(pqj - r.pq[i] - X * X / W, 0.0);
}

__device__ __forceinline__ void take_min(double &bv, int &bi, double v, int i) {
    if (v < bv || (v == bv && i < bi)) { bv = v; bi = i; }
}

__global__ void kmeans1d_kernel(const float *__restrict__ w_sorted, const float *__restrict__ s_sorted,
                                                           const float *__restrict__ w_orig, int n, int k, double *__restrict__ ws_pref,
                                                           double *__restrict__ ws_d, uint16_t *__restrict__ ws_opt,
                                                           float *__restrict__ centroids, uint8_t *__restrict__ labels) {
    __shared__ double part[3][THREADS];
    __shared__ double red_v[THREADS / 32];
    __shared__ int red_i[THREADS / 32];
    __shared__ double s_mu;
    __shared__ int s_uniform;
    __shared__ float s_thr[MAX_K];
    __shared__ float s_c[MAX_K];
    __shared__ int s_bound[MAX_K + 1];

    const int t = threadIdx.x, row = blockIdx.x;
    const size_t n1 = (size_t)n + 1;
    Row r;
    r.n = n; r.k = k;
    r.ws = w_sorted + (size_t)row * n;
    r.ss = s_sorted + (size_t)row * n;
    r.pw = ws_pref + (size_t)row * 3 * n1;
    r.px = r.pw + n1;
    r.pq = r.px + n1;
    r.d0 = ws_d + (size_t)row * 2 * n1;
    r.d1 = r.d0 + n1;
    r.opt = ws_opt + (size_t)row * (k - 1) * n1;

    // ---- 1. weighted mean and prefix sums (each thread a contiguous run, combined by thread 0 in index order) -------------
    const int per = (n + THREADS - 1) / THREADS;
    const int e0 = min(n, t * per), e1 = min(n, e0 + per);
    {
        double a = 0.0, b = 0.0;
        for (int e = e0; e < e1; ++e) { a += (double)r.ss[e]; b += (double)r.ss[e] * (double)r.ws[e]; }
        part[0][t] = a; part[1][t] = b;
    }
    __syncthreads();
    if (t == 0) {
        double a = 0.0, b = 0.0, c = 0.0;
        for (int i = 0; i < THREADS; ++i) { a += part[0][i]; b += part[1][i]; }
        s_uniform = !(a > 0.0);
        if (s_uniform) {
            for (int e = 0; e < n; ++e) c += (double)r.ws[e];
            s_mu = c / n;
        } else {
            s_mu = b / a;
        }
    }
    __syncthreads();
    const double mu = s_mu;
    const bool uniform = s_uniform;
    {
        double a = 0.0, b = 0.0, c = 0.0;
        for (int e = e0; e < e1; ++e) {
            const double s = uniform ? 1.0 : (double)r.ss[e], d = (double)r.ws[e] - mu;
            a += s; b += s * d; c += s * d * d;
        }
        part[0][t] = a; part[1][t] = b; part[2][t] = c;
    }
    __syncthreads();
    if (t == 0) {  // exclusive scan of the runs' totals
        double a = 0.0, b = 0.0, c = 0.0;
        for (int i = 0; i < THREADS; ++i) {
            const double ta = part[0][i], tb = part[1][i], tc = part[2][i];
            part[0][i] = a; part[1][i] = b; part[2][i] = c;
            a += ta; b += tb; c += tc;
        }
        r.pw[0] = r.px[0] = r.pq[0] = 0.0;
    }
    __syncthreads();
    {
        double a = part[0][t], b = part[1][t], c = part[2][t];
        for (int e = e0; e < e1; ++e) {
            const double s = uniform ? 1.0 : (double)r.ss[e], d = (double)r.ws[e] - mu;
            a += s; b += s * d; c += s * d * d;
            r.pw[e + 1] = a; r.px[e + 1] = b; r.pq[e + 1] = c;
        }
    }
    __syncthreads();

    // ---- 2. the DP: level 1 directly, levels 2..k by breadth-first divide and conquer ---------------------------------------
    for (int j = t; j <= n; j += THREADS) r.d1[j] = seg_cost(r, 0, r.pw[j], r.px[j], r.pq[j]);
    __syncthreads();
    for (int m = 2; m <= k; ++m) {
        const double *dprev = (m & 1) ? r.d0 : r.d1;
        double *dcur = (m & 1) ? r.d1 : r.d0;
        uint16_t *opt = r.opt + (size_t)(m - 2) * n1;
        const int jlo = m < k ? m : n;  // the last level needs only j = n
        const int L = n - jlo + 1;
        for (int d = 0; (1 << d) <= L; ++d) {
            const int nodes = 1 << d;
            const int G = nodes >= THREADS ? 1 : THREADS / nodes;  // threads per node
            const int concurrent = THREADS / G;
            const int g = t % G;
            for (int base = 0; base < nodes; base += concurrent) {  // same trip count in every thread
                const int p = base + t / G;
                double bv = INFINITY;
                int bi = INT_MAX, mid = -1;
                if (p < nodes) {
                    int lo = jlo, hi = n;
                    for (int b = d - 1; b >= 0 && lo <= hi; --b) {
                        const int md = (lo + hi) >> 1;
                        if ((p >> b) & 1) lo = md + 1; else hi = md - 1;
                    }
                    if (lo <= hi) {
                        mid = (lo + hi) >> 1;
                        const int ol = lo - 1 >= jlo ? (int)opt[lo - 1] : m - 1;
                        const int oh = min(hi + 1 <= n ? (int)opt[hi + 1] : n - 1, mid - 1);
                        const double pwj = r.pw[mid], pxj = r.px[mid], pqj = r.pq[mid];
                        for (int i = ol + g; i <= oh; i += G) {
                            const double v = dprev[i] + seg_cost(r, i, pwj, pxj, pqj);
                            if (v < bv) { bv = v; bi = i; }  // i increases: strict < keeps the smallest i
                        }
                    }
                }
                for (int off = min(G, 32) >> 1; off > 0; off >>= 1) {
                    const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                    take_min(bv, bi, ov, oi);
                }
                if (G > 32) {  // one node per group of whole warps: combine the warps' results
                    if ((t & 31) == 0) { red_v[t >> 5] = bv; red_i[t >> 5] = bi; }
                    __syncthreads();
                    if (g == 0)
                        for (int w = (t >> 5) + 1; w < (t + G) >> 5; ++w) take_min(bv, bi, red_v[w], red_i[w]);
                    __syncthreads();
                }
                if (g == 0 && mid >= 0) { dcur[mid] = bv; opt[mid] = (uint16_t)bi; }
            }
            __syncthreads();
        }
    }

    // ---- 3. backtrack, centroids ------------------------------------------------------------------------------------------
    if (t == 0) {
        int *bound = s_bound;
        bound[k] = n;
        for (int m = k; m >= 2; --m) bound[m - 1] = r.opt[(size_t)(m - 2) * n1 + bound[m]];
        bound[0] = 0;
    }
    __syncthreads();
    if (t < k) {  // segment t; a segment without weight is marked NaN and filled below
        const double W = r.pw[s_bound[t + 1]] - r.pw[s_bound[t]];
        s_c[t] = W > 0.0 ? (float)((r.px[s_bound[t + 1]] - r.px[s_bound[t]]) / W + mu) : __int_as_float(0x7fc00000);
    }
    __syncthreads();
    if (t == 0) {
        float *c = s_c;
        for (int q = 0; q < k; ++q) {
            if (!isnan(c[q])) continue;
            float v = 0.0f;
            bool found = false;
            for (int b = q - 1; b >= 0 && !found; --b) if (!isnan(c[b])) { v = c[b]; found = true; }
            for (int b = q + 1; b < k && !found; ++b) if (!isnan(c[b])) { v = c[b]; found = true; }
            c[q] = v;  // a filled segment below holds the value its nearest non-empty one would give
        }
        for (int q = 1; q < k; ++q) c[q] = fmaxf(c[q], c[q - 1]);  // rounding of X / W + mu must not break the order
        for (int q = 1; q < k; ++q) s_thr[q] = 0.5f * (c[q - 1] + c[q]);
    }
    __syncthreads();
    if (t < k) centroids[(size_t)row * k + t] = s_c[t];

    // ---- 4. labels of the original row: nearest centroid, ties to the lower index ------------------------------------------
    const float *wrow = w_orig + (size_t)row * n;
    uint8_t *lrow = labels + (size_t)row * n;
    for (int e = t; e < n; e += THREADS) {
        const float v = wrow[e];
        int lab = 0;
        for (int q = 1; q < k; ++q) lab += v > s_thr[q];
        lrow[e] = (uint8_t)lab;
    }
}

// labels uint8 [N, K] (row = output channel) -> qweight int32 [K/32*bits, N] in the layout of the reference's pack2
// (quant.py:171-208): 4-bit, word r of a column holds indices 8r..8r+7 at 4-bit steps; 3-bit, 32 indices in 3 words with
// index 10 and 21 straddling word boundaries.  One thread per (column, group of 32 indices).
__global__ void pack_indices_kernel(int bits, const uint8_t *__restrict__ labels, int K, int N, uint32_t *__restrict__ q) {
    const int groups = K / 32;
    const size_t total = (size_t)groups * N;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(e / N), c = (int)(e % N);
        const uint8_t *src = labels + (size_t)c * K + (size_t)g * 32;
        uint32_t v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = src[i] & ((1u << bits) - 1u);
        if (bits == 4) {
#pragma unroll
            for (int wd = 0; wd < 4; ++wd) {
                uint32_t x = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) x |= v[8 * wd + i] << (4 * i);
                q[(size_t)(4 * g + wd) * N + c] = x;
            }
        } else {
            uint32_t w0 = v[10] << 30, w1 = (v[10] >> 2) & 1u, w2 = (v[21] >> 1) & 3u;
#pragma unroll
            for (int i = 0; i < 10; ++i) {
                w0 |= v[i] << (3 * i);
                w1 |= v[11 + i] << (3 * i + 1);
                w2 |= v[22 + i] << (3 * i + 2);
            }
            w1 |= v[21] << 31;
            q[(size_t)(3 * g) * N + c] = w0;
            q[(size_t)(3 * g + 1) * N + c] = w1;
            q[(size_t)(3 * g + 2) * N + c] = w2;
        }
    }
}

__global__ void segment_offsets_kernel(int *offs, int rows, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= rows; i += gridDim.x * blockDim.x) offs[i] = i * n;
}

}  // namespace km
