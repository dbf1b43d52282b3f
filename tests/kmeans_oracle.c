/*
 * TEST INFRASTRUCTURE ONLY - exact weighted 1-D k-means, the checker of the GPU quantizer (squeezellm_b200/quantize.py,
 * csrc/kmeans1d.cuh).  Compiled by tests/kmeans_oracle.py into a temporary directory (gcc -O2 -fopenmp); never linked into
 * the product.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>
/* ---------------------------------------------------------------------------------------------
 * Exact weighted 1-D k-means of each row (the problem reference quantization/nuq.py:50-58 poses to sklearn's
 * KMeans per output channel), as the checker of the GPU quantizer.  Independent of the CUDA code: qsort by (w, index),
 * long double prefix sums centred on the row's weighted mean, a depth-first divide-and-conquer DP per level (leftmost
 * argmin), OpenMP over rows.  A row whose sample weights are all zero is weighted uniformly (nuq.py:174-175).
 * Out: opt[r] = the minimum of sum s (w - c)^2; centroids[r][k] = the segment means (a segment without weight takes the
 * nearest weighted segment's mean below it, else above); labels[r][n] = each element's segment.
 * ------------------------------------------------------------------------------------------- */
#include <math.h>
#include <stdlib.h>

typedef struct { float w, s; int i; } km_pt;

static int km_cmp(const void *a, const void *b) {
    const km_pt *x = (const km_pt *)a, *y = (const km_pt *)b;
    if (x->w < y->w) return -1;
    if (x->w > y->w) return 1;
    return (x->i > y->i) - (x->i < y->i);
}

typedef struct {
    const long double *W, *X, *Q, *prev;
    long double *cur;
    int *opt;
} km_level;

static long double km_cost(const km_level *L, int i, int j) {
    const long double W = L->W[j] - L->W[i];
    if (!(W > 0)) return 0;
    const long double X = L->X[j] - L->X[i], c = L->Q[j] - L->Q[i] - X * X / W;
    return c > 0 ? c : 0;
}

static void km_solve(const km_level *L, int lo, int hi, int ol, int oh) {
    if (lo > hi) return;
    const int mid = lo + (hi - lo) / 2, top = oh < mid - 1 ? oh : mid - 1;
    long double best = INFINITY;
    int arg = ol;
    for (int i = ol; i <= top; ++i) {
        const long double v = L->prev[i] + km_cost(L, i, mid);
        if (v < best) { best = v; arg = i; }
    }
    L->cur[mid] = best;
    L->opt[mid] = arg;
    km_solve(L, lo, mid - 1, ol, arg);
    km_solve(L, mid + 1, hi, arg, oh);
}

void sq_kmeans1d(const float *w, const float *s, int rows, int n, int k, double *opt, double *centroids, uint8_t *labels) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int r = 0; r < rows; ++r) {
        const size_t n1 = (size_t)n + 1;
        km_pt *p = malloc(sizeof(km_pt) * n);
        long double *pre = malloc(sizeof(long double) * 3 * n1), *D = malloc(sizeof(long double) * (size_t)k * n1);
        int *arg = malloc(sizeof(int) * (size_t)k * n1);
        long double tot = 0, mom = 0;
        for (int e = 0; e < n; ++e) {
            p[e].w = w[(size_t)r * n + e]; p[e].s = s[(size_t)r * n + e]; p[e].i = e;
            tot += p[e].s; mom += (long double)p[e].s * p[e].w;
        }
        const int uniform = !(tot > 0);
        if (uniform) {
            mom = 0;
            for (int e = 0; e < n; ++e) { p[e].s = 1.0f; mom += p[e].w; }
            tot = n;
        }
        const long double mu = mom / tot;
        qsort(p, n, sizeof(km_pt), km_cmp);
        long double *W = pre, *X = pre + n1, *Q = pre + 2 * n1;
        W[0] = X[0] = Q[0] = 0;
        for (int e = 0; e < n; ++e) {
            const long double d = (long double)p[e].w - mu;
            W[e + 1] = W[e] + p[e].s; X[e + 1] = X[e] + p[e].s * d; Q[e + 1] = Q[e] + p[e].s * d * d;
        }
        km_level L = {W, X, Q, NULL, NULL, NULL};
        for (int j = 0; j <= n; ++j) D[j] = km_cost(&L, 0, j);
        for (int m = 2; m <= k; ++m) {
            L.prev = D + (size_t)(m - 2) * n1;
            L.cur = D + (size_t)(m - 1) * n1;
            L.opt = arg + (size_t)(m - 1) * n1;
            km_solve(&L, m, n, m - 1, n - 1);
        }
        opt[r] = (double)D[(size_t)(k - 1) * n1 + n];
        int b[256 + 1];
        b[k] = n;
        for (int m = k; m >= 2; --m) b[m - 1] = arg[(size_t)(m - 1) * n1 + b[m]];
        b[0] = 0;
        double *c = centroids + (size_t)r * k;
        for (int q = 0; q < k; ++q) {
            const long double Wq = W[b[q + 1]] - W[b[q]];
            c[q] = Wq > 0 ? (double)((X[b[q + 1]] - X[b[q]]) / Wq + mu) : NAN;
            for (int e = b[q]; e < b[q + 1]; ++e) labels[(size_t)r * n + p[e].i] = (uint8_t)q;
        }
        for (int q = 0; q < k; ++q) {
            if (!isnan(c[q])) continue;
            int src = -1;
            for (int t = q - 1; t >= 0 && src < 0; --t) if (!isnan(c[t])) src = t;
            for (int t = q + 1; t < k && src < 0; ++t) if (!isnan(c[t])) src = t;
            c[q] = src >= 0 ? c[src] : 0.0;
        }
        free(p); free(pre); free(D); free(arg);
    }
}
