/*
 * TEST INFRASTRUCTURE ONLY - CPU restatement of SqueezeLLM's dense-and-sparse LUT GEMV path.
 *
 * This file is the parity oracle for squeezellm_b200's CUDA kernels.  It is never linked into or
 * called from the product (squeezellm_b200/, the C-ABI library, the `quant_cuda` module): only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may use it.
 *
 * Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4), and its only
 * compute path is CUDA.  The oracle is pinned two ways:
 *   (1) format: tests/golden/pack2_*.npz are produced by the reference's own
 *       QuantLinearLUT.pack2 (squeezellm/quant.py:97-208) run in this container; the unpack below
 *       must reproduce the packed indices bit-exactly (tests/test_oracle_golden.py);
 *   (2) arithmetic: tests/golden/refkernel_*.npz are outputs of the reference's own kernels
 *       (oracle/_ref, built by oracle/build_ref.py) executed on an H100; the fp64 results below must
 *       agree with them to fp32-accumulation tolerance.
 *
 * Every function cites the reference lines it restates (paths relative to /root/reference).
 *
 * Build: see oracle/Makefile  (gcc -O2 -fopenmp -shared -fPIC).
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

int sq_oracle_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ---------------------------------------------------------------------------------------------
 * Index extraction.  4-bit: squeezellm/quant_cuda_kernel.cu:863-877 (word r holds inputs 8r..8r+7,
 * input 8r+j at bits [4j,4j+4)), inverse of squeezellm/quant.py:180-184.
 * 3-bit: squeezellm/quant_cuda_kernel.cu:776-825 (three words hold 32 inputs: 10 + straddler + 10
 * + straddler + 10), inverse of squeezellm/quant.py:185-203.
 * ------------------------------------------------------------------------------------------- */
static inline unsigned idx4(const uint32_t *q, size_t N, size_t k, size_t c) {
    uint32_t w = q[(k >> 3) * N + c];
    return (w >> (4 * (k & 7))) & 0xF;
}

static inline unsigned idx3(const uint32_t *q, size_t N, size_t k, size_t c) {
    size_t g = k >> 5;           /* group of 32 inputs = 3 words */
    unsigned j = (unsigned)(k & 31);
    const uint32_t *p = q + (3 * g) * N + c;
    uint32_t w0 = p[0], w1 = p[N], w2 = p[2 * N];
    if (j < 10) return (w0 >> (3 * j)) & 7;                       /* :779-788 */
    if (j == 10) return (w0 >> 30) | ((w1 << 2) & 4);            /* :792 */
    if (j < 21) return ((w1 >> 1) >> (3 * (j - 11))) & 7;        /* :793-805 */
    if (j == 21) return ((w1 >> 1) >> 30) | ((w2 << 1) & 6);     /* :809 */
    return ((w2 >> 2) >> (3 * (j - 22))) & 7;                    /* :810-822 */
}

/* idx[k*N + c] = index of input k for output channel c */
void sq_unpack(int bits, const int32_t *qweight, int K, int N, uint8_t *idx) {
    const uint32_t *q = (const uint32_t *)qweight;
#pragma omp parallel for schedule(static)
    for (int k = 0; k < K; ++k)
        for (int c = 0; c < N; ++c)
            idx[(size_t)k * N + c] = (uint8_t)(bits == 4 ? idx4(q, N, k, c) : idx3(q, N, k, c));
}

/* Inverse: restates QuantLinearLUT.pack2's packing loop, squeezellm/quant.py:171-208.
 * idx is [K, N] (already transposed, as `intweight.t()` in :172). */
void sq_pack(int bits, const uint8_t *idx, int K, int N, int32_t *qweight) {
    uint32_t *q = (uint32_t *)qweight;
    size_t rows = (size_t)K / 32 * bits;
    memset(q, 0, rows * N * sizeof(uint32_t));
    if (bits == 4) {
        for (int k = 0; k < K; ++k)
            for (int c = 0; c < N; ++c)
                q[(size_t)(k >> 3) * N + c] |= (uint32_t)idx[(size_t)k * N + c] << (4 * (k & 7));
        return;
    }
    for (int g = 0; g < K / 32; ++g)
        for (int c = 0; c < N; ++c) {
            const uint8_t *v = idx + (size_t)(32 * g) * N + c;
#define V(j) ((uint32_t)v[(size_t)(j) * N])
            uint32_t w0 = 0, w1 = 0, w2 = 0;
            for (int j = 0; j < 10; ++j) w0 |= V(j) << (3 * j);          /* quant.py:186-187 */
            w0 |= V(10) << 30;                                           /* :189 */
            w1 |= (V(10) >> 2) & 1;                                      /* :191 */
            for (int j = 0; j < 10; ++j) w1 |= V(11 + j) << (3 * j + 1); /* :193-194 */
            w1 |= V(21) << 31;                                           /* :196 */
            w2 |= (V(21) >> 1) & 3;                                      /* :198 */
            for (int j = 0; j < 10; ++j) w2 |= V(22 + j) << (3 * j + 2); /* :200-201 */
#undef V
            q[(size_t)(3 * g) * N + c] = w0;
            q[(size_t)(3 * g + 1) * N + c] = w1;
            q[(size_t)(3 * g + 2) * N + c] = w2;
        }
}

/* ---------------------------------------------------------------------------------------------
 * fp64 "truth":  out[b][c] = init[b][c] + sum_k LUT[c][idx(k,c)] * vec[b][k]
 *                           + sum_{i in CSR row c} vals[i] * vec[b][cols[i]]
 *                           + sum_{j: full_row_indices[j]==c} sum_k full_rows[k][j] * vec[b][k]
 * LUT-GEMV  : quant_cuda_kernel.cu:741-828 (w3) / :831-880 (w4), batched :884-1038
 * CSR SpMV  : quant_cuda_kernel.cu:1040-1059, batched :1061-1089  (row = output channel)
 * dense rows: quant_cuda_kernel.cu:1092-1123, batched :1127-1164
 * All of them accumulate into `mul` (atomicAdd at :827,:879,:1057,:1121), so `out` starts from the
 * caller's `mul` contents (zeros or bias, squeezellm/quant.py:214-218).  Any pointer may be NULL
 * to skip that term.
 * ------------------------------------------------------------------------------------------- */
void sq_forward_f64(int bits, int K, int N, int batch,
                    const int32_t *qweight, const float *lut,
                    const int32_t *rows, const int32_t *cols, const float *vals,
                    const float *full_rows, const int32_t *full_row_indices, int topX,
                    const float *vec, const float *mul_init, double *out) {
    const uint32_t *q = (const uint32_t *)qweight;
    const int L = 1 << bits;
#pragma omp parallel for schedule(static)
    for (int c = 0; c < N; ++c) {
        for (int b = 0; b < batch; ++b) {
            const float *x = vec + (size_t)b * K;
            double acc = mul_init ? (double)mul_init[(size_t)b * N + c] : 0.0;
            if (q) {
                const float *t = lut + (size_t)c * L;
                for (int k = 0; k < K; ++k) {
                    unsigned v = bits == 4 ? idx4(q, N, k, c) : idx3(q, N, k, c);
                    acc += (double)t[v] * (double)x[k];
                }
            }
            if (rows)
                for (int i = rows[c]; i < rows[c + 1]; ++i)
                    acc += (double)vals[i] * (double)x[cols[i]];
            out[(size_t)b * N + c] = acc;
        }
    }
    if (full_rows) {
        for (int j = 0; j < topX; ++j) {
            int c = full_row_indices[j];
            for (int b = 0; b < batch; ++b) {
                const float *x = vec + (size_t)b * K;
                double acc = 0.0;
                for (int k = 0; k < K; ++k) acc += (double)full_rows[(size_t)k * topX + j] * (double)x[k];
                out[(size_t)b * N + c] += acc;
            }
        }
    }
}

/* fp32 emulation of the reference's own arithmetic for ONE admissible atomic ordering:
 * each 128-input block produces an fp32 partial in ascending-k order (the `res +=` chains at
 * :779-822 / :866-873), partials are added to mul in ascending block order; the CSR row dot is a
 * sequential fp32 sum (:1053-1056) added after; dense-row 128-blocks likewise (:1114-1121).
 * Used to show how far apart two legal executions of the reference can be. */
void sq_forward_f32_blocked(int bits, int K, int N, int batch,
                            const int32_t *qweight, const float *lut,
                            const int32_t *rows, const int32_t *cols, const float *vals,
                            const float *full_rows, const int32_t *full_row_indices, int topX,
                            const float *vec, float *mul) {
    const uint32_t *q = (const uint32_t *)qweight;
    const int L = 1 << bits;
#pragma omp parallel for schedule(static)
    for (int c = 0; c < N; ++c) {
        for (int b = 0; b < batch; ++b) {
            const float *x = vec + (size_t)b * K;
            float m = mul[(size_t)b * N + c];
            if (q) {
                const float *t = lut + (size_t)c * L;
                for (int k0 = 0; k0 < K; k0 += 128) {
                    float res = 0.f;
                    int k1 = k0 + 128 < K ? k0 + 128 : K;
                    for (int k = k0; k < k1; ++k) {
                        unsigned v = bits == 4 ? idx4(q, N, k, c) : idx3(q, N, k, c);
                        res += t[v] * x[k];
                    }
                    m += res;
                }
            }
            if (rows) {
                float dot = 0.f;
                for (int i = rows[c]; i < rows[c + 1]; ++i) dot += vals[i] * x[cols[i]];
                m += dot;
            }
            mul[(size_t)b * N + c] = m;
        }
    }
    if (full_rows) {
        for (int j = 0; j < topX; ++j) {
            int c = full_row_indices[j];
            for (int b = 0; b < batch; ++b) {
                const float *x = vec + (size_t)b * K;
                for (int k0 = 0; k0 < K; k0 += 128) {
                    float res = 0.f;
                    int k1 = k0 + 128 < K ? k0 + 128 : K;
                    for (int k = k0; k < k1; ++k) res += full_rows[(size_t)k * topX + j] * x[k];
                    mul[(size_t)b * N + c] += res;
                }
            }
        }
    }
}

/* Dequantise to a dense fp32 [K, N] matrix W[k][c] = LUT[c][idx(k,c)] - the first half of
 * BASELINE.json configs[0] ("fp16 dequant + torch.matmul on CPU"); the cast to fp16 and the matmul
 * are done by the caller in torch (oracle/oracle.py: cpu_dequant_matmul). */
void sq_dequant_f32(int bits, const int32_t *qweight, const float *lut, int K, int N, float *W) {
    const uint32_t *q = (const uint32_t *)qweight;
    const int L = 1 << bits;
#pragma omp parallel for schedule(static)
    for (int k = 0; k < K; ++k)
        for (int c = 0; c < N; ++c) {
            unsigned v = bits == 4 ? idx4(q, N, k, c) : idx3(q, N, k, c);
            W[(size_t)k * N + c] = lut[(size_t)c * L + v];
        }
}
