// tools.cu - the quantizer's and the checkpoint's kernels: the dense weight of a layer (dequant.cuh) behind sqllm_dequantize, the
// weighted 1-D k-means and the GPU pack (kmeans1d.cuh) behind sqllm_kmeans1d and sqllm_pack_indices, and the unpack test hook.
#include <cub/device/device_segmented_radix_sort.cuh>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "dequant.cuh"
#include "host.h"
#include "kmeans1d.cuh"

using namespace sqllm;

namespace {

// test hook: unpack exactly like the GEMV path (same shift/mask expressions)
__global__ void unpack_kernel(int bits, const uint32_t *__restrict__ q, int K, int N, uint8_t *__restrict__ idx) {
    const size_t n = (size_t)K * N;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(e / N), c = (int)(e % N);
        uint32_t v;
        if (bits == 4) {
            const uint32_t w = q[(size_t)(k >> 3) * N + c];
            const int n8 = k & 7;
            const uint32_t EO = (n8 & 1) ? ((w >> 4) & 0x0F0F0F0Fu) : (w & 0x0F0F0F0Fu);
            v = __byte_perm(EO, 0u, 0x4440 | (n8 >> 1)) & 0xFFu;
        } else {
            const int g = k >> 5, j = k & 31;
            const uint32_t *pq = q + (size_t)(3 * g) * N + c;
            const uint32_t w0 = pq[0], w1 = pq[N], w2 = pq[2 * (size_t)N];
            uint32_t f;  // field moved to bits 8..10, as in consume3_col
            if (j < 10) f = (3 * j < 8) ? (w0 << (8 - 3 * j)) : (w0 >> (3 * j - 8));
            else if (j == 10) f = __funnelshift_r(w0, w1, 22);
            else if (j < 21) { const int s = 1 + 3 * (j - 11); f = (s < 8) ? (w1 << (8 - s)) : (w1 >> (s - 8)); }
            else if (j == 21) f = __funnelshift_r(w1, w2, 23);
            else { const int s = 2 + 3 * (j - 22); f = (s < 8) ? (w2 << (8 - s)) : (w2 >> (s - 8)); }
            v = (f & 0x700u) >> 8;
        }
        idx[e] = (uint8_t)v;
    }
}

}  // namespace

extern "C" {

int sqllm_dequantize(const sqllm_lutgemv_args *a, int col0, int ncols, void *w, int w_dtype, void *stream) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->in_features + dq::BK - 1) / dq::BK > 65535) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d", a->in_features, 65535 * dq::BK);
    if (col0 < 0 || ncols < 1 || col0 > a->out_features - ncols)
        return fail(SQLLM_EINVAL, "column range col0=%d, ncols=%d must be non-empty and lie in [0, out_features=%d)", col0, ncols, a->out_features);
    if (!w) return fail(SQLLM_EINVAL, "w must not be null");
    if (!dt_valid(w_dtype)) return fail(SQLLM_EINVAL, "w_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", w_dtype);
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3))
        return fail(SQLLM_EINVAL, "qweight and lookup_table must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(w) & 15) return fail(SQLLM_EINVAL, "w must be 16-byte aligned");
    void (*kern)(const dq::PD);
    if (w_dtype == SQLLM_DT_F32) kern = a->bits == 4 ? dq::dequant_kernel<4, float> : dq::dequant_kernel<3, float>;
    else if (w_dtype == SQLLM_DT_F16) kern = a->bits == 4 ? dq::dequant_kernel<4, __half> : dq::dequant_kernel<3, __half>;
    else kern = a->bits == 4 ? dq::dequant_kernel<4, __nv_bfloat16> : dq::dequant_kernel<3, __nv_bfloat16>;
    if ((rc = dev_setup({{kern, dq::SMEM}}))) return rc;
    dq::PD p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.K = a->in_features; p.N = a->out_features; p.c0 = col0; p.n = ncols; p.w = w;
    const dim3 grid((ncols + dq::BN - 1) / dq::BN, (a->in_features + dq::BK - 1) / dq::BK);
    kern<<<grid, dq::THREADS, dq::SMEM, static_cast<cudaStream_t>(stream)>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "dequantize launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_unpack_indices(int bits, const int32_t *qweight, int in_features, int out_features, uint8_t *idx, void *stream) {
    if ((bits != 3 && bits != 4) || !qweight || !idx || in_features % 32 || in_features <= 0 || out_features <= 0)
        return fail(SQLLM_EINVAL, "bad arguments to sqllm_unpack_indices");
    unpack_kernel<<<1024, 256, 0, static_cast<cudaStream_t>(stream)>>>(bits, reinterpret_cast<const uint32_t *>(qweight),
                                                                       in_features, out_features, idx);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "unpack launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

// ---- weighted 1-D k-means and the GPU pack (kmeans1d.cuh) ----------------------------------------------------------------
namespace {
constexpr size_t KM_BUDGET = (size_t)512 << 20;  // workspace rows are chunked to about this many bytes

size_t km_align(size_t b) { return (b + 255) & ~(size_t)255; }

size_t km_row_bytes(int n, int k) {
    const size_t n1 = (size_t)n + 1;
    return 2 * sizeof(float) * n + (3 + 2) * sizeof(double) * n1 + (size_t)(k - 1) * sizeof(uint16_t) * n1;
}

int km_chunk(int rows, int n, int k) { return (int)std::max<size_t>(1, std::min<size_t>(rows, KM_BUDGET / km_row_bytes(n, k))); }

struct KmLayout {
    size_t offs, keys, vals, pref, d, opt, temp, temp_bytes, total;
};

int km_check(int rows, int n, int k) {
    if (rows < 1) return fail(SQLLM_EINVAL, "kmeans1d: rows=%d must be >= 1", rows);
    if (k < 2 || k > km::MAX_K) return fail(SQLLM_EINVAL, "kmeans1d: k=%d must be in [2, %d]", k, km::MAX_K);
    if (n < k || n > km::MAX_N) return fail(SQLLM_EINVAL, "kmeans1d: n=%d must be in [k=%d, %d]", n, k, km::MAX_N);
    return SQLLM_OK;
}

int km_layout(int rows, int n, int k, KmLayout &L) {
    const int C = km_chunk(rows, n, k);
    const size_t n1 = (size_t)n + 1, items = (size_t)C * n;
    size_t temp = 0;
    const cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(nullptr, temp, (const float *)nullptr, (float *)nullptr,
                                                                   (const float *)nullptr, (float *)nullptr, (int)items, C,
                                                                   (const int *)nullptr, (const int *)nullptr);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d: sort workspace query failed: %s", cudaGetErrorString(e));
    size_t o = 0;
    L.offs = o; o += km_align(sizeof(int) * (C + 1));
    L.keys = o; o += km_align(sizeof(float) * items);
    L.vals = o; o += km_align(sizeof(float) * items);
    L.pref = o; o += km_align(3 * sizeof(double) * n1 * C);
    L.d = o; o += km_align(2 * sizeof(double) * n1 * C);
    L.opt = o; o += km_align((size_t)(k - 1) * sizeof(uint16_t) * n1 * C);
    L.temp = o; L.temp_bytes = temp; o += km_align(temp);
    L.total = o;
    return SQLLM_OK;
}
}  // namespace

int sqllm_kmeans1d_workspace_bytes(int rows, int n, int k, size_t *bytes) {
    if (!bytes) return fail(SQLLM_EINVAL, "kmeans1d_workspace_bytes: bytes must not be null");
    int rc = km_check(rows, n, k);
    if (rc) return rc;
    KmLayout L;
    if ((rc = km_layout(rows, n, k, L))) return rc;
    *bytes = L.total;
    return SQLLM_OK;
}

int sqllm_kmeans1d(const float *w, const float *s, int rows, int n, int k, float *centroids, uint8_t *labels, void *workspace,
                   size_t workspace_bytes, void *stream) {
    int rc = km_check(rows, n, k);
    if (rc) return rc;
    if (!w || !s || !centroids || !labels) return fail(SQLLM_EINVAL, "kmeans1d: w / s / centroids / labels must not be null");
    if (((uintptr_t)w | (uintptr_t)s | (uintptr_t)centroids) & 3) return fail(SQLLM_EINVAL, "kmeans1d: w / s / centroids must be 4-byte aligned");
    if (!workspace) return fail(SQLLM_EWORKSPACE, "kmeans1d: workspace must not be null");
    if ((uintptr_t)workspace & 255) return fail(SQLLM_EINVAL, "kmeans1d: workspace must be 256-byte aligned");
    KmLayout L;
    if ((rc = km_layout(rows, n, k, L))) return rc;
    if (workspace_bytes < L.total)
        return fail(SQLLM_EWORKSPACE, "kmeans1d: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    char *ws = static_cast<char *>(workspace);
    int *offs = reinterpret_cast<int *>(ws + L.offs);
    float *keys = reinterpret_cast<float *>(ws + L.keys), *vals = reinterpret_cast<float *>(ws + L.vals);
    const int C = km_chunk(rows, n, k);
    km::segment_offsets_kernel<<<(C + 256) / 256, 256, 0, st>>>(offs, C, n);
    for (int r0 = 0; r0 < rows; r0 += C) {
        const int c = std::min(C, rows - r0);
        const size_t at = (size_t)r0 * n;
        size_t temp = L.temp_bytes;
        cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairs(ws + L.temp, temp, w + at, keys, s + at, vals, c * n, c, offs,
                                                                 offs + 1, 0, 32, st);
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d: segmented sort failed: %s", cudaGetErrorString(e));
        km::kmeans1d_kernel<<<c, km::THREADS, 0, st>>>(keys, vals, w + at, n, k, reinterpret_cast<double *>(ws + L.pref),
                                                       reinterpret_cast<double *>(ws + L.d), reinterpret_cast<uint16_t *>(ws + L.opt),
                                                       centroids + (size_t)r0 * k, labels + at);
        e = cudaGetLastError();
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kmeans1d launch failed: %s", cudaGetErrorString(e));
    }
    return SQLLM_OK;
}

int sqllm_pack_indices(int bits, const uint8_t *labels, int in_features, int out_features, int32_t *qweight, void *stream) {
    if (bits != 3 && bits != 4) return fail(SQLLM_EINVAL, "pack_indices: bits=%d must be 3 or 4", bits);
    if (in_features <= 0 || in_features % 32)
        return fail(SQLLM_EINVAL, "pack_indices: in_features=%d must be a positive multiple of 32", in_features);
    if (out_features <= 0) return fail(SQLLM_EINVAL, "pack_indices: out_features=%d must be >= 1", out_features);
    if (!labels || !qweight) return fail(SQLLM_EINVAL, "pack_indices: labels / qweight must not be null");
    if ((uintptr_t)qweight & 3) return fail(SQLLM_EINVAL, "pack_indices: qweight must be 4-byte aligned");
    const size_t work = (size_t)in_features / 32 * out_features;
    const int grid = (int)std::min<size_t>(4096, (work + 255) / 256);
    km::pack_indices_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(bits, labels, in_features, out_features,
                                                                                 reinterpret_cast<uint32_t *>(qweight));
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "pack_indices launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // extern "C"
