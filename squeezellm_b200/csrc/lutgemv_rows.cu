// lutgemv_rows.cu - the GEMVs of several rows on the CUDA cores: the batched tile kernel and its outlier kernels behind the *_batched
// symbols (lutgemm_batched.cuh), and the multi-row LUT-GEMV with a cluster split-K behind sqllm_lutgemv_rows_dt and the deterministic
// fused mode (lutgemv_rows.cuh), which shares the batched kernel's table layout and decode.
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "host.h"
#include "lutgemv_rows.cuh"

using namespace sqllm;

namespace __attribute__((visibility("hidden"))) sqllm {

// ---- batched symbols: tile kernel + outlier kernels (lutgemm_batched.cuh) ----------------------------------------------
int launch_batched(const sqllm_lutgemv_args *a, cudaStream_t st) {
    using namespace batched;
    const auto kern = a->bits == 4 ? lutgemm_batched_kernel<4> : lutgemm_batched_kernel<3>;
    const int rc = dev_setup({{kern, 227 * 1024}});
    if (rc) return rc;
    const int K = a->in_features, N = a->out_features, B = a->batch;
    const int XU = a->bits == 4 ? 8 : 32, tab = a->bits == 4 ? CB<4>::TAB : CB<3>::TAB;
    PB p;
    p.qw = reinterpret_cast<const uint32_t *>(a->qweight); p.lut = a->lookup_table; p.x = a->vec; p.mul = a->mul;
    p.K = K; p.N = N; p.B = B; p.R = K / XU;
    // K-slabs: the BT x rows of a slab sit in shared memory next to the table and the partial sums; <= 2048 inputs per slab keeps a
    // CTA under 90 KB, i.e. two CTAs (16 warps) per SM
    int slabs = (K + 2047) / 2048;
    p.ks = 2 * ((p.R + 2 * slabs - 1) / (2 * slabs));
    slabs = (p.R + p.ks - 1) / p.ks;
    const int kslab = p.ks * XU;
    const size_t smem = (size_t)2 * tab + (size_t)BT * (kslab * 4 + 16) + (size_t)BW * BT * STRIP * 4;
    if (smem > 227 * 1024) return fail(SQLLM_EINVAL, "batched tile needs %zu B of shared memory", smem);
    const int strips = (N + STRIP - 1) / STRIP, btiles = (B + BT - 1) / BT;
    if (btiles > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", B, 65535 * BT);
    const dim3 grid(strips, slabs, btiles);
    kern<<<grid, BTHREADS, smem, st>>>(p);
    if (a->rows) {
        const dim3 blk(32, 8), g((N + 7) / 8, std::min((B + 31) / 32, 64));
        csr_batched_kernel<<<g, blk, 0, st>>>(a->rows, a->cols, a->vals, a->vec, a->mul, K, N, B);
    }
    if (a->full_rows && a->topX > 0) {
        if (a->topX > 256) return fail(SQLLM_EINVAL, "batched path supports topX <= 256");
        const int per = 256 / a->topX;
        dense_rows_batched_kernel<<<B, per * a->topX, 0, st>>>(a->full_rows, a->full_row_indices, a->topX, a->vec, a->mul, K, N, B);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "batched launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // namespace sqllm

namespace {

// ---- a few rows (lutgemv_rows.cuh): plan + launch ------------------------------------------------------------------------------
// Slabs per strip S (the cluster size) from K, N and the SM count only - never from M, so that a row's result does not depend on
// M: the smallest S in {1, 2, 4, 8} that gives at least two CTAs per SM and a slab of at most SLAB_GOAL inputs, with no more
// slabs than units.  Rows per CTA RB from M: 2, 4 or 8 (a row computes the same bits whatever RB is).
struct RowsPlan { int S, ks, kpad, RB, smem; };
int rows_plan(int bits, int K, int N, int M, int sm, RowsPlan &pl) {
    using namespace rows;
    const int XU = bits == 4 ? 8 : 32, R = K / XU, strips = (N + STRIP - 1) / STRIP;
    int S = 1;
    while (S < MAX_SLABS && 2 * S <= R && ((long long)strips * S < 2LL * sm || (long long)(R + S - 1) / S * XU > SLAB_GOAL)) S *= 2;
    pl.S = S;
    pl.ks = (R + S - 1) / S;
    pl.kpad = (pl.ks + (pl.ks & 1)) * XU;
    pl.RB = M <= 2 ? 2 : M <= 4 ? 4 : 8;
#define RS(B, RBV) SR<B, RBV>::total(pl.kpad)
    pl.smem = bits == 4 ? (pl.RB == 2 ? RS(4, 2) : pl.RB == 4 ? RS(4, 4) : RS(4, 8)) : (pl.RB == 2 ? RS(3, 2) : pl.RB == 4 ? RS(3, 4) : RS(3, 8));
#undef RS
    if (pl.smem > 227 * 1024) return fail(SQLLM_EINVAL, "in_features=%d needs %d B of shared memory per CTA (> 227 KB)", K, pl.smem);
    return SQLLM_OK;
}

typedef void (*KRows)(const rows::PR);
template <typename XT>
KRows krows_lookup_t(int bits, int RB) {
    using namespace rows;
    if (bits == 4) return RB == 2 ? lutgemv_rows_kernel<4, 2, XT> : RB == 4 ? lutgemv_rows_kernel<4, 4, XT> : lutgemv_rows_kernel<4, 8, XT>;
    return RB == 2 ? lutgemv_rows_kernel<3, 2, XT> : RB == 4 ? lutgemv_rows_kernel<3, 4, XT> : lutgemv_rows_kernel<3, 8, XT>;
}
// fp32 x is instantiated at RB = 2 only: it comes from the deterministic fused mode, which runs one row
KRows krows_lookup(int bits, int RB, int x_dt) {
    using namespace rows;
    if (x_dt == SQLLM_DT_F32) return RB != 2 ? nullptr : bits == 4 ? lutgemv_rows_kernel<4, 2, float> : lutgemv_rows_kernel<3, 2, float>;
    return x_dt == SQLLM_DT_BF16 ? krows_lookup_t<__nv_bfloat16>(bits, RB) : krows_lookup_t<__half>(bits, RB);
}

}  // namespace

namespace __attribute__((visibility("hidden"))) sqllm {

int launch_rows(const sqllm_lutgemv_args *a, const void *x, int x_dt, void *y, int y_dt, const float *bias, cudaStream_t st) {
    int sm = 0;
    int rc = dev_setup({}, &sm);
    if (rc) return rc;
    RowsPlan pl;
    if ((rc = rows_plan(a->bits, a->in_features, a->out_features, a->batch, sm, pl))) return rc;
    const KRows kern = krows_lookup(a->bits, pl.RB, x_dt);
    if (!kern) return fail(SQLLM_EINVAL, "fp32 x is taken for one or two rows only (got batch=%d)", a->batch);
    if ((rc = dev_setup({{kern, 227 * 1024}}))) return rc;
    const int groups = (a->batch + pl.RB - 1) / pl.RB;
    if (groups > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", a->batch, 65535 * pl.RB);
    rows::PR p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.x = x; p.y = y; p.y_16 = y_dt != SQLLM_DT_F32; p.bias = bias;
    p.K = a->in_features; p.N = a->out_features; p.M = a->batch; p.R = a->bits == 4 ? p.K / 8 : p.K / 32;
    p.ks = pl.ks; p.kpad = pl.kpad;
    p.qw_al16 = (reinterpret_cast<uintptr_t>(a->qweight) & 15) == 0;
    // the S CTAs of a strip's cluster split its K
    const cudaError_t e = launch_ex(kern, dim3(pl.S, (a->out_features + STRIP - 1) / STRIP, groups), rows::RTHREADS, pl.smem, st,
                                    cluster_of(pl.S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemv_rows launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // namespace sqllm

extern "C" {

int sqllm_lutgemv_rows(const sqllm_lutgemv_args *a, const void *x, void *y, int y_is_half, const float *bias, void *stream) {
    return sqllm_lutgemv_rows_dt(a, x, SQLLM_DT_F16, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias, stream);
}

int sqllm_lutgemv_rows_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias, void *stream) {
    int rc = check_layer(a, 32, 4);
    if (rc) return rc;
    if ((x_dtype != SQLLM_DT_F16 && x_dtype != SQLLM_DT_BF16) || (y_dtype != SQLLM_DT_F32 && y_dtype != x_dtype))
        return fail(SQLLM_EINVAL, "x_dtype=%d, y_dtype=%d: x must be SQLLM_DT_F16 or SQLLM_DT_BF16, y SQLLM_DT_F32 or x's dtype", x_dtype, y_dtype);
    if (a->in_features > SQLLM_ROWS_MAX_IN) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d: the slab of x a CTA stages would not fit its shared memory", a->in_features, SQLLM_ROWS_MAX_IN);
    if ((a->out_features + STRIP - 1) / STRIP > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * STRIP);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x) must be >= 1 (got %d)", a->batch);
    if (!x || !y) return fail(SQLLM_EINVAL, "x / y must not be null");
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3) || (reinterpret_cast<uintptr_t>(bias) & 3))
        return fail(SQLLM_EINVAL, "qweight, lookup_table and bias must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(y) & 15) return fail(SQLLM_EINVAL, "y must be 16-byte aligned");
    return launch_rows(a, x, x_dtype, y, y_dtype, bias, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
