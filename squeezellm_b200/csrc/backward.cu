// backward.cu - the gradients of QuantLinearLUT and the Fisher information: the input gradient dx = dy . W^T on the tensor cores
// (lutgemm_tc_t.cuh) or the CUDA cores (lutgemm_t.cuh) behind sqllm_lutgemm_t, the gradients of the codebook, the CSR values and the
// dense rows on the tensor cores (lut_grad_tc.cuh) or the CUDA cores (lut_grad.cuh) behind sqllm_lut_grad, and the diagonal of the
// empirical Fisher information (fisher.cuh) behind sqllm_fisher_accumulate.
#include <stdint.h>
#include <string.h>

#include "fisher.cuh"
#include "host.h"
#include "lut_grad.cuh"
#include "lut_grad_tc.cuh"
#include "lutgemm_t.cuh"
#include "lutgemm_tc_t.cuh"

using namespace sqllm;

namespace {

// ---- input gradient (lutgemm_t.cuh): plan + launch --------------------------------------------------------------------------
// Strip splits S (the cluster size) from K, N and the SM count only - never from M, so that a row's result does not depend on M:
// the smallest S in {1, 2, 4, 8} that gives at least two CTAs per SM, with at least two strips per CTA.  Rows per CTA RB from M:
// 1, 2, 4 or 8 (a row computes the same bits whatever RB is).
struct TPlan { int S, RB, smem; };
void t_plan(int K, int N, int M, int sm, TPlan &pl) {
    using namespace bwd;
    const int slabs = (K + KS - 1) / KS, strips = (N + STRIP - 1) / STRIP;
    int S = 1;
    while (S < MAX_SPLIT && 4 * S <= strips && (long long)slabs * S < 2LL * sm) S *= 2;
    pl.S = S;
    pl.RB = M <= 1 ? 1 : M <= 2 ? 2 : M <= 4 ? 4 : 8;
    pl.smem = pl.RB == 1 ? ST<1>::TOTAL : pl.RB == 2 ? ST<2>::TOTAL : pl.RB == 4 ? ST<4>::TOTAL : ST<8>::TOTAL;
}

typedef void (*KT)(const bwd::PT);
KT kt_lookup(int bits, int RB) {
    using namespace bwd;
    if (bits == 4) return RB == 1 ? lutgemm_t_kernel<4, 1> : RB == 2 ? lutgemm_t_kernel<4, 2> : RB == 4 ? lutgemm_t_kernel<4, 4> : lutgemm_t_kernel<4, 8>;
    return RB == 1 ? lutgemm_t_kernel<3, 1> : RB == 2 ? lutgemm_t_kernel<3, 2> : RB == 4 ? lutgemm_t_kernel<3, 4> : lutgemm_t_kernel<3, 8>;
}

// ---- codebook gradient (lut_grad.cuh, lut_grad_tc.cuh): plan -------------------------------------------------------------
// K splits S (the cluster size) from K, N and the SM count only: the smallest S in {1, 2, 4, 8} that gives at least one CTA per
// SM, with at least two k-tiles per CTA.
int lg_split(int K, int N, int sm) {
    using namespace lg;
    const int ktiles = (K + TK - 1) / TK, ctiles = (N + TC - 1) / TC;
    int S = 1;
    while (S < MAX_SPLIT && 4 * S <= ktiles && (long long)ctiles * S < sm) S *= 2;
    return S;
}

}  // namespace

extern "C" {

int sqllm_lutgemm_t(const sqllm_lutgemv_args *a, const void *dy, int dy_dtype, void *dx, int dx_dtype, int path, void *stream) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->in_features + bwd::KS - 1) / bwd::KS > 65535) return fail(SQLLM_EINVAL, "in_features=%d exceeds %d", a->in_features, 65535 * bwd::KS);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of dy) must be >= 1 (got %d)", a->batch);
    if (!dy || !dx) return fail(SQLLM_EINVAL, "dy / dx must not be null");
    if (!dt_valid(dy_dtype)) return fail(SQLLM_EINVAL, "dy_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", dy_dtype);
    if (dx_dtype != SQLLM_DT_F32 && dx_dtype != dy_dtype) return fail(SQLLM_EINVAL, "dx_dtype=%d must be SQLLM_DT_F32 or dy's dtype (%d)", dx_dtype, dy_dtype);
    if (path < 0 || path > 2) return fail(SQLLM_EINVAL, "path=%d must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)", path);
    if (path == 1 && dy_dtype == SQLLM_DT_F32) return fail(SQLLM_EINVAL, "path=1 (tensor cores) takes fp16 or bf16 dy, not fp32");
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3))
        return fail(SQLLM_EINVAL, "qweight and lookup_table must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(dy) & (dy_dtype == SQLLM_DT_F32 ? 3 : 1)) return fail(SQLLM_EINVAL, "dy must be aligned to its element size");
    if (reinterpret_cast<uintptr_t>(dx) & 15) return fail(SQLLM_EINVAL, "dx must be 16-byte aligned");
    if (path == 0) path = dy_dtype != SQLLM_DT_F32 && a->batch >= SQLLM_BWD_TC_MIN_ROWS ? 1 : 2;
    if (path == 1) {
        const bool bf = dy_dtype == SQLLM_DT_BF16;
        const auto kern = a->bits == 4 ? (bf ? tct::lutgemm_tc_t_kernel<4, true> : tct::lutgemm_tc_t_kernel<4, false>)
                                       : (bf ? tct::lutgemm_tc_t_kernel<3, true> : tct::lutgemm_tc_t_kernel<3, false>);
        const int smem = bf ? tct::L<3>::SMEM : tct::L<2>::SMEM;
        if ((rc = dev_setup({{kern, smem}}))) return rc;
        tct::PT p;
        memset(&p, 0, sizeof(p));
        set_layer(p, *a);
        p.dy = dy; p.dx = dx; p.dx_dt = dx_dtype;
        p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
        p.dy_al16 = (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && a->out_features % 8 == 0;
        const dim3 grid((a->batch + tc::BM - 1) / tc::BM, (a->in_features + tct::BK - 1) / tct::BK);
        kern<<<grid, tct::THREADS, smem, static_cast<cudaStream_t>(stream)>>>(p);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_t (tensor cores) launch failed: %s", cudaGetErrorString(e));
        return SQLLM_OK;
    }
    int sm = 0;
    if ((rc = dev_setup({}, &sm))) return rc;
    TPlan pl;
    t_plan(a->in_features, a->out_features, a->batch, sm, pl);
    const KT kern = kt_lookup(a->bits, pl.RB);
    if ((rc = dev_setup({{kern, pl.smem}}))) return rc;
    const int groups = (a->batch + pl.RB - 1) / pl.RB;
    if (groups > 65535) return fail(SQLLM_EINVAL, "batch=%d is too large for one call (max %d)", a->batch, 65535 * pl.RB);
    bwd::PT p;
    memset(&p, 0, sizeof(p));
    set_layer(p, *a);
    p.dy = dy; p.dx = dx; p.dy_dt = dy_dtype; p.dx_dt = dx_dtype;
    p.K = a->in_features; p.N = a->out_features; p.M = a->batch;
    p.strips = (a->out_features + STRIP - 1) / STRIP;
    p.qw_al16 = (reinterpret_cast<uintptr_t>(a->qweight) & 15) == 0 && a->out_features % 4 == 0;
    const cudaError_t e = launch_ex(kern, dim3(pl.S, (a->in_features + bwd::KS - 1) / bwd::KS, groups), bwd::TTHREADS, pl.smem,
                                    static_cast<cudaStream_t>(stream), cluster_of(pl.S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_t launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_lut_grad(const sqllm_lutgemv_args *a, const void *x, int x_dtype, const void *dy, int dy_dtype, float *dlut, float *dvals,
                   float *dfull_rows, int path, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    if (a->bits != 3 && a->bits != 4) return fail(SQLLM_EINVAL, "bits must be 3 or 4 (got %d)", a->bits);
    if (a->in_features <= 0 || a->in_features % 32) return fail(SQLLM_EINVAL, "in_features=%d must be a positive multiple of 32", a->in_features);
    if (a->out_features <= 0) return fail(SQLLM_EINVAL, "out_features=%d must be positive", a->out_features);
    if ((a->out_features + lg::TC - 1) / lg::TC > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * lg::TC);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x and dy) must be >= 1 (got %d)", a->batch);
    if (!a->qweight) return fail(SQLLM_EINVAL, "qweight must not be null");
    if (!x || !dy) return fail(SQLLM_EINVAL, "x / dy must not be null");
    if (!dt_valid(x_dtype)) return fail(SQLLM_EINVAL, "x_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", x_dtype);
    if (!dt_valid(dy_dtype)) return fail(SQLLM_EINVAL, "dy_dtype=%d is not SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16", dy_dtype);
    if (path < 0 || path > 2) return fail(SQLLM_EINVAL, "path=%d must be 0 (auto), 1 (tensor cores) or 2 (CUDA cores)", path);
    const bool tc_dtypes = x_dtype == dy_dtype && x_dtype != SQLLM_DT_F32;
    if (path == 1 && !tc_dtypes)
        return fail(SQLLM_EINVAL, "path=1 (tensor cores) takes x and dy both fp16 or both bf16 (got x_dtype=%d, dy_dtype=%d)", x_dtype, dy_dtype);
    if (!dlut && !dvals && !dfull_rows) return fail(SQLLM_EINVAL, "no output requested: dlut, dvals and dfull_rows are all null");
    if (dvals && (!a->rows || !a->cols)) return fail(SQLLM_EINVAL, "dvals needs the CSR arrays (rows, cols)");
    if (a->topX < 0) return fail(SQLLM_EINVAL, "topX < 0");
    if (dfull_rows && (!a->full_row_indices || a->topX < 1)) return fail(SQLLM_EINVAL, "dfull_rows needs the dense rows (full_row_indices, topX >= 1)");
    if (reinterpret_cast<uintptr_t>(a->qweight) & 3) return fail(SQLLM_EINVAL, "qweight must be 4-byte aligned");
    if ((reinterpret_cast<uintptr_t>(x) & (x_dtype == SQLLM_DT_F32 ? 3 : 1)) || (reinterpret_cast<uintptr_t>(dy) & (dy_dtype == SQLLM_DT_F32 ? 3 : 1)))
        return fail(SQLLM_EINVAL, "x and dy must be aligned to their element size");
    if ((reinterpret_cast<uintptr_t>(dlut) & 3) || (reinterpret_cast<uintptr_t>(dvals) & 3) || (reinterpret_cast<uintptr_t>(dfull_rows) & 3))
        return fail(SQLLM_EINVAL, "dlut, dvals and dfull_rows must be 4-byte aligned");
    if (path == 0) path = tc_dtypes && a->batch >= SQLLM_LUT_GRAD_TC_MIN_ROWS ? 1 : 2;

    lg::PG p;
    memset(&p, 0, sizeof(p));
    p.qw = reinterpret_cast<const uint32_t *>(a->qweight);
    p.x = x; p.dy = dy; p.x_dt = x_dtype; p.dy_dt = dy_dtype;
    p.rows = dvals ? a->rows : nullptr; p.cols = dvals ? a->cols : nullptr;
    p.fri = dfull_rows ? a->full_row_indices : nullptr; p.topX = dfull_rows ? a->topX : 0;
    p.dlut = dlut; p.dvals = dvals; p.dfull = dfull_rows;
    p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
    p.ktiles = (a->in_features + lg::TK - 1) / lg::TK;
    p.x_al16 = (reinterpret_cast<uintptr_t>(x) & 15) == 0;  // in_features % 32 == 0: every row is then 16-byte aligned
    p.dy_al16 = (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && a->out_features % 8 == 0;
    const bool bf = dy_dtype == SQLLM_DT_BF16;
    void (*kern)(const lg::PG);
    int smem;
    if (path == 1) {
        kern = bf ? (a->bits == 4 ? lgt::lut_grad_tc_kernel<4, true> : lgt::lut_grad_tc_kernel<3, true>)
                  : (a->bits == 4 ? lgt::lut_grad_tc_kernel<4, false> : lgt::lut_grad_tc_kernel<3, false>);
        smem = lgt::SMEM;
    } else {
        kern = a->bits == 4 ? lg::lut_grad_kernel<4> : lg::lut_grad_kernel<3>;
        smem = lg::SMEM;
    }
    int sm = 0;
    const int rc = dev_setup({{kern, smem}}, &sm);
    if (rc) return rc;
    const int S = lg_split(a->in_features, a->out_features, sm);
    const cudaError_t e = launch_ex(kern, dim3(S, (a->out_features + lg::TC - 1) / lg::TC), lg::THREADS, smem,
                                    static_cast<cudaStream_t>(stream), cluster_of(S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lut_grad launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_fisher_accumulate(const void *x, const void *dy, int dtype, int rows, int seq_len, int in_features, int out_features,
                            float *fisher, void *stream) {
    if (dtype != SQLLM_DT_F16 && dtype != SQLLM_DT_BF16)
        return fail(SQLLM_EINVAL, "fisher_accumulate: dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", dtype);
    if (rows < 1) return fail(SQLLM_EINVAL, "fisher_accumulate: rows=%d must be >= 1", rows);
    if (seq_len < 1) return fail(SQLLM_EINVAL, "fisher_accumulate: seq_len=%d must be >= 1", seq_len);
    if (rows % seq_len) return fail(SQLLM_EINVAL, "fisher_accumulate: rows=%d must be a multiple of seq_len=%d", rows, seq_len);
    if (in_features < 1 || in_features % 8)
        return fail(SQLLM_EINVAL, "fisher_accumulate: in_features=%d must be a positive multiple of 8", in_features);
    if (out_features < 1 || out_features % 8)
        return fail(SQLLM_EINVAL, "fisher_accumulate: out_features=%d must be a positive multiple of 8", out_features);
    if ((out_features + fis::TN - 1) / fis::TN > 65535)
        return fail(SQLLM_EINVAL, "fisher_accumulate: out_features=%d exceeds %d", out_features, 65535 * fis::TN);
    if (!x || !dy || !fisher) return fail(SQLLM_EINVAL, "fisher_accumulate: x / dy / fisher must not be null");
    if (((uintptr_t)x | (uintptr_t)dy | (uintptr_t)fisher) & 15)
        return fail(SQLLM_EINVAL, "fisher_accumulate: x / dy / fisher must be 16-byte aligned");
    void (*kern)(const fis::PF) = dtype == SQLLM_DT_BF16 ? fis::fisher_kernel<true> : fis::fisher_kernel<false>;
    const int rc = dev_setup({{kern, fis::SMEM}});
    if (rc) return rc;
    fis::PF p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.dy = dy; p.f = fisher;
    p.rows = rows; p.T = seq_len; p.K = in_features; p.N = out_features;
    const dim3 grid((in_features + fis::TK - 1) / fis::TK, (out_features + fis::TN - 1) / fis::TN);
    // a cluster of one, not PDL: the kernel does not wait on the grid dependency, it reads x, dy and F as the previous kernel left them
    const cudaError_t e = launch_ex(kern, grid, fis::THREADS, fis::SMEM, static_cast<cudaStream_t>(stream), cluster_of(1), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "fisher_accumulate launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // extern "C"
