// lutgemm_tc.cu - the tensor-core LUT-GEMM of prefill-sized batches (lutgemm_tc.cuh) behind sqllm_lutgemm_fused, _dt and _f32.
#include <stdint.h>

#include "host.h"
#include "lutgemm_tc.cuh"

using namespace sqllm;

extern "C" {

int sqllm_lutgemm_fused(const sqllm_lutgemv_args *a, const void *x, void *y, int y_is_half, const float *bias, void *stream) {
    return sqllm_lutgemm_fused_dt(a, x, SQLLM_DT_F16, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias, stream);
}

// sqllm_lutgemm_fused_dt (f32 = false) and sqllm_lutgemm_fused_f32 (f32 = true: x and y fp32, the dtype codes are not looked at):
// the argument checks, in this order and all before any device access, then the launch
static int lutgemm_tc_launch(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                             void *stream, bool f32) {
    int rc = check_layer(a, 32, 1);
    if (rc) return rc;
    if ((a->out_features + tc::BN - 1) / tc::BN > 65535) return fail(SQLLM_EINVAL, "out_features=%d exceeds %d", a->out_features, 65535 * tc::BN);
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch (rows of x) must be >= 1 (got %d)", a->batch);
    if (!x || !y) return fail(SQLLM_EINVAL, "x / y must not be null");
    if (!f32) {
        if (x_dtype != SQLLM_DT_F16 && x_dtype != SQLLM_DT_BF16) return fail(SQLLM_EINVAL, "x_dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", x_dtype);
        if (y_dtype != SQLLM_DT_F32 && y_dtype != x_dtype) return fail(SQLLM_EINVAL, "y_dtype=%d must be SQLLM_DT_F32 or x's dtype (%d)", y_dtype, x_dtype);
    }
    if ((reinterpret_cast<uintptr_t>(a->qweight) & 3) || (reinterpret_cast<uintptr_t>(a->lookup_table) & 3) || (reinterpret_cast<uintptr_t>(bias) & 3))
        return fail(SQLLM_EINVAL, "qweight, lookup_table and bias must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(y) & 15) return fail(SQLLM_EINVAL, "y must be 16-byte aligned");
    if (f32) { x_dtype = SQLLM_DT_F32; y_dtype = SQLLM_DT_F32; }
    const bool bf = x_dtype == SQLLM_DT_BF16;
    const auto kern = f32 ? (a->bits == 4 ? tc::lutgemm_tc_kernel<4, true, true> : tc::lutgemm_tc_kernel<3, true, true>)
                    : a->bits == 4 ? (bf ? tc::lutgemm_tc_kernel<4, true> : tc::lutgemm_tc_kernel<4, false>)
                                   : (bf ? tc::lutgemm_tc_kernel<3, true> : tc::lutgemm_tc_kernel<3, false>);
    const int smem = f32 ? tc::L<3, 3>::SMEM : bf ? tc::L<3>::SMEM : tc::L<2>::SMEM;
    if ((rc = dev_setup({{kern, smem}}))) return rc;
    tc::PT p;
    set_layer(p, *a);
    p.x = static_cast<const unsigned short *>(x); p.y = y; p.y_16 = y_dtype != SQLLM_DT_F32; p.bias = bias;
    p.M = a->batch; p.K = a->in_features; p.N = a->out_features;
    const dim3 grid((a->batch + tc::BM - 1) / tc::BM, (a->out_features + tc::BN - 1) / tc::BN);
    kern<<<grid, tc::THREADS, smem, static_cast<cudaStream_t>(stream)>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "lutgemm_fused launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

int sqllm_lutgemm_fused_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *stream) {
    return lutgemm_tc_launch(a, x, x_dtype, y, y_dtype, bias, stream, false);
}

int sqllm_lutgemm_fused_f32(const sqllm_lutgemv_args *a, const float *x, float *y, const float *bias, void *stream) {
    return lutgemm_tc_launch(a, x, SQLLM_DT_F32, y, SQLLM_DT_F32, bias, stream, true);
}

}  // extern "C"
