// host.cu - the process-wide state of the library, defined once, and the C entry points that only read or set it: the last error,
// the mode switches, the device's SM count and the debug hooks.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <unordered_map>

#include "common.cuh"
#include "host.h"

namespace __attribute__((visibility("hidden"))) sqllm {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

std::recursive_mutex g_state_mu;

DevInfo g_dev[64];

bool dt_valid(int dt) { return dt == SQLLM_DT_F32 || dt == SQLLM_DT_F16 || dt == SQLLM_DT_BF16; }

// The descriptor checks every GEMV / GEMM entry point shares, in this order: in_features a positive multiple of k_mult (64 or 32),
// out_features a positive multiple of n_mult (4, or 1 for "positive"), the packed matrix and codebook given, and dense rows only with
// their indices.  Each entry point makes its own checks after these.
int check_layer(const sqllm_lutgemv_args *a, int k_mult, int n_mult) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    if (a->bits != 3 && a->bits != 4) return fail(SQLLM_EINVAL, "bits must be 3 or 4 (got %d)", a->bits);
    if (a->in_features <= 0 || a->in_features % k_mult)
        return fail(SQLLM_EINVAL, "in_features=%d must be a positive multiple of %d", a->in_features, k_mult);
    if (a->out_features <= 0 || a->out_features % n_mult) {
        if (n_mult == 1) return fail(SQLLM_EINVAL, "out_features=%d must be positive", a->out_features);
        return fail(SQLLM_EINVAL, "out_features=%d must be a positive multiple of %d", a->out_features, n_mult);
    }
    if (!a->qweight || !a->lookup_table) return fail(SQLLM_EINVAL, "qweight / lookup_table must not be null");
    if (a->topX < 0) return fail(SQLLM_EINVAL, "topX < 0");
    if (a->full_rows && a->topX > 0 && !a->full_row_indices) return fail(SQLLM_EINVAL, "full_rows given without full_row_indices");
    return SQLLM_OK;
}

int g_det = -1;
int det_mode() {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    if (g_det < 0) { const char *e = getenv("SQLLM_DETERMINISTIC"); g_det = (e && e[0] == '1') ? 1 : 0; }
    return g_det;
}
// g_det - fused mode: 1 = v1, deterministic per-strip tickets (SQLLM_DETERMINISTIC=1 or sqllm_set_deterministic), 0 = v2 (default)
int g_last_grid = 0;
unsigned long long *g_trace = nullptr;
size_t g_trace_stride = 0;

// ---- 2-D tensor maps for the packed matrix (one per (pointer, shape, box)), created through the driver entry point ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct TmKey {
    const void *ptr; int rows, cols, box_rows;
    bool operator==(const TmKey &o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box_rows == o.box_rows; }
};
struct TmHash {
    size_t operator()(const TmKey &k) const {
        return std::hash<const void *>()(k.ptr) ^ ((size_t)k.rows * 1000003u) ^ ((size_t)k.cols * 10007u) ^ (size_t)k.box_rows;
    }
};
std::mutex g_tm_mutex;
std::unordered_map<TmKey, CUtensorMap, TmHash> g_tm_cache;
EncodeTiledFn g_encode = nullptr;

int get_tensor_map(const void *qweight, int rows, int cols, int box_rows, CUtensorMap &out) {
    std::lock_guard<std::mutex> lock(g_tm_mutex);
    const TmKey key{qweight, rows, cols, box_rows};
    auto it = g_tm_cache.find(key);
    if (it != g_tm_cache.end()) { out = it->second; return SQLLM_OK; }
    if (!g_encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
            return fail(SQLLM_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
        g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    }
    const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)cols * 4};
    const cuuint32_t box[2] = {(cuuint32_t)STRIP, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    const CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<void *>(qweight), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(SQLLM_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    if (g_tm_cache.size() > 8192) g_tm_cache.clear();
    g_tm_cache.emplace(key, m);
    out = m;
    return SQLLM_OK;
}

// the descriptor checks of sqllm_lutgemv, the fused one-GEMV entry points and the sequence: the shared ones with in_features a
// multiple of 64 and out_features a multiple of 4, then a 16-byte aligned matrix and codebook
int check_common(const sqllm_lutgemv_args *a) {
    const int rc = check_layer(a, 64, 4);
    if (rc) return rc;
    if (reinterpret_cast<uintptr_t>(a->qweight) & 15) return fail(SQLLM_EINVAL, "qweight must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(a->lookup_table) & 15) return fail(SQLLM_EINVAL, "lookup_table must be 16-byte aligned");
    return SQLLM_OK;
}

int g_lut_mode = -1;     // 0: exact fp32 table, 1: fp16 pair table when x is fp16 (SQLLM_LUT_MODE=fp16 / sqllm_set_lut_mode)

int lut_mode() {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    if (g_lut_mode < 0) {
        const char *e = getenv("SQLLM_LUT_MODE");
        g_lut_mode = (e && (!strcmp(e, "fp16") || !strcmp(e, "pair") || !strcmp(e, "1"))) ? 1 : 0;
    }
    return g_lut_mode;
}

}  // namespace sqllm

using namespace sqllm;

extern "C" {

int sqllm_abi_version(void) { return SQLLM_ABI_VERSION; }
void sqllm_set_deterministic(int on) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    g_det = on ? 1 : 0;
}
void sqllm_set_lut_mode(int mode) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    g_lut_mode = mode == SQLLM_LUT_FP16_PAIR ? 1 : 0;
}
int sqllm_get_lut_mode(void) { return lut_mode(); }

// debug hook (not in the public header): successive launches write their timeline at buf, buf+stride, ...
void sqllm_debug_set_trace(unsigned long long *buf, size_t stride_words) { g_trace = buf; g_trace_stride = stride_words; }
int sqllm_debug_last_grid(void) { return g_last_grid; }
const char *sqllm_last_error(void) { return g_err; }

int sqllm_device_sm_count(void) {
    int sm = 0;
    return dev_setup({}, &sm) ? 0 : sm;
}

}  // extern "C"
