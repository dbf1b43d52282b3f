// attn_decode.cu - decode attention with rotary and KV-cache append (attn_decode.cuh) behind sqllm_attn_decode (one sequence) and
// sqllm_attn_decode_batch (several, each at its own position).
#include <math.h>
#include <stdint.h>

#include "attn_decode.cuh"
#include "host.h"

using namespace sqllm;

namespace {

template <typename T, int D, bool BATCH>
KernelSmem attn_kernel_of(int G) {
    if (BATCH) {
        switch (G) {
            case 1: return {attn::attn_decode_batch_kernel<T, D, 1>, 0};
            case 2: return {attn::attn_decode_batch_kernel<T, D, 2>, 0};
            case 4: return {attn::attn_decode_batch_kernel<T, D, 4>, 0};
            default: return {attn::attn_decode_batch_kernel<T, D, 8>, 0};
        }
    }
    switch (G) {
        case 1: return {attn::attn_decode_kernel<T, D, 1>, 0};
        case 2: return {attn::attn_decode_kernel<T, D, 2>, 0};
        case 4: return {attn::attn_decode_kernel<T, D, 4>, 0};
        default: return {attn::attn_decode_kernel<T, D, 8>, 0};
    }
}

bool aligned16(const void *ptr) { return ptr && !(reinterpret_cast<uintptr_t>(ptr) & 15); }

constexpr int MAX_BATCH = 65535;  // gridDim.z

int splits(int n_heads, int n_kv, int batch, int sm_count) {
    if (n_kv < 1 || n_heads < n_kv || n_heads % n_kv || sm_count < 1 || batch < 1 || batch > MAX_BATCH) return 0;
    const int g = n_heads / n_kv, hchunks = (g + attn::GMAX - 1) / attn::GMAX;
    const long long clusters = (long long)batch * n_kv * hchunks;
    return (int)std::max(1LL, std::min((long long)attn::MAX_CLUSTER, sm_count / clusters));
}

// the checks and the launch of both entry points; `batch` sequences (the batch-1 entry: 1, on the batch-1 kernel)
template <bool BATCH, typename Args>
int attn_launch(const Args *a, int batch, void *stream) {
    if (a->dtype != SQLLM_DT_F16 && a->dtype != SQLLM_DT_BF16)
        return fail(SQLLM_EINVAL, "dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", a->dtype);
    if (BATCH && (batch < 1 || batch > MAX_BATCH)) return fail(SQLLM_EINVAL, "batch=%d must be in [1, %d]", batch, MAX_BATCH);
    if (a->n_kv < 1 || a->n_heads < 1 || a->n_heads % a->n_kv)
        return fail(SQLLM_EINVAL, "n_heads=%d must be a positive multiple of n_kv=%d", a->n_heads, a->n_kv);
    if (a->head_dim != 64 && a->head_dim != 128) return fail(SQLLM_EINVAL, "head_dim=%d is not 64 or 128", a->head_dim);
    if (a->capacity < 1) return fail(SQLLM_EINVAL, "capacity=%d must be >= 1", a->capacity);
    if (!(isfinite(a->scale) && a->scale > 0.f)) return fail(SQLLM_EINVAL, "scale=%g must be finite and > 0", (double)a->scale);
    const struct { const void *p; const char *name; } ptrs[] = {{a->qkv, "qkv"}, {a->pos, "pos"}, {a->rope_cos, "rope_cos"},
                                                               {a->rope_sin, "rope_sin"}, {a->k_cache, "k_cache"},
                                                               {a->v_cache, "v_cache"}, {a->out, "out"}};
    for (const auto &q : ptrs)
        if (!aligned16(q.p)) return fail(SQLLM_EINVAL, "%s must be a non-null 16-byte aligned pointer", q.name);
    const int g = a->n_heads / a->n_kv, gc = std::min(g, attn::GMAX);
    const int G = gc <= 1 ? 1 : gc <= 2 ? 2 : gc <= 4 ? 4 : 8;
    const bool bf = a->dtype == SQLLM_DT_BF16;
    const KernelSmem k = a->head_dim == 128
                             ? (bf ? attn_kernel_of<__nv_bfloat16, 128, BATCH>(G) : attn_kernel_of<__half, 128, BATCH>(G))
                             : (bf ? attn_kernel_of<__nv_bfloat16, 64, BATCH>(G) : attn_kernel_of<__half, 64, BATCH>(G));
    int sm = 0;
    int rc = dev_setup({}, &sm);
    if (rc) return rc;
    attn::Params p;
    p.qkv = a->qkv; p.pos = a->pos; p.cos = a->rope_cos; p.sin = a->rope_sin;
    p.k_cache = a->k_cache; p.v_cache = a->v_cache; p.out = a->out;
    p.n_heads = a->n_heads; p.n_kv = a->n_kv; p.g = g; p.hchunks = (g + attn::GMAX - 1) / attn::GMAX; p.capacity = a->capacity;
    p.qscale = a->scale * attn::LOG2E;
    const int S = splits(a->n_heads, a->n_kv, batch, sm);
    const dim3 grid(S, a->n_kv * p.hchunks, batch);
    const cudaError_t e = launch_ex(reinterpret_cast<void (*)(attn::Params)>(const_cast<void *>(k.fn)), grid, attn::THREADS, 0,
                                    static_cast<cudaStream_t>(stream), cluster_of(S), p);
    if (e != cudaSuccess)
        return fail(SQLLM_ECUDA, "%s launch failed: %s", BATCH ? "attn_decode_batch" : "attn_decode", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // namespace

extern "C" {

int sqllm_attn_decode_splits(int n_heads, int n_kv, int sm_count) { return splits(n_heads, n_kv, 1, sm_count); }

int sqllm_attn_decode_batch_splits(int n_heads, int n_kv, int batch, int sm_count) { return splits(n_heads, n_kv, batch, sm_count); }

int sqllm_attn_decode(const sqllm_attn_decode_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return attn_launch<false>(a, 1, stream);
}

int sqllm_attn_decode_batch(const sqllm_attn_decode_batch_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return attn_launch<true>(a, a->batch, stream);
}

}  // extern "C"
