// attn_decode.cu - decode attention with rotary and KV-cache append (attn_decode.cuh) behind sqllm_attn_decode (one sequence),
// sqllm_attn_decode_batch (several, each at its own position) and sqllm_attn_decode_paged (several, in one pool of KV pages); causal attention of a chunk of new tokens with the same rotary and
// append (attn_extend.cuh) behind sqllm_attn_extend; decode attention of up to 16 new tokens of one sequence at a device position
// (attn_verify.cuh) behind sqllm_attn_verify; the chunk attention on KV pages behind sqllm_attn_extend_paged; the chunk attention of
// several sequences in one call behind sqllm_attn_extend_batch and sqllm_attn_extend_batch_paged.
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <map>
#include <tuple>
#include <type_traits>

#include "attn_decode.cuh"
#include "attn_extend.cuh"
#include "attn_verify.cuh"
#include "host.h"

using namespace sqllm;

namespace {

// The kernel templates, one tag each: Tag::of<T, D, G>() is the instance for dtype T, head_dim D and G rows per CTA (the chunk kernels
// have no G and ignore it).
struct Decode {
    template <typename T, int D, int G> static auto of() { return attn::attn_decode_kernel<T, D, G>; }
};
struct DecodeBatch {
    template <typename T, int D, int G> static auto of() { return attn::attn_decode_batch_kernel<T, D, G>; }
};
struct DecodePaged {
    template <typename T, int D, int G> static auto of() { return attn::attn_decode_paged_kernel<T, D, G>; }
};
struct Verify {
    template <typename T, int D, int G> static auto of() { return attn::attn_verify_kernel<T, D, G>; }
};
template <typename P> struct Extend {
    template <typename T, int D, int> static auto of() {
        if constexpr (attn::is_paged<P>) return attn::attn_extend_paged_kernel<T, D>;
        else return attn::attn_extend_kernel<T, D>;
    }
};
template <typename P> struct Append {
    template <typename T, int D, int> static auto of() {
        if constexpr (attn::is_paged<P>) return attn::attn_append_paged_kernel<T, D>;
        else return attn::attn_append_kernel<T, D>;
    }
};

template <bool PAGED> struct ExtendBatch {
    template <typename T, int D, int> static auto of() {
        if constexpr (PAGED) return attn::attn_extend_batch_paged_kernel<T, D>;
        else return attn::attn_extend_batch_kernel<T, D>;
    }
};
template <bool PAGED> struct AppendBatch {
    template <typename T, int D, int> static auto of() {
        return attn::attn_append_batch_kernel<T, D, std::conditional_t<PAGED, attn::ExtPagedParams, attn::ExtParams>>;
    }
};

template <typename K, typename T, int D>
auto instance_g(int G) {
    switch (G) {
        case 1: return K::template of<T, D, 1>();
        case 2: return K::template of<T, D, 2>();
        case 4: return K::template of<T, D, 4>();
        default: return K::template of<T, D, 8>();
    }
}

// the instance of kernel template K for a launch's dtype (SQLLM_DT_F16 or SQLLM_DT_BF16), head_dim (64 or 128) and G (group_of)
template <typename K>
auto instance(int dtype, int head_dim, int G = 1) {
    const bool bf = dtype == SQLLM_DT_BF16;
    return head_dim == 128 ? (bf ? instance_g<K, __nv_bfloat16, 128>(G) : instance_g<K, __half, 128>(G))
                           : (bf ? instance_g<K, __nv_bfloat16, 64>(G) : instance_g<K, __half, 64>(G));
}

// G of a CTA of `rows` query rows: rows, at most GMAX, rounded up to the instances' 1, 2, 4 or 8
int group_of(int rows) {
    rows = std::min(rows, attn::GMAX);
    return rows <= 1 ? 1 : rows <= 2 ? 2 : rows <= 4 ? 4 : 8;
}

bool aligned16(const void *ptr) { return ptr && !(reinterpret_cast<uintptr_t>(ptr) & 15); }

// the argument checks every attention entry point shares, in the order they run: the dtype, (the batch,) the head layout, head_dim,
// capacity and scale, (the chunk,) the pointers
int check_dtype(int dtype) {
    if (dtype != SQLLM_DT_F16 && dtype != SQLLM_DT_BF16) return fail(SQLLM_EINVAL, "dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", dtype);
    return SQLLM_OK;
}

template <typename Args>
int check_heads(const Args *a) {
    if (a->n_kv < 1 || a->n_heads < 1 || a->n_heads % a->n_kv)
        return fail(SQLLM_EINVAL, "n_heads=%d must be a positive multiple of n_kv=%d", a->n_heads, a->n_kv);
    if (a->head_dim != 64 && a->head_dim != 128) return fail(SQLLM_EINVAL, "head_dim=%d is not 64 or 128", a->head_dim);
    if (a->capacity < 1) return fail(SQLLM_EINVAL, "capacity=%d must be >= 1", a->capacity);
    if (!(isfinite(a->scale) && a->scale > 0.f)) return fail(SQLLM_EINVAL, "scale=%g must be finite and > 0", (double)a->scale);
    return SQLLM_OK;
}

struct NamedPtr {
    const void *p;
    const char *name;
};
int check_ptrs(std::initializer_list<NamedPtr> ptrs) {
    for (const NamedPtr &q : ptrs)
        if (!aligned16(q.p)) return fail(SQLLM_EINVAL, "%s must be a non-null 16-byte aligned pointer", q.name);
    return SQLLM_OK;
}

constexpr int MAX_BATCH = 65535;  // gridDim.z

int splits(int n_heads, int n_kv, int batch, int sm_count) {
    if (n_kv < 1 || n_heads < n_kv || n_heads % n_kv || sm_count < 1 || batch < 1 || batch > MAX_BATCH) return 0;
    const int g = n_heads / n_kv, hchunks = (g + attn::GMAX - 1) / attn::GMAX;
    const long long clusters = (long long)batch * n_kv * hchunks;
    return (int)std::max(1LL, std::min((long long)attn::MAX_CLUSTER, sm_count / clusters));
}

// the checks of the page arguments both paged entry points share, after check_heads: the pool size, the table width against capacity,
// the pointers of the pools and the table
template <typename Args>
int check_pages(const Args *a) {
    if (a->n_pages < 1) return fail(SQLLM_EINVAL, "n_pages=%d must be >= 1", a->n_pages);
    const int width = (a->capacity + attn::PAGE - 1) / attn::PAGE;
    if (a->table_width != width)
        return fail(SQLLM_EINVAL, "table_width=%d must be ceil(capacity=%d / %d) = %d", a->table_width, a->capacity, attn::PAGE, width);
    if (int rc = check_ptrs({{a->k_pages, "k_pages"}, {a->v_pages, "v_pages"}})) return rc;
    if (!a->block_table || (reinterpret_cast<uintptr_t>(a->block_table) & 3))
        return fail(SQLLM_EINVAL, "block_table must be a non-null 4-byte aligned pointer");
    return SQLLM_OK;
}

// the checks and the launch of sqllm_attn_decode (P = Params, one sequence on the batch-1 kernel), sqllm_attn_decode_batch (Params,
// BATCH: `batch` sequences) and sqllm_attn_decode_paged (PagedParams, BATCH)
template <typename P, bool BATCH, typename Args>
int attn_launch(const Args *a, int batch, void *stream) {
    constexpr bool PAGED = std::is_same<P, attn::PagedParams>::value;
    using K = std::conditional_t<PAGED, DecodePaged, std::conditional_t<BATCH, DecodeBatch, Decode>>;
    if (int rc = check_dtype(a->dtype)) return rc;
    if (BATCH && (batch < 1 || batch > MAX_BATCH)) return fail(SQLLM_EINVAL, "batch=%d must be in [1, %d]", batch, MAX_BATCH);
    if (int rc = check_heads(a)) return rc;
    P p;
    if constexpr (PAGED) {
        if (int rc = check_pages(a)) return rc;
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->pos, "pos"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"}, {a->out, "out"}}))
            return rc;
        p.k_cache = a->k_pages; p.v_cache = a->v_pages; p.table = a->block_table; p.width = a->table_width; p.n_pages = a->n_pages;
    } else {
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->pos, "pos"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"},
                                 {a->k_cache, "k_cache"}, {a->v_cache, "v_cache"}, {a->out, "out"}}))
            return rc;
        p.k_cache = a->k_cache; p.v_cache = a->v_cache;
    }
    const int g = a->n_heads / a->n_kv;
    const auto fn = instance<K>(a->dtype, a->head_dim, group_of(g));
    int sm = 0;
    int rc = dev_setup({}, &sm);
    if (rc) return rc;
    p.qkv = a->qkv; p.pos = a->pos; p.cos = a->rope_cos; p.sin = a->rope_sin; p.out = a->out;
    p.n_heads = a->n_heads; p.n_kv = a->n_kv; p.g = g; p.hchunks = (g + attn::GMAX - 1) / attn::GMAX; p.capacity = a->capacity;
    p.qscale = a->scale * attn::LOG2E;
    const int S = splits(a->n_heads, a->n_kv, batch, sm);   // the paged kernel: the rule of sqllm_attn_decode_batch, the same bits per row
    const dim3 grid(S, a->n_kv * p.hchunks, batch);
    const cudaError_t e = launch_ex(fn, grid, attn::THREADS, 0, static_cast<cudaStream_t>(stream), cluster_of(S), p);
    if (e != cudaSuccess)
        return fail(SQLLM_ECUDA, "%s launch failed: %s", PAGED ? "attn_decode_paged" : BATCH ? "attn_decode_batch" : "attn_decode",
                    cudaGetErrorString(e));
    return SQLLM_OK;
}

// the rows of the chunk's query tiles (T tokens x g heads of a group), 0 when they need more tiles than the grid holds
long long ext_tiles(int n_heads, int n_kv, int T) {
    const long long tiles = ((long long)T * (n_heads / n_kv) + attn::BM - 1) / attn::BM;
    return tiles <= attn::MAX_TILES ? tiles : 0;
}

// CTAs per cluster of sqllm_attn_extend: 1 when the query tiles alone fill the SMs, else as many as the SMs left per tile allow, at
// most MAX_CLUSTER and at most the key blocks of the longest tile (start + T keys)
int ext_splits(int n_heads, int n_kv, int T, int start, int sm_count) {
    if (n_kv < 1 || n_heads < n_kv || n_heads % n_kv || T < 1 || start < 0 || sm_count < 1 || (long long)start + T > INT_MAX) return 0;
    const long long tiles = ext_tiles(n_heads, n_kv, T) * n_kv;
    if (tiles == 0) return 0;
    const long long blocks = ((long long)start + T + attn::BN - 1) / attn::BN;
    return (int)std::max(1LL, std::min({(long long)attn::MAX_CLUSTER, sm_count / tiles, blocks}));
}

// the checks and both launches of sqllm_attn_extend (P = ExtParams) and sqllm_attn_extend_paged (P = ExtPagedParams)
template <typename P, typename Args>
int extend_launch(const Args *a, void *stream) {
    constexpr bool PAGED = attn::is_paged<P>;
    if (int rc = check_dtype(a->dtype)) return rc;
    if (int rc = check_heads(a)) return rc;
    if (a->n_tokens < 1) return fail(SQLLM_EINVAL, "n_tokens=%d must be >= 1", a->n_tokens);
    if (a->start < 0) return fail(SQLLM_EINVAL, "start=%d must be >= 0", a->start);
    if ((long long)a->start + a->n_tokens > a->capacity)
        return fail(SQLLM_EINVAL, "start=%d + n_tokens=%d must be <= capacity=%d", a->start, a->n_tokens, a->capacity);
    if (ext_tiles(a->n_heads, a->n_kv, a->n_tokens) == 0 || a->n_kv > 65535)
        return fail(SQLLM_EINVAL, "n_tokens=%d x %d heads per KV head needs more than %d query tiles of %d, or n_kv=%d > 65535",
                    a->n_tokens, a->n_heads / a->n_kv, attn::MAX_TILES, attn::BM, a->n_kv);
    P p;
    if constexpr (PAGED) {
        if (int rc = check_pages(a)) return rc;
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"}, {a->out, "out"}})) return rc;
        p.k_cache = a->k_pages; p.v_cache = a->v_pages; p.table = a->block_table; p.n_pages = a->n_pages;
    } else {
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"}, {a->k_cache, "k_cache"},
                                 {a->v_cache, "v_cache"}, {a->out, "out"}}))
            return rc;
        p.k_cache = a->k_cache; p.v_cache = a->v_cache;
    }
    const auto fn = instance<Extend<P>>(a->dtype, a->head_dim);
    const int bytes = attn::ext_smem_bytes(a->head_dim);
    int sm = 0;
    int rc = dev_setup({KernelSmem(fn, bytes)}, &sm);
    if (rc) return rc;
    p.qkv = a->qkv; p.cos = a->rope_cos; p.sin = a->rope_sin; p.out = a->out;
    p.n_heads = a->n_heads; p.n_kv = a->n_kv; p.g = a->n_heads / a->n_kv; p.capacity = a->capacity; p.start = a->start; p.T = a->n_tokens;
    p.qscale = a->scale * attn::LOG2E / attn::QPRE;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const auto append = instance<Append<P>>(a->dtype, a->head_dim);
    const char *name = PAGED ? "attn_extend_paged" : "attn_extend";
    append<<<a->n_tokens, attn::APPEND_THREADS, 0, st>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "%s append launch failed: %s", name, cudaGetErrorString(e));
    const int S = ext_splits(a->n_heads, a->n_kv, a->n_tokens, a->start, sm);
    const dim3 grid(S, (unsigned)ext_tiles(a->n_heads, a->n_kv, a->n_tokens), a->n_kv);
    e = launch_ex(fn, grid, attn::XTHREADS, bytes, st, cluster_of(S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "%s launch failed: %s", name, cudaGetErrorString(e));
    return SQLLM_OK;
}

static_assert(attn::MAX_SEGMENTS == SQLLM_ATTN_EXTEND_MAX_SEGMENTS, "one segment limit for the kernels and the header");

// the checks and the launches of sqllm_attn_extend_batch (Args = sqllm_attn_extend_batch_args) and sqllm_attn_extend_batch_paged: the
// append of every segment's rows, then one attention launch per distinct split S_i, its segments by key range start + T longest first
template <bool PAGED, typename Args>
int extend_batch_launch(const Args *a, void *stream) {
    if (int rc = check_dtype(a->dtype)) return rc;
    if (int rc = check_heads(a)) return rc;
    const int n = a->n_segments;
    if (n < 1 || n > attn::MAX_SEGMENTS) return fail(SQLLM_EINVAL, "n_segments=%d must be in [1, %d]", n, attn::MAX_SEGMENTS);
    if (a->n_slots < 1) return fail(SQLLM_EINVAL, "n_slots=%d must be >= 1", a->n_slots);
    if (!a->slots || !a->starts || !a->n_tokens) return fail(SQLLM_EINVAL, "slots, starts and n_tokens must be non-null host arrays");
    if (a->n_kv > 65535) return fail(SQLLM_EINVAL, "n_kv=%d > 65535", a->n_kv);
    long long tiles = 0;
    for (int i = 0; i < n; ++i) {
        const int slot = a->slots[i], start = a->starts[i], T = a->n_tokens[i];
        if (slot < 0 || slot >= a->n_slots) return fail(SQLLM_EINVAL, "slots[%d]=%d must be in [0, n_slots=%d)", i, slot, a->n_slots);
        for (int j = 0; j < i; ++j)
            if (a->slots[j] == slot) return fail(SQLLM_EINVAL, "slots[%d]=%d repeats slots[%d]", i, slot, j);
        if (T < 1) return fail(SQLLM_EINVAL, "n_tokens[%d]=%d must be >= 1", i, T);
        if (start < 0) return fail(SQLLM_EINVAL, "starts[%d]=%d must be >= 0", i, start);
        if ((long long)start + T > a->capacity)
            return fail(SQLLM_EINVAL, "starts[%d]=%d + n_tokens[%d]=%d must be <= capacity=%d", i, start, i, T, a->capacity);
        tiles += ((long long)T * (a->n_heads / a->n_kv) + attn::BM - 1) / attn::BM;
    }
    if (tiles > attn::MAX_TILES)
        return fail(SQLLM_EINVAL, "the segments need %lld query tiles of %d per KV head, more than %d", tiles, attn::BM, attn::MAX_TILES);
    attn::ExtBatchParams b;
    if constexpr (PAGED) {
        if (int rc = check_pages(a)) return rc;
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"}, {a->out, "out"}})) return rc;
        b.k_cache = a->k_pages; b.v_cache = a->v_pages; b.table = a->block_table; b.width = a->table_width; b.n_pages = a->n_pages;
    } else {
        if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"}, {a->k_cache, "k_cache"},
                                 {a->v_cache, "v_cache"}, {a->out, "out"}}))
            return rc;
        b.k_cache = a->k_cache; b.v_cache = a->v_cache; b.table = nullptr; b.width = 0; b.n_pages = 0;
    }
    const auto fn = instance<ExtendBatch<PAGED>>(a->dtype, a->head_dim);
    const int bytes = attn::ext_smem_bytes(a->head_dim);
    int sm = 0;
    int rc = dev_setup({KernelSmem(fn, bytes)}, &sm);
    if (rc) return rc;
    b.qkv = a->qkv; b.cos = a->rope_cos; b.sin = a->rope_sin; b.out = a->out;
    b.n_heads = a->n_heads; b.n_kv = a->n_kv; b.g = a->n_heads / a->n_kv; b.capacity = a->capacity; b.start = 0; b.T = 0;
    b.qscale = a->scale * attn::LOG2E / attn::QPRE;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const char *name = PAGED ? "attn_extend_batch_paged" : "attn_extend_batch";

    // the append: every segment's rows in the caller's order
    b.n = n;
    int rows = 0, S[attn::MAX_SEGMENTS];
    attn::ExtSegment all[attn::MAX_SEGMENTS];
    for (int i = 0; i < n; ++i) {
        all[i] = {a->slots[i], a->starts[i], a->n_tokens[i], rows};
        b.first[i] = rows;
        b.seg[i] = all[i];
        rows += a->n_tokens[i];
        S[i] = ext_splits(a->n_heads, a->n_kv, a->n_tokens[i], a->starts[i], sm);
    }
    const auto append = instance<AppendBatch<PAGED>>(a->dtype, a->head_dim);
    append<<<rows, attn::APPEND_THREADS, 0, st>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "%s append launch failed: %s", name, cudaGetErrorString(e));

    // the attention: per split, its segments by key range, longest first (ties in the caller's order)
    for (int s = attn::MAX_CLUSTER; s >= 1; --s) {
        int order[attn::MAX_SEGMENTS], m = 0;
        for (int i = 0; i < n; ++i)
            if (S[i] == s) order[m++] = i;
        if (m == 0) continue;
        std::stable_sort(order, order + m, [&](int x, int y) {
            return (long long)all[x].start + all[x].T > (long long)all[y].start + all[y].T;
        });
        int tiles_s = 0;
        for (int k = 0; k < m; ++k) {
            b.first[k] = tiles_s;
            b.seg[k] = all[order[k]];
            tiles_s += (int)ext_tiles(a->n_heads, a->n_kv, all[order[k]].T);
        }
        b.n = m;
        e = launch_ex(fn, dim3(s, tiles_s, a->n_kv), attn::XTHREADS, bytes, st, cluster_of(s), b);
        if (e != cudaSuccess) return fail(SQLLM_ECUDA, "%s launch failed: %s", name, cudaGetErrorString(e));
    }
    return SQLLM_OK;
}

// clusters per KV head of sqllm_attn_verify: chunks of GMAX of the T * g (token, query head) rows of its group
int ver_chunks(int n_heads, int n_kv, int T) { return (T * (n_heads / n_kv) + attn::GMAX - 1) / attn::GMAX; }

// the split rule of sqllm_attn_verify: as splits() for the n_kv * ver_chunks clusters, an upper bound on what a launch uses (below);
// 0 for invalid arguments
int ver_splits(int n_heads, int n_kv, int T, int sm_count) {
    if (n_kv < 1 || n_heads < n_kv || n_heads % n_kv || sm_count < 1 || T < 1 || T > attn::VMAX) return 0;
    const long long clusters = (long long)n_kv * ver_chunks(n_heads, n_kv, T);
    if (clusters > MAX_BATCH) return 0;
    return (int)std::max(1LL, std::min((long long)attn::MAX_CLUSTER, sm_count / clusters));
}

// the checks of a verify launch that need no pointers, in the order they run
template <typename Args>
int ver_check(const Args *a) {
    if (int rc = check_dtype(a->dtype)) return rc;
    if (int rc = check_heads(a)) return rc;
    if (a->n_tokens < 1 || a->n_tokens > attn::VMAX) return fail(SQLLM_EINVAL, "n_tokens=%d must be in [1, %d]", a->n_tokens, attn::VMAX);
    if ((long long)a->n_kv * ver_chunks(a->n_heads, a->n_kv, a->n_tokens) > MAX_BATCH)
        return fail(SQLLM_EINVAL, "n_kv=%d x %d clusters per KV head exceeds %d", a->n_kv, ver_chunks(a->n_heads, a->n_kv, a->n_tokens),
                    MAX_BATCH);
    return SQLLM_OK;
}

// the kernel instance of a verify launch: a CTA's rows are T g, at most GMAX
auto ver_kernel(int n_heads, int n_kv, int T, int head_dim, int dtype) {
    return instance<Verify>(dtype, head_dim, group_of(T * (n_heads / n_kv)));
}

// The CTAs per cluster a verify launch of `clusters` clusters of kernel `fn` uses on the current device: the rule's S, lowered until
// every cluster is resident at once (cudaOccupancyMaxActiveClusters, asked once per device, kernel and S).  At 115 to 253 registers
// per thread one or two CTAs of an instance fit an SM, and a cluster's CTAs must share a GPC, so the rule's S can leave clusters
// for a second wave, which costs more than the longer position ranges of a smaller S.  S = 1 has no cluster constraint.
int ver_launch_splits(const void *fn, int S, long long clusters, int *out) {
    static std::map<std::tuple<int, const void *, int>, int> active;  // (device, kernel, S) -> max active clusters
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(SQLLM_ECUDA, "cudaGetDevice failed");
    for (; S > 1; --S) {
        auto it = active.find({dev, fn, S});
        if (it == active.end()) {
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3(S, (unsigned)clusters);
            cfg.blockDim = dim3(attn::THREADS);
            cudaLaunchAttribute attr;
            attr.id = cudaLaunchAttributeClusterDimension;
            attr.val.clusterDim.x = S; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
            cfg.attrs = &attr;
            cfg.numAttrs = 1;
            int n = 0;
            if (cudaOccupancyMaxActiveClusters(&n, fn, &cfg) != cudaSuccess)
                return fail(SQLLM_ECUDA, "cudaOccupancyMaxActiveClusters failed: %s", cudaGetErrorString(cudaGetLastError()));
            it = active.emplace(std::make_tuple(dev, fn, S), n).first;
        }
        if (it->second >= clusters) break;
    }
    *out = S;
    return SQLLM_OK;
}

int verify_launch(const sqllm_attn_verify_args *a, void *stream) {
    if (int rc = ver_check(a)) return rc;
    if (int rc = check_ptrs({{a->qkv, "qkv"}, {a->pos, "pos"}, {a->rope_cos, "rope_cos"}, {a->rope_sin, "rope_sin"},
                             {a->k_cache, "k_cache"}, {a->v_cache, "v_cache"}, {a->out, "out"}}))
        return rc;
    const auto fn = ver_kernel(a->n_heads, a->n_kv, a->n_tokens, a->head_dim, a->dtype);
    int sm = 0;
    int rc = dev_setup({}, &sm);
    if (rc) return rc;
    attn::VerParams p;
    p.qkv = a->qkv; p.pos = a->pos; p.cos = a->rope_cos; p.sin = a->rope_sin;
    p.k_cache = a->k_cache; p.v_cache = a->v_cache; p.out = a->out;
    p.n_heads = a->n_heads; p.n_kv = a->n_kv; p.g = a->n_heads / a->n_kv; p.chunks = ver_chunks(a->n_heads, a->n_kv, a->n_tokens);
    p.capacity = a->capacity; p.T = a->n_tokens;
    p.qscale = a->scale * attn::LOG2E;
    int S = 0;
    if ((rc = ver_launch_splits((const void *)fn, ver_splits(a->n_heads, a->n_kv, a->n_tokens, sm), (long long)a->n_kv * p.chunks, &S)))
        return rc;
    const dim3 grid(S, a->n_kv * p.chunks);
    const cudaError_t e = launch_ex(fn, grid, attn::THREADS, 0, static_cast<cudaStream_t>(stream), cluster_of(S), p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "attn_verify launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

}  // namespace

extern "C" {

int sqllm_attn_decode_splits(int n_heads, int n_kv, int sm_count) { return splits(n_heads, n_kv, 1, sm_count); }

int sqllm_attn_decode_batch_splits(int n_heads, int n_kv, int batch, int sm_count) { return splits(n_heads, n_kv, batch, sm_count); }

int sqllm_attn_decode(const sqllm_attn_decode_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return attn_launch<attn::Params, false>(a, 1, stream);
}

int sqllm_attn_decode_batch(const sqllm_attn_decode_batch_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return attn_launch<attn::Params, true>(a, a->batch, stream);
}

int sqllm_attn_extend_splits(int n_heads, int n_kv, int n_tokens, int start, int sm_count) {
    return ext_splits(n_heads, n_kv, n_tokens, start, sm_count);
}

int sqllm_attn_extend(const sqllm_attn_extend_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return extend_launch<attn::ExtParams>(a, stream);
}

int sqllm_attn_decode_paged(const sqllm_attn_decode_paged_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return attn_launch<attn::PagedParams, true>(a, a->batch, stream);
}

int sqllm_attn_extend_paged(const sqllm_attn_extend_paged_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return extend_launch<attn::ExtPagedParams>(a, stream);
}

int sqllm_attn_extend_batch(const sqllm_attn_extend_batch_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return extend_batch_launch<false>(a, stream);
}

int sqllm_attn_extend_batch_paged(const sqllm_attn_extend_batch_paged_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return extend_batch_launch<true>(a, stream);
}

int sqllm_attn_verify_splits(int n_heads, int n_kv, int n_tokens, int sm_count) { return ver_splits(n_heads, n_kv, n_tokens, sm_count); }

int sqllm_attn_verify_launch_splits(int dtype, int n_heads, int n_kv, int head_dim, int n_tokens) {
    struct { int dtype, n_heads, n_kv, head_dim, capacity, n_tokens; float scale; } a = {dtype, n_heads, n_kv, head_dim, 1, n_tokens, 1.f};
    if (ver_check(&a)) return 0;
    int sm = 0, S = 0;
    if (dev_setup({}, &sm)) return 0;
    if (ver_launch_splits((const void *)ver_kernel(n_heads, n_kv, n_tokens, head_dim, dtype), ver_splits(n_heads, n_kv, n_tokens, sm),
                          (long long)n_kv * ver_chunks(n_heads, n_kv, n_tokens), &S))
        return 0;
    return S;
}

int sqllm_attn_verify(const sqllm_attn_verify_args *a, void *stream) {
    if (!a) return fail(SQLLM_EINVAL, "null args");
    return verify_launch(a, stream);
}

}  // extern "C"
