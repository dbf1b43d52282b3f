// attn_decode.cuh - decode attention of one layer for one token of one sequence (sqllm_attn_decode) or of B sequences at once
// (sqllm_attn_decode_batch): rotary on q and the new k, the append of k / v at slot `pos` of the KV cache, and
// softmax(scale q.K^T[0..pos]) V[0..pos] per query head with grouped KV heads.
//
// Shape.  One thread-block cluster of S CTAs per (sequence, KV head, chunk of up to GMAX query heads of its group); S depends on the
// batch, n_kv and the SM count only.  The batched kernel is the batch-1 kernel's device code per sequence, blockIdx.z the sequence.  The positions 0..pos are dealt to the S CTAs in blocks of BLOCK_POS, a range each CTA computes from the device
// `pos`, and inside a CTA to its 8 warps, U * RPW positions per warp step.  A K / V row is D/8 lanes of 16 bytes (RPW rows per warp
// load), read straight into registers with no L1 allocation; every K / V load serves the G query heads of the CTA.  Each lane keeps an
// online softmax (m, l, acc) per head for the positions of its row slot; the partial states are combined in a fixed order: the row
// slots of a warp by an xor tree, the warps of a CTA in warp order, the CTAs of the cluster in rank order over distributed shared
// memory.  No workspace, no atomics: bit-reproducible.
//
// The CTA whose range holds `pos` takes the new k (rotated, rounded to the dtype) and v from its shared memory, where every CTA
// computes them from qkv; one CTA stores them into the cache.  So no CTA reads a cache slot another CTA of the launch writes, and no
// slot past `pos` is read.
//
// The paged kernel (sqllm_attn_decode_paged) is the batched kernel with the caches in a pool of PAGE-position pages: row b's position
// t is row t % PAGE of page table[b][t / PAGE].  A CTA's range starts at a block of BLOCK_POS = PAGE positions, so each warp step
// looks its page up once.
#pragma once
#include "common.cuh"

namespace {
namespace attn {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_CLUSTER = 8;   // portable cluster size
constexpr int BLOCK_POS = 64;    // positions are dealt to the CTAs of a cluster in blocks of this many
constexpr int GMAX = 8;          // query heads per CTA: a larger group is split over several clusters, each reading the K / V again
constexpr float LOG2E = 1.4426950408889634f;
constexpr int PAGE = 64;         // positions per KV page of the paged kernels: one page is one BLOCK_POS block of a CTA's range
static_assert(PAGE == BLOCK_POS, "a KV page must be exactly one block of positions");

struct Params {                // the batched kernel: each of qkv, pos, the caches and out [batch] times over
    const void *qkv;             // [n_heads*D | n_kv*D | n_kv*D]
    const int *pos;
    const float *cos, *sin;      // [capacity][D/2]
    void *k_cache, *v_cache;     // [n_kv][capacity][D]
    void *out;                   // [n_heads*D]
    int n_heads, n_kv, g, hchunks, capacity;
    float qscale;                // scale * log2(e): scores in base 2
};

// the paged batched kernel: the caches are page pools [n_pages][n_kv][PAGE][D] shared by the rows; row b's position t is row t % PAGE
// of page table[b * width + t / PAGE]
struct PagedParams : Params {
    const int *table;            // [batch][width]
    int width, n_pages;
};

// one row's block table, as attn_decode_row.inc reads it (the contiguous kernels pass an empty one they never read)
struct Pages {
    const int *table;
    int n_pages;
};

// the CTA's verdict on a row at `pos`: every entry of blocks 0 .. pos / PAGE names a page of the pool.  Every thread takes part.
__device__ __forceinline__ bool pages_valid(const Pages pg, int pos) {
    bool bad = false;
    for (int i = threadIdx.x; i <= pos / PAGE; i += blockDim.x) {
        const int id = pg.table[i];
        bad |= id < 0 || id >= pg.n_pages;
    }
    return !__syncthreads_or(bad);
}

// element offset of page `id`'s rows of KV head kvh in a pool [n_pages][n_kv][PAGE][D]
template <int D>
__device__ __forceinline__ size_t page_base(int id, int n_kv, int kvh) { return ((size_t)id * n_kv + kvh) * PAGE * D; }

// positions [p0, p1) of CTA `rank` of S for pos + 1 positions: blocks of BLOCK_POS, ceil(blocks / S) per CTA
__device__ __forceinline__ void cta_range(int pos, int rank, int S, int &p0, int &p1) {
    const int blocks = (pos + BLOCK_POS) / BLOCK_POS;
    const int chunk = (blocks + S - 1) / S * BLOCK_POS;
    p0 = rank * chunk;
    p1 = min(pos + 1, p0 + chunk);
}

__device__ __forceinline__ float ld_cluster_f32(const float *local, uint32_t rank) {
    uint32_t a;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(smem_u32(local)), "r"(rank));
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// the 8 values of a 16-byte word of T as fp32 (exact)
template <typename T>
__device__ __forceinline__ void unpack8(const uint4 w, float (&f)[8]) {
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 t = x16x2_to_f32x2<T>(u[j]);
        f[2 * j] = t.x;
        f[2 * j + 1] = t.y;
    }
}

// exp2(a - b) with exp2(-inf) = 0 whatever b is (an empty state or a masked position weighs nothing)
__device__ __forceinline__ float wexp2(float a, float b) { return a == -INFINITY ? 0.f : exp2f(a - b); }

// rotary (rotate-half) in fp32: element i of the rotated x, from the pair (a, b) = (x[j], x[j + D/2]) and the row (cs, sn) of the
// cos / sin tables at x's position, j = i % (D/2).  Every kernel rotates q and k with this one expression, so a cache slot holds the
// same bits whichever kernel wrote it (decode, batched, paged, verify or append), and q' is the same whichever kernel attends with it.
template <int D>
__device__ __forceinline__ float rope(float a, float b, const float *cs, const float *sn, int i) {
    const int j = i % (D / 2);
    return i < D / 2 ? a * cs[j] - b * sn[j] : b * cs[j] + a * sn[j];
}

// batch 1: one sequence at *p.pos.  Kept beside the batched kernel, which computes the same bits at batch 1 but up to 0.9 % slower
// (DESIGN §3.18)
template <typename T, int D, int G>
__global__ void __launch_bounds__(THREADS, 1) attn_decode_kernel(const Params p) {
    constexpr bool PAGED = false;
    const Pages pg{};
#include "attn_decode_row.inc"
}

// gridDim.z sequences: sequence b = blockIdx.z at all.pos[b], with its own qkv row, caches and out row (the batch-1 layouts, one
// after another); the rotary tables are shared
template <typename T, int D, int G>
__global__ void __launch_bounds__(THREADS, 1) attn_decode_batch_kernel(const Params all) {
    const int b = blockIdx.z;
    const size_t cache = (size_t)b * all.n_kv * all.capacity * D;
    Params p = all;
    p.qkv = static_cast<const T *>(all.qkv) + (size_t)b * (all.n_heads + 2 * all.n_kv) * D;
    p.pos = all.pos + b;
    p.k_cache = static_cast<T *>(all.k_cache) + cache;
    p.v_cache = static_cast<T *>(all.v_cache) + cache;
    p.out = static_cast<T *>(all.out) + (size_t)b * all.n_heads * D;
    constexpr bool PAGED = false;
    const Pages pg{};
#include "attn_decode_row.inc"
}

// gridDim.z sequences in one page pool: sequence b = blockIdx.z at all.pos[b] through row b of the block table, with its own qkv and out
// rows; a row with an entry outside [0, n_pages) among the blocks it reads or writes is idle.  The same code as the batched kernel but
// for the addressing, so a row is bitwise what the batched kernel computes on the row's pages gathered into a contiguous cache.
template <typename T, int D, int G>
__global__ void __launch_bounds__(THREADS, 1) attn_decode_paged_kernel(const PagedParams all) {
    const int b = blockIdx.z;
    Params p = all;
    p.qkv = static_cast<const T *>(all.qkv) + (size_t)b * (all.n_heads + 2 * all.n_kv) * D;
    p.pos = all.pos + b;
    p.out = static_cast<T *>(all.out) + (size_t)b * all.n_heads * D;
    constexpr bool PAGED = true;
    const Pages pg{all.table + (size_t)b * all.width, all.n_pages};
#include "attn_decode_row.inc"
}

}  // namespace attn
}  // namespace
