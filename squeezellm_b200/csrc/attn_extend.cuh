// attn_extend.cuh - attention of one layer for a chunk of T new tokens of one sequence at positions start .. start+T-1
// (sqllm_attn_extend): the append of the chunk's rotated k and its v at slots start .. start+T-1 of the KV cache, then causal
// softmax(scale q'.K^T[0..p]) V[0..p] for every token (p = start + t) and query head, with grouped KV heads.  Two launches on one stream:
//
//   attn_append_kernel   one CTA per token: k' = rotary(k) in fp32 rounded to the dtype once - rope() of attn_decode.cuh, so a slot
//                        holds the same bits whichever kernel wrote it - and v unchanged.
//   attn_extend_kernel   FlashAttention-2 style, K / V read from the cache only (so no CTA reads a slot written in the same launch).
//
// Shape of attn_extend_kernel.  A query tile is BM = 64 (token, query head) rows of one KV head's group, token-major (row r of the
// group's T*g rows is token r / g, head r % g), so every K / V tile serves all g heads of the group: GQA without repeating K / V.
// grid (S, tiles, n_kv), clusters of S CTAs along x; the tiles run last-first (the longest key ranges start first).  The tile's keys
// 0 .. start + t_last are dealt to the S CTAs of its cluster in blocks of BN = 64, ceil(blocks / S) per CTA.  A CTA streams its blocks
// through shared memory with cp.async, double-buffered (16-byte chunks xor-swizzled by row against ldmatrix bank conflicts); keys at
// or past the tile's limit are zero-filled, never read.  Each of the 4 warps owns 16 rows: S = Q K^T and O += P V on mma.sync m16n8k16
// with fp32 accumulation.  K and V are exact in the dtype; q' (fp32) and P (fp32) are each split into hi + lo
// parts in the dtype (q' staged in shared memory, P straight from the score registers), two MMAs per product, so the operands carry
// about 22 (fp16) or 16 (bf16) bits instead of 11 or 8.  Only blocks that cross the causal edge are masked; the softmax is online, in fp32 with exp2.  With S > 1 the CTAs' (m, l, acc) states are combined in rank order over
// distributed shared memory, as attn_decode's are.  No workspace, no atomics: bit-reproducible.
//
// Paged (sqllm_attn_extend_paged): attn_append_paged_kernel and attn_extend_paged_kernel are the same code with the cache addressed
// through the sequence's block table (ExtPagedParams): key block kb is page table[kb] of the pools, so a K / V block is one page.
//
// Several sequences (sqllm_attn_extend_batch, _paged): attn_append_batch_kernel, attn_extend_batch_kernel and
// attn_extend_batch_paged_kernel run the same code per segment of a segment table in the kernel parameters (below).
#pragma once
#include "attn_decode.cuh"

namespace {
namespace attn {

constexpr int XTHREADS = 128;      // 4 warps x 16 query rows
constexpr int BM = 64;             // (token, head) rows per query tile
constexpr int BN = 64;             // keys per K / V block
constexpr int APPEND_THREADS = 256;
constexpr float QPRE = 0.25f;      // q' is split at q'/4 (exact): |q'| <= sqrt(2) * 65504 stays finite in fp16; 4 goes into the scale
constexpr int MAX_TILES = 65535;   // gridDim.y
static_assert(PAGE == BN, "a KV page must be exactly one K / V block");

struct ExtParams {
    const void *qkv;             // [T][n_heads*D | n_kv*D | n_kv*D]
    const float *cos, *sin;      // [capacity][D/2]
    void *k_cache, *v_cache;     // [n_kv][capacity][D]
    void *out;                   // [T][n_heads*D]
    int n_heads, n_kv, g, capacity, start, T;
    float qscale;                // scale * log2(e) / QPRE: scores in base 2
};

// the paged kernels: the caches are page pools [n_pages][n_kv][PAGE][D]; position t is row t % PAGE of page table[t / PAGE]
struct ExtPagedParams : ExtParams {
    const int *table;            // the sequence's block table, entries 0 .. (start + T - 1) / PAGE read
    int n_pages;
};

template <typename P> constexpr bool is_paged = std::is_same<P, ExtPagedParams>::value;

// the CTA's verdict on a paged launch: every entry of blocks 0 .. (start + T - 1) / PAGE names a page of the pool (every launch of the
// chunk checks the same entries, so either all write or none does).  Every thread takes part.
template <typename P>
__device__ __forceinline__ bool ext_pages_valid(const P &p) {
    if constexpr (is_paged<P>) return pages_valid(Pages{p.table, p.n_pages}, p.start + p.T - 1);
    else return true;
}

// dynamic shared memory of attn_extend_kernel: K and V, two stages each (the cluster combine reuses them for [BM][D] fp32), q' hi and lo
constexpr int ext_smem_bytes(int d) { return (2 * 2 * BN + 2 * BM) * d * 2; }

template <typename T> struct Pair;
template <> struct Pair<__half> { using type = __half2; };
template <> struct Pair<__nv_bfloat16> { using type = __nv_bfloat162; };

// (a, b) rounded to T, a in the low half
template <typename T>
__device__ __forceinline__ uint32_t pack_t(float a, float b) {
    typename Pair<T>::type v;
    v.x = f32_to<T>(a);
    v.y = f32_to<T>(b);
    return *reinterpret_cast<uint32_t *>(&v);
}

// x = hi + lo + r: hi = T(x), lo = T(x - hi) for the pair (a, b)
template <typename T>
__device__ __forceinline__ void split_pair(float a, float b, uint32_t &hi, uint32_t &lo) {
    const T ha = f32_to<T>(a), hb = f32_to<T>(b);
    typename Pair<T>::type h;
    h.x = ha;
    h.y = hb;
    hi = *reinterpret_cast<uint32_t *>(&h);
    lo = pack_t<T>(a - to_f32(ha), b - to_f32(hb));
}

template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if constexpr (std::is_same<T, __half>::value) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// element offset of (row, 16-byte chunk) in a [BN][D] tile: the chunk xor-swizzled by the row's low 3 bits
template <int D>
__device__ __forceinline__ int swz(int row, int chunk) { return row * D + ((chunk ^ (row & 7)) << 3); }

// the CTA of token t: k' and v of every KV head into slot start + t.  P: ExtParams (a contiguous cache) or ExtPagedParams (pools).
template <typename T, int D, typename P>
__device__ __forceinline__ void append_body(const P &p, int t) {
    if (!ext_pages_valid(p)) return;
    const int pos = p.start + t;
    const T *qkv = static_cast<const T *>(p.qkv) + (size_t)t * (p.n_heads + 2 * p.n_kv) * D;
    const float *cs = p.cos + (size_t)pos * (D / 2), *sn = p.sin + (size_t)pos * (D / 2);
    for (int idx = threadIdx.x; idx < p.n_kv * D; idx += APPEND_THREADS) {
        const int kvh = idx / D, i = idx % D, j = i % (D / 2);
        const T *k = qkv + (size_t)p.n_heads * D + (size_t)kvh * D;
        const float a = to_f32(k[j]), b = to_f32(k[j + D / 2]);
        size_t slot;
        if constexpr (is_paged<P>) slot = page_base<D>(p.table[pos / PAGE], p.n_kv, kvh) + (size_t)(pos % PAGE) * D + i;
        else slot = ((size_t)kvh * p.capacity + pos) * D + i;
        static_cast<T *>(p.k_cache)[slot] = f32_to<T>(rope<D>(a, b, cs, sn, i));
        static_cast<T *>(p.v_cache)[slot] = qkv[(size_t)(p.n_heads + p.n_kv) * D + (size_t)kvh * D + i];
    }
}

template <typename T, int D>
__global__ void __launch_bounds__(APPEND_THREADS) attn_append_kernel(const ExtParams p) { append_body<T, D>(p, blockIdx.x); }
template <typename T, int D>
__global__ void __launch_bounds__(APPEND_THREADS) attn_append_paged_kernel(const ExtPagedParams p) { append_body<T, D>(p, blockIdx.x); }

template <typename T, int D>
__global__ void __launch_bounds__(XTHREADS, 1) attn_extend_kernel(const ExtParams p) {
    constexpr bool PAGED = false;
    const Pages pg{};
    const int tile = gridDim.y - 1 - blockIdx.y;   // last-first
#include "attn_extend_tile.inc"
}

// the same tile on page pools; key block kb is page p.table[kb]
template <typename T, int D>
__global__ void __launch_bounds__(XTHREADS, 1) attn_extend_paged_kernel(const ExtPagedParams p) {
    constexpr bool PAGED = true;
    const Pages pg{p.table, p.n_pages};
    const int tile = gridDim.y - 1 - blockIdx.y;
#include "attn_extend_tile.inc"
}

// ---- several sequences' chunks in one launch (sqllm_attn_extend_batch, sqllm_attn_extend_batch_paged) ----
//
// Segment i of a call is the chunk (slot_i, start_i, T_i): rows row0_i .. row0_i + T_i - 1 of qkv and out, row0_i = the sum of T_j over
// the segments before it in the caller's order.  Each kernel finds its segment by binary search over `first`, the launch's first unit
// (a row of the append, a query tile of the attention) of each segment, and then runs the single-sequence kernel's code on the segment
// alone: the segment's qkv and out rows and, contiguous, its slot's caches; paged, its slot's block table row.  So a segment's bits are
// those of the single-sequence launches with (start_i, T_i) on its slot, whatever the other segments are.
constexpr int MAX_SEGMENTS = 128;  // SQLLM_ATTN_EXTEND_MAX_SEGMENTS

struct ExtSegment {
    int slot, start, T, row0;
};

struct ExtBatchParams : ExtParams {  // qkv [sum T][...], out [sum T][...]; k_cache / v_cache [n_slots][n_kv][capacity][D] or page pools
    const int *table;                // paged: [n_slots][width]
    int width, n_pages;
    int n;                           // segments in this launch
    int first[MAX_SEGMENTS];         // ascending: segment i's units are first[i] .. first[i + 1] - 1
    ExtSegment seg[MAX_SEGMENTS];
};
static_assert(sizeof(ExtBatchParams) <= 4096, "the segment table travels in the kernel parameters, at most 4 KB");

// the segment of unit u: the last i with first[i] <= u
__device__ __forceinline__ int segment_of(const ExtBatchParams &b, int u) {
    int lo = 0, hi = b.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (b.first[mid] <= u) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// the parameters of the single-sequence kernels for segment s alone (P: ExtParams or ExtPagedParams)
template <typename T, int D, typename P>
__device__ __forceinline__ P segment_params(const ExtBatchParams &b, const ExtSegment &s) {
    P p;
    static_cast<ExtParams &>(p) = b;
    p.qkv = static_cast<const T *>(b.qkv) + (size_t)s.row0 * (b.n_heads + 2 * b.n_kv) * D;
    p.out = static_cast<T *>(b.out) + (size_t)s.row0 * b.n_heads * D;
    p.start = s.start;
    p.T = s.T;
    if constexpr (is_paged<P>) {
        p.table = b.table + (size_t)s.slot * b.width;
        p.n_pages = b.n_pages;
    } else {
        const size_t cache = (size_t)s.slot * b.n_kv * b.capacity * D;
        p.k_cache = static_cast<T *>(b.k_cache) + cache;
        p.v_cache = static_cast<T *>(b.v_cache) + cache;
    }
    return p;
}

// one CTA per row of every segment (first[i] = row0_i)
template <typename T, int D, typename P>
__global__ void __launch_bounds__(APPEND_THREADS) attn_append_batch_kernel(const ExtBatchParams b) {
    const ExtSegment s = b.seg[segment_of(b, blockIdx.x)];
    append_body<T, D>(segment_params<T, D, P>(b, s), (int)blockIdx.x - s.row0);
}

// grid (S, the launch's tiles, n_kv): the segments of one split S, each segment's tiles last-first from first[i] on
template <typename T, int D>
__global__ void __launch_bounds__(XTHREADS, 1) attn_extend_batch_kernel(const ExtBatchParams b) {
    const int i = segment_of(b, blockIdx.y);
    const ExtParams p = segment_params<T, D, ExtParams>(b, b.seg[i]);
    constexpr bool PAGED = false;
    const Pages pg{};
    const int tile = (p.T * p.g + BM - 1) / BM - 1 - ((int)blockIdx.y - b.first[i]);
#include "attn_extend_tile.inc"
}

template <typename T, int D>
__global__ void __launch_bounds__(XTHREADS, 1) attn_extend_batch_paged_kernel(const ExtBatchParams b) {
    const int i = segment_of(b, blockIdx.y);
    const ExtPagedParams p = segment_params<T, D, ExtPagedParams>(b, b.seg[i]);
    constexpr bool PAGED = true;
    const Pages pg{p.table, p.n_pages};
    const int tile = (p.T * p.g + BM - 1) / BM - 1 - ((int)blockIdx.y - b.first[i]);
#include "attn_extend_tile.inc"
}

}  // namespace attn
}  // namespace
