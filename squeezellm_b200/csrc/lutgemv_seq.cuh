// lutgemv_seq.cuh - the SEQUENCE kernel: one persistent launch runs a whole list of dependent LUT-GEMVs (a decode token's QuantLinear
// matvecs: llama.py:226-234 calls them one by one, 224 launches per LLaMA-7B token).  Built on lutgemv_v2.cuh:
// the per-position math, table builders, outlier warps (sparse3), mailboxes, CTA span (Span) and strip flush (flush_strip) are v2's
// (namespace v2), and so are the texts of the warp roles' per-segment work: the producer's stream of a segment (lutgemv_stream.inc),
// the builders' loop (lutgemv_tables.inc) and finishing pass (lutgemv_finish.inc), and the consumers' segment (lutgemv_segment.inc),
// here with C2's 32-unit stages.  What is new is everything BETWEEN two GEMVs.
//
// Why: with one launch per GEMV (v2 + PDL + CUDA graph) a 4096x4096 layer takes several times its HBM time in the chain: every launch
// carries a fixed cost (CTA exit -> grid completion -> dependency release -> CTA start, barrier init, tensor
// map fetch, x staging, ring fill from cold) - 128 launches per token.  Here
//   * grid = #SMs, launched ONCE per token; every CTA walks the same list of GEMV descriptors (global memory, written at create time);
//   * the TMA producer warp never stops at a GEMV boundary: while the consumers finish GEMV g and wait for its result, the ring already
//     holds the first 128 KB per SM of GEMV g+1 - weights do not depend on activations;
//   * the dependency itself is data flow, not a grid-wide event: y is written as SELF-VALIDATING 32-bit words {16-bit value, 16-bit tag
//     of the token} (single-copy atomic: no fence, no flag, no second round trip), the consumers of the next GEMV poll the words of their
//     x straight out of L2 and repack the values in shared memory.  The value is the sequence's activation type (fp16 or bf16: the XT
//     template parameter); only the word's maker converts, everything else moves bits.  A stale word carries the previous token's tag,
//     so nothing is ever reset.  The cross-CTA mailboxes of v2 carry a (token, GEMV) tag the same way.
//   * on several GPUs (column shards) the owner of a strip stores its tagged words into EVERY rank's arena over NVLink; the poll of the
//     next GEMV is the whole exchange - no collective, no flag round trip (v2's exchange waits on a system-scope flag per launch).
#pragma once
#include "common.cuh"
#include "lutgemv_v2.cuh"

namespace {

namespace seq {
using namespace v2;

struct alignas(128) SeqDesc {
    CUtensorMap tm_big, tm_small;   // 64 columns x (32 units | 2 units) boxes over the packed matrix
    P2 p;                           // the GEMV: buffers, stream-K plan, workspace pointers (accumulator / flags alternate by GEMV parity)
    const uint32_t *x_tag;          // first tagged word of x in the local arena; null: p.x is a plain 16-bit vector (the token's input)
    unsigned long long y_off;       // byte offset of this GEMV's tagged output vector in every rank's arena
};
struct SeqExport {
    const uint32_t *src;            // tagged words in the local arena
    void *dst;                      // plain 16-bit vector (the sequence's activation type)
    int n;
};
// What an item of an OPS instance does besides its matvec (sqllm_sequence_create_ops), one per item in a parallel array: a transform
// of the staged x (RMSNorm, or SiLU gating with a second polled slice) and a residual added to the output inside its one rounding.
enum : int { SEQ_X_PLAIN = 0, SEQ_X_RMSNORM = 1, SEQ_X_SILU_MUL = 2 };
struct SeqOp {
    const void *gamma;              // RMSNorm: weight [K] of XT
    const uint32_t *x2_tag;         // SiLU gating: first tagged word of the up slice in the local arena (x is the gate)
    const uint32_t *res_tag;        // residual: first tagged word of an earlier item's full-length vector in the local arena, or null
    const void *res_ext;            // ... or a plain XT vector of the item's full output length, or null
    float eps;
    int x_op;                       // SEQ_X_*
};
struct SeqCfg {
    const SeqDesc *descs;
    int ngemv;
    const unsigned *epoch;          // token counter (bumped by a one-thread kernel before every launch)
    int *err;                       // a bounded wait gave up
    unsigned smem_raw;
    int xbytes, nstage;
    int world, rank;
    const unsigned long long *peer_base;  // arena base address of every rank (world > 1)
    unsigned long long arena_base;        // ... and our own
    const SeqExport *exports;
    int nexport;
    const SeqOp *ops;               // [ngemv]: read by the OPS instances only
};

__global__ void seq_bump_epoch(unsigned *epoch) { *epoch = *epoch + 1u; }

__device__ __forceinline__ void bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
template <bool SYS>
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint32_t *p) {
    uint4 v;
    if constexpr (SYS) asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned short bits16(const __half v) { return __half_as_ushort(v); }
__device__ __forceinline__ unsigned short bits16(const __nv_bfloat16 v) { return __bfloat16_as_ushort(v); }
__device__ __forceinline__ bool tags_ok(const uint4 w, const uint32_t want) {
    return (((w.x ^ want) | (w.y ^ want) | (w.z ^ want) | (w.w ^ want)) >> 16) == 0u;
}
// Four tagged words (16 bytes) at a time, up to four pieces per thread in flight; a piece that is not there yet is simply read again
// (bounded: 2 s, then the error word).  Returns through `sink(piece index, lo, hi)`: two packed pairs of 16-bit values.
template <bool SYS, typename F>
__device__ __forceinline__ void poll_tagged(const uint32_t *src, const int n4, const int tid, const int nthr, const uint32_t want, int *err, F sink) {
    for (int i0 = tid; i0 < n4; i0 += 4 * nthr) {
        uint4 w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (i0 + j * nthr < n4) w[j] = ld_relaxed_v4<SYS>(src + 4 * (size_t)(i0 + j * nthr));
        unsigned long long t0 = 0ull, t1;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int i = i0 + j * nthr;
            if (i < n4) {
                while (!tags_ok(w[j], want)) {
                    w[j] = ld_relaxed_v4<SYS>(src + 4 * (size_t)i);
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                    if (t0 == 0ull) t0 = t1;
                    if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile int *>(err) = 1; break; }
                }
                sink(i, __byte_perm(w[j].x, w[j].y, 0x5410), __byte_perm(w[j].z, w[j].w, 0x5410));
            }
        }
    }
}

// ---- the OPS instances' extras ----
template <bool SYS>
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t *p) {
    uint32_t v;
    if constexpr (SYS) asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
template <typename XT>
__device__ __forceinline__ uint32_t f32x2_to_xt2(float lo, float hi) {
    return (uint32_t)bits16(f32_to<XT>(lo)) | ((uint32_t)bits16(f32_to<XT>(hi)) << 16);
}
// silu(g) u on two packed pairs, in fp32 (silu(g) = g / (1 + e^-g): -0 for g -> -inf, g for g -> +inf), one rounding to XT per value
template <typename XT>
__device__ __forceinline__ uint32_t silu_mul2(uint32_t g2, uint32_t u2) {
    const float2 g = x16x2_to_f32x2<XT>(g2), u = x16x2_to_f32x2<XT>(u2);
    return f32x2_to_xt2<XT>(g.x / (1.f + expf(-g.x)) * u.x, g.y / (1.f + expf(-g.y)) * u.y);
}
// RMSNorm of the staged x in place, by the NCT consumer threads (x complete in shared memory, and again at the end for the caller's
// barrier): S = sum x_k^2 in fp32 in an order fixed by the thread layout alone - thread t takes the 8-element pieces t, t + NCT, ...
// one fma after the other, the warp adds its lanes by the fixed xor tree, every thread adds the 16 warp sums 0..15 from `scratch` - so
// every CTA holds the same bits; r = 1 / sqrt(S / K + eps); x'_k = round_XT(gamma_k (x_k r)).  (HF's LlamaRMSNorm rounds twice:
// (x r).to(dtype), then gamma times that; here x r stays in fp32 and only the product with gamma is rounded.)
template <typename XT>
__device__ __forceinline__ void rmsnorm_x(uint32_t xs, int K, const XT *gamma, float eps, uint32_t scratch, int tid) {
    const int n8 = K / 8;
    float s = 0.f;
    for (int e = tid; e < n8; e += NCT) {
        uint32_t w[4];
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(xs + 16u * (uint32_t)e));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = x16x2_to_f32x2<XT>(w[j]);
            s = fmaf(f.x, f.x, s);
            s = fmaf(f.y, f.y, s);
        }
    }
    s = warp_sum(s);
    if ((tid & 31) == 0) sts_u32(scratch + 4u * (uint32_t)(tid >> 5), __float_as_uint(s));
    named_bar_sync(1, NCT);
    float S = 0.f;
#pragma unroll
    for (int w = 0; w < NWC; ++w) S += lds_f32(scratch + 4u * w);
    const float r = 1.f / sqrtf(S / (float)K + eps);
    for (int e = tid; e < n8; e += NCT) {
        uint32_t w[4];
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(xs + 16u * (uint32_t)e));
        const uint4 gw = __ldg(reinterpret_cast<const uint4 *>(gamma) + e);
        const uint32_t gg[4] = {gw.x, gw.y, gw.z, gw.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = x16x2_to_f32x2<XT>(w[j]), g = x16x2_to_f32x2<XT>(gg[j]);
            w[j] = f32x2_to_xt2<XT>(g.x * (f.x * r), g.y * (f.y * r));
        }
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(xs + 16u * (uint32_t)e), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
    }
}


// XT: the sequence's 16-bit activation type (__half or __nv_bfloat16): the type of x_ext, of the value half of every tagged word, of
// the items' plain y copies and of the exports.  The poll, the staging and the exports only move bits; a word is made in store_y.
// OPS: the instance that also runs every item's SeqOp (c.ops): RMSNorm or SiLU gating of the staged x before barrier 2, a residual in
// store_y.  The instances without it never read c.ops.
template <int BITS, int MODE, bool MULTI, typename XT = __half, bool OPS = false>
__global__ void __launch_bounds__(THREADS2, 1) lutgemv_seq_kernel(const SeqCfg c) {
    using C = C2<BITS, MODE>;
    static_assert(std::is_same<XT, __half>::value || std::is_same<XT, __nv_bfloat16>::value, "x is fp16 or bf16");
    static_assert(MODE == 0 || std::is_same<XT, __half>::value, "the pair table multiplies fp16 by fp16: it needs fp16 x");
    constexpr int NTB = C::NTB;
    constexpr int TFREE = 288;   // tfree[b] at bar_u32 + TFREE + 8b (after up to four tfull barriers)
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    if (raw != c.smem_raw) __trap();
    uint32_t base = (raw + 127u) & ~127u;
    asm volatile("mov.u32 %0, %0;" : "+r"(base));
    unsigned char *sm = smem_raw + (base - raw);
    const uint32_t bar_u32 = base + OFF_BAR;   // full[s] +8s, empty[s] +128+8s, tfull[b] +256+8b, tfree[b] +288+8b
    const uint32_t xs_u32 = base + OFF_X;
    const uint32_t sacc0 = xs_u32 + (uint32_t)c.xbytes;                 // float [NTB][64]
    const int nstage = c.nstage;
    const Carve cv(base, (uint32_t)c.xbytes, NTB * STRIP * 4, C::TAB, NTB, C::STAGE, nstage);
    const uint32_t lo_base = cv.lo_base, tab0 = cv.tab0, hi_base = cv.hi_base;
    const int n_lo = cv.n_lo;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < nstage; ++s) {
            mbar_init(bar_u32 + 8 * s, 1);
            mbar_init(bar_u32 + 128 + 8 * s, NWC);
        }
        for (int b = 0; b < NTB; ++b) {
            mbar_init(bar_u32 + 256 + 8 * b, NBW);
            mbar_init(bar_u32 + TFREE + 8 * b, NWC);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t epoch = *reinterpret_cast<const volatile unsigned *>(c.epoch);
    const uint32_t xtag = (epoch & 0x7fffu) | 0x8000u;   // 16-bit tag of this token's activation words
    const uint32_t xwant = xtag << 16;
    const int ngemv = c.ngemv;

    if (warp == WARP_PROD) {
        // =========================== TMA producer: runs ahead of the consumers across GEMV boundaries ===========================
        const uint64_t pol = l2_evict_first_policy();
        int slot = 0;
        uint32_t ph = 0;
        bool refill = false;
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[0].tm_big)) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[0].tm_small)) : "memory");
        }
        for (int g = 0; g < ngemv; ++g) {
            const SeqDesc &d = c.descs[g];
            const P2 &p = d.p;
            const int N = p.N, R = p.R;
            const Span sp(p);
            if (lane == 0 && g + 1 < ngemv) {
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[g + 1].tm_big)) : "memory");
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[g + 1].tm_small)) : "memory");
            }
            warm_l2<BITS>(p, N, lane);  // (cold otherwise: a token never finds them in L2)
            const int len = sp.len, s0 = sp.s0, r0 = sp.r0;
            for (int seg = 0; seg < sp.nseg; ++seg) {
                // (inside the loop: taken ahead of it, the descriptor's address is computed before the nseg test; C2 has no mid box)
                const CUtensorMap *const tmap_big = &d.tm_big, *const tmap_small = &d.tm_small, *const tmap_mid = nullptr;
#include "lutgemv_stream.inc"
            }
        }
    } else if (warp >= WARP_SP) {
        // =========================== outlier warps (v2::sparse3, once per GEMV) ===========================
        for (int g = 0; g < ngemv; ++g) {
            const P2 &p = c.descs[g].p;
            sparse3<XT, true>(p, base, warp - WARP_SP, lane, nullptr, (epoch << 10) | (uint32_t)(g + 1));
            TRACE(10, lane == 0);
            if (g + 1 < ngemv) bar_arrive(6, NCT + NSPW * 32);  // done reading this GEMV's x from shared memory
        }
    } else if (warp >= WARP_BLD) {
        // =========================== table builders + strip finishers (2 warps, thread = column slot) ===========================
        const int bt = tid - WARP_BLD * 32;
        const uint32_t lutbuf = base + OFF_LUT;
#pragma unroll
        for (int b = 0; b < NTB; ++b) sts_u32(sacc0 + 4 * (b * STRIP + bt), 0u);
        int q0 = 0;  // segments of earlier GEMVs: segment s of this one uses table buffer / accumulator (q0 + s) % NTB
        auto tab_of = [&](int s) { return (q0 + s) % NTB; };
        auto prefetch_first = [&](const P2 &p) {  // the raw LUT rows of a GEMV's first two strips
            const Span sp(p);
            if (sp.nseg > 0) lut_prefetch<BITS>(p, lutbuf, sp.s0, bt);
            if (sp.nseg > 1) lut_prefetch<BITS>(p, lutbuf + LUTBUF, sp.s0 + 1, bt);
        };
        prefetch_first(c.descs[0].p);
        for (int g = 0; g < ngemv; ++g) {
            const SeqDesc &d = c.descs[g];
            const P2 &p = d.p;
            const int N = p.N, R = p.R;
            const Span sp(p);
            const int s0 = sp.s0, r0 = sp.r0, nseg = sp.nseg;
            const uint32_t boxtag = (epoch << 10) | (uint32_t)(g + 1);
            float *const acc_out = p.ws_acc;
            auto sacc_of = [&](int s) { return sacc0 + 4u * (uint32_t)(tab_of(s) * STRIP + bt); };
            auto tfree_wait = [&](int s) { mbar_wait(bar_u32 + TFREE + 8 * tab_of(s), (uint32_t)(((q0 + s) / NTB) & 1)); };
            auto reuse_wait = [&](int s) { tfree_wait(s - NTB); };
            const uint32_t sown = base + OFF_FIN;   // float [SOWN][64]
            const int ofs = r0 != 0 ? 1 : 0;        // segment s is owned strip s - ofs
            auto flush = [&](int s) { flush_strip<true>(p, sacc_of(s), s, ofs, sp, N, base, bt, acc_out, boxtag); };
#include "lutgemv_tables.inc"
            if (g + 1 < ngemv) prefetch_first(c.descs[g + 1].p);  // the next GEMV's rows travel while this one is being finished
            // the finishing pass (lutgemv_finish.inc): mailbox words are never reset (a stale word carries an older tag); y is a tagged
            // word in every rank's arena, and a plain XT copy if the item has one
            constexpr bool box_keep = true;
            auto err_word = [&]() { return c.err; };
            // OPS residual: one word per owned column, issued with the mailbox words (res_load).  An external vector's element is given
            // the token's tag here; an earlier item's word is taken like x (read again until it carries the tag, bounded).  Column col
            // reads the element of the full-length vector that store_y writes: col on one GPU, e below on several.
            const uint32_t *res_tag = nullptr;
            const XT *res_ext = nullptr;
            auto res_index = [&](int col) -> unsigned {
                if constexpr (!MULTI) return (unsigned)col;
                const int wm = N / p.xw_members, mm = col / wm;
                return (unsigned)(mm * p.xw_nfull + c.rank * wm + (col - mm * wm));
            };
            auto res_word = [&](int col) -> uint32_t {
                if (res_tag) return ld_relaxed_u32<MULTI>(res_tag + res_index(col));
                if (res_ext) return xwant | (uint32_t)bits16(res_ext[res_index(col)]);
                return 0u;
            };
            auto res_load = [&](uint32_t *rw, uint32_t &rlast, const int so0, const int nown, const int lidx) {
                if constexpr (OPS) {
                    res_tag = c.ops[g].res_tag;
                    res_ext = static_cast<const XT *>(c.ops[g].res_ext);
                    if (res_tag || res_ext) {
#pragma unroll
                        for (int u = 0; u < FAST; ++u) {
                            const int col = (so0 + u) * STRIP + bt;
                            rw[u] = u < nown && u != lidx && col < N ? res_word(col) : 0u;   // (the last owned strip's word: rlast)
                        }
                        const int lcol = (so0 + lidx) * STRIP + bt;
                        if (lidx >= 0 && lcol < N) rlast = res_word(lcol);
                    }
                } else {
                    for (int u = 0; u < FAST; ++u) rw[u] = 0u;
                }
            };
            auto make_store_y = [&]() {
                const int w = MULTI ? N / p.xw_members : 0;
                return [&, w](int col, float yv, uint32_t rword) {
                    if (p.bias) yv += __ldg(p.bias + col);
                    if constexpr (OPS) {
                        if (res_tag || res_ext) {  // y = round_XT(sum + bias + r): the residual too is inside the one rounding
                            if ((rword ^ xwant) >> 16) {
                                const uint32_t *const src = res_tag + res_index(col);
                                unsigned long long t0, t1;
                                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
                                do {
                                    rword = ld_relaxed_u32<MULTI>(src);
                                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                                    if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile int *>(c.err) = 1; break; }
                                } while ((rword ^ xwant) >> 16);
                            }
                            yv += x16x2_to_f32x2<XT>(rword & 0xFFFFu).x;
                        }
                    }
                    const XT yh = f32_to<XT>(yv);   // the one rounding: the bias is inside the fp32 sum
                    const uint32_t word = (xtag << 16) | (uint32_t)bits16(yh);
                    if constexpr (!MULTI) {
                        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(c.arena_base + d.y_off + 4ull * (unsigned)col), "r"(word) : "memory");
                    } else {
                        // local column col of the stacked shard = column j of member m -> element [m][rank*w + j] of the full-length vector, in EVERY rank's arena
                        const int mm = col / w, j = col - mm * w;
                        const unsigned long long e = (unsigned long long)mm * p.xw_nfull + (unsigned long long)c.rank * w + j;
                        for (int pr = 0; pr < c.world; ++pr)
                            asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(__ldg(c.peer_base + pr) + d.y_off + 4ull * e), "r"(word) : "memory");
                    }
                    // (the same value as yh, converted again as before bf16 existed: reusing yh reschedules the fp16 MULTI instantiations)
                    if (p.out) reinterpret_cast<XT *>(p.out)[col] = f32_to<XT>(yv);
                };
            };
#include "lutgemv_finish.inc"
            TRACE(9, bt == 0);
            q0 += nseg;
        }
    } else {
        // =========================== consumers ===========================
        const int i16 = lane & 15, jsel = lane >> 4;
        Acc A;
#pragma unroll
        for (int t = 0; t < 4; ++t) A.a[t] = 0ull;
#pragma unroll
        for (int t = 0; t < 8; ++t) A.f[t] = 0.f;
        const uint32_t slotb[4] = {(uint32_t)((((0 ^ jsel) << 4) | i16) << 2), (uint32_t)((((1 ^ jsel) << 4) | i16) << 2),
                                   (uint32_t)((((2 ^ jsel) << 4) | i16) << 2), (uint32_t)((((3 ^ jsel) << 4) | i16) << 2)};
        const uint32_t lane_in_stage = (uint32_t)((2 * warp + jsel) * C::UNIT + i16 * 16);
        int slot = 0, q0 = 0;
        uint32_t par = 0;
        auto sacc_row = [&](int b) { return sacc0 + (uint32_t)(b * STRIP + 4 * i16) * 4u; };
        auto stage_of = [&](int sl) { return (sl < n_lo ? lo_base : hi_base) + sl * C::STAGE + lane_in_stage; };
        auto advance = [&]() { if (++slot == nstage) { slot = 0; par ^= 1u; } };
        for (int g = 0; g < ngemv; ++g) {
            const SeqDesc &d = c.descs[g];
            const P2 &p = d.p;
            const int R = p.R;
            const Span sp(p);
            const int len = sp.len, r0 = sp.r0;
            // (q0 by value: captured by reference, it changes the order in which q0, slot and par are promoted to registers, and with
            // it the register allocation)
            auto tab_of = [q0](int s) { return (q0 + s) % NTB; };
            auto tab_phase = [q0](int s) { return (uint32_t)(((q0 + s) / NTB) & 1); };
            TRACE(2, tid == 0);
            if (g > 0) named_bar_sync(6, NCT + NSPW * 32);  // every consumer warp and the outlier warps are done with the previous x
            if (d.x_tag == nullptr) {
                const int n16 = p.K * 2 / 16;
                for (int e = tid; e < n16; e += NCT) cp_async16(xs_u32 + 16 * e, reinterpret_cast<const unsigned char *>(p.x) + 16 * (size_t)e);
                cp_async_commit();
                cp_async_wait_all();
            } else {
                poll_tagged<MULTI>(d.x_tag, p.K / 4, tid, NCT, xwant, c.err, [&](int i, uint32_t lo, uint32_t hi) {
                    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(xs_u32 + 8u * (uint32_t)i), "r"(lo), "r"(hi) : "memory");
                });
            }
            if constexpr (OPS) {
                const SeqOp &o = c.ops[g];
                const int xop = o.x_op;
                if (xop != SEQ_X_PLAIN) {
                    named_bar_sync(1, NCT);  // the whole x is staged (a copied or polled piece may come from another thread)
                    if (xop == SEQ_X_RMSNORM) {
                        // scratch: the 16 warp sums in the fixed area's strip-sum rows, which only the one-GEMV kernel uses
                        rmsnorm_x<XT>(xs_u32, p.K, static_cast<const XT *>(o.gamma), o.eps, base + OFF_SACC, tid);
                    } else {
                        poll_tagged<MULTI>(o.x2_tag, p.K / 4, tid, NCT, xwant, c.err, [&](int i, uint32_t lo, uint32_t hi) {
                            const uint32_t a = xs_u32 + 8u * (uint32_t)i;
                            uint32_t g0, g1;
                            asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(g0), "=r"(g1) : "r"(a));
                            asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(silu_mul2<XT>(g0, lo)), "r"(silu_mul2<XT>(g1, hi)) : "memory");
                        });
                    }
                }
            }
            named_bar_sync(2, NCT + NSPW * 32);  // x visible to the consumers and the outlier warps
            TRACE(4, tid == 0);
            for (int seg = 0; seg < sp.nseg; ++seg) {
#include "lutgemv_segment.inc"
            }
            TRACE(6, tid == 0);
            q0 += sp.nseg;
        }
        // exports: plain 16-bit copies of the vectors the caller asked for (on several GPUs this is also where the last exchange completes)
        for (int e = (int)blockIdx.x; e < c.nexport; e += (int)gridDim.x) {
            const SeqExport ex = c.exports[e];
            poll_tagged<MULTI>(ex.src, ex.n / 4, tid, NCT, xwant, c.err, [&](int i, uint32_t lo, uint32_t hi) {
                *reinterpret_cast<uint2 *>(reinterpret_cast<unsigned char *>(ex.dst) + 8 * (size_t)i) = make_uint2(lo, hi);
            });
        }
    }
}

}  // namespace seq

}  // namespace
