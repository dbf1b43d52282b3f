// lutgemv_seq.cuh - the SEQUENCE kernel: one persistent launch runs a whole list of dependent LUT-GEMVs (a decode token's QuantLinear
// matvecs: llama.py:226-234 calls them one by one, 224 launches per LLaMA-7B token).  Built on lutgemv_v2.cuh:
// the per-position math, table builders, outlier warps (sparse3) and mailboxes are v2's (namespace v2), what is new is everything BETWEEN two GEMVs.
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
            mbar_init(bar_u32 + 288 + 8 * b, NWC);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t epoch = *reinterpret_cast<const volatile unsigned *>(c.epoch);
    const uint32_t xtag = (epoch & 0x7fffu) | 0x8000u;   // 16-bit tag of this token's activation words
    const uint32_t xwant = xtag << 16;
    const int ngemv = c.ngemv;

    // the CTA's part of GEMV `p`: units [g0, g0 + len) of the strip-major [strip][unit] space
#define SEQ_GEOMETRY(p)                                                                   \
    const int N = (p).N, R = (p).R;                                                       \
    const int g0 = min((int)blockIdx.x * (p).chunk, (p).T), g1 = min(g0 + (p).chunk, (p).T); \
    const int len = g1 - g0;                                                              \
    const int s0 = g0 / R, r0 = g0 - s0 * R;                                              \
    const int nseg = len > 0 ? (g1 - 1) / R - s0 + 1 : 0;                                 \
    (void)N; (void)r0; (void)s0; (void)nseg;

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
            SEQ_GEOMETRY(p)
            if (lane == 0 && g + 1 < ngemv) {
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[g + 1].tm_big)) : "memory");
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&c.descs[g + 1].tm_small)) : "memory");
            }
            {   // a 1/grid slice of the GEMV's look-up table and row pointers -> L2, for everybody (cold otherwise: a token never finds them there)
                const int G = (int)gridDim.x;
                const size_t lut_lines = ((size_t)N * C::L * 4 + 127) / 128, per = (lut_lines + G - 1) / G;
                for (size_t i = (size_t)blockIdx.x * per + lane; i < min(lut_lines, ((size_t)blockIdx.x + 1) * per); i += 32)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(p.lut) + 128 * i));
                if (p.rows) {
                    const size_t row_lines = ((size_t)(N + 1) * 4 + 127) / 128, rper = (row_lines + G - 1) / G;
                    for (size_t i = (size_t)blockIdx.x * rper + lane; i < min(row_lines, ((size_t)blockIdx.x + 1) * rper); i += 32)
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(p.rows) + 128 * i));
                }
            }
            for (int seg = 0; seg < nseg; ++seg) {
                const int sstart = seg == 0 ? 0 : seg * R - r0, send = min(len, (seg + 1) * R - r0);
                const int seglen = send - sstart;
                const int u0 = r0 + sstart - seg * R;
                const int col0 = (s0 + seg) * STRIP;
                for (int u = 0; u < seglen; u += SU2) {
                    if (refill) mbar_wait(bar_u32 + 128 + 8 * slot, ph);
                    const int nu = min(SU2, seglen - u);
                    const uint32_t full = bar_u32 + 8 * slot;
                    const uint32_t dst = (slot < n_lo ? lo_base : hi_base) + slot * C::STAGE;
                    const int row0 = (u0 + u) * C::ROWS;
                    if (lane == 0) mbar_expect_tx(full, (uint32_t)nu * C::UNIT);
                    __syncwarp();
                    if (nu == SU2) {
                        if (lane == 0) tma_tile2d_g2s(dst, &d.tm_big, col0, row0, full, pol);
                    } else if (2 * lane < nu) {
                        tma_tile2d_g2s(dst + lane * 2 * C::UNIT, &d.tm_small, col0, row0 + lane * 2 * C::ROWS, full, pol);
                    }
                    if (++slot == nstage) {
                        slot = 0;
                        if (refill) ph ^= 1u;
                        refill = true;
                    }
                }
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
        int *const err = c.err;
        int q0 = 0;  // segments of earlier GEMVs: segment s of this one uses table buffer / accumulator (q0 + s) % NTB
        {
            const P2 &p = c.descs[0].p;
            SEQ_GEOMETRY(p)
            if (nseg > 0) lut_prefetch<BITS>(p, lutbuf, s0, bt);
            if (nseg > 1) lut_prefetch<BITS>(p, lutbuf + LUTBUF, s0 + 1, bt);
        }
        for (int g = 0; g < ngemv; ++g) {
            const SeqDesc &d = c.descs[g];
            const P2 &p = d.p;
            SEQ_GEOMETRY(p)
            const uint32_t boxtag = (epoch << 10) | (uint32_t)(g + 1);
            float *const acc_out = p.ws_acc;
            int *const flags = p.ws_cnt + 64;
            auto sacc_of = [&](int s) { return sacc0 + 4u * (uint32_t)(((q0 + s) % NTB) * STRIP + bt); };
            auto tfree_wait = [&](int s) { mbar_wait(bar_u32 + 288 + 8 * ((q0 + s) % NTB), (uint32_t)(((q0 + s) / NTB) & 1)); };
            // Strip sums of segment s go to the strip's owner: another CTA (mailbox row) if the strip started before our range, else ourselves -
            // and then they never leave the SM: sown[u][column] for the u-th owned strip (a strip inside one CTA is exactly one segment).
            // (v2 and the first sequence build sent them through the global accumulator - a RED and, in the finishing pass, a load that has to
            // wait for it: L2 round trips on the critical path between the last weight and y.)
            const uint32_t sown = base + OFF_FIN;   // float [SOWN][64], as in lutgemv2_kernel
            constexpr int SOWN = 8;
            const int ofs = r0 != 0 ? 1 : 0;        // segment s is owned strip s - ofs
            auto flush = [&](int s) {
                const uint32_t a = sacc_of(s);
                const float v = lds_f32(a);
                sts_u32(a, 0u);
                const int col = (s0 + s) * STRIP + bt;
                if (s == 0 && r0 != 0) st_relaxed_u64(p.ws_hbox + (size_t)blockIdx.x * STRIP + bt, box_word(v, boxtag));
                else if (s - ofs < SOWN) sts_u32(sown + 4u * (uint32_t)((s - ofs) * STRIP + bt), __float_as_uint(v));
                else if (col < N) atomicAdd(acc_out + col, v);
            };
            for (int s = 0; s < nseg; ++s) {
                const int b = (q0 + s) % NTB;
                if (s >= NTB) {
                    tfree_wait(s - NTB);
                    flush(s - NTB);
                }
                if (s + 1 < nseg) cp_async_wait_pending<1>();
                else cp_async_wait_all();
                named_bar_sync(3, NBT);
                build_table<BITS, MODE>(tab0 + b * C::TAB, lutbuf + (s & 1) * LUTBUF, bt);
                named_bar_sync(3, NBT);
                if (lane == 0) mbar_arrive(bar_u32 + 256 + 8 * b);
                if (s + 2 < nseg) lut_prefetch<BITS>(p, lutbuf + (s & 1) * LUTBUF, s0 + s + 2, bt);
            }
            if (g + 1 < ngemv) {  // the next GEMV's first raw LUT rows travel while this one is being finished
                const P2 &pn = c.descs[g + 1].p;
                const int gn0 = min((int)blockIdx.x * pn.chunk, pn.T), gn1 = min(gn0 + pn.chunk, pn.T);
                const int sn0 = gn0 / pn.R, nsegn = gn1 > gn0 ? (gn1 - 1) / pn.R - sn0 + 1 : 0;
                if (nsegn > 0) lut_prefetch<BITS>(pn, lutbuf, sn0, bt);
                if (nsegn > 1) lut_prefetch<BITS>(pn, lutbuf + LUTBUF, sn0 + 1, bt);
            }
            // ---- finish the strips this CTA owns (those that start in its range); see lutgemv_v2.cuh for the protocol ----
            TRACE(12, bt == 0);
            const long long cb0 = (long long)blockIdx.x * p.chunk, cb1 = min((long long)p.T, cb0 + p.chunk);
            const int so0 = (int)((cb0 + R - 1) / R), so1 = (int)((cb1 + R - 1) / R), nown = so1 - so0;
            const bool last_owned = nseg >= 2 || r0 == 0;
            constexpr int FAST = 4;
            const int lidx = last_owned && nseg > 0 ? nown - 1 : -1;
            const int nh = lidx >= 0 ? (int)((((long long)(so1 - 1) + 1) * R - 1) / p.chunk) - (int)blockIdx.x : 0;
            // Dense rows whose channel lies in a strip we own: listed now (static), summed below.  sdj[i] = dense row, sden[i] = its sum.
            int *const sdj = reinterpret_cast<int *>(sm + OFF_FIN + 2048);
            const uint32_t sden = base + OFF_FIN + 2048 + 4 * 128, sdn_a = base + OFF_FIN + 2048 + 8 * 128;
            if (p.full_rows) {
                // (one warp, registers and shuffles: a serial scan of full_row_indices by one thread cost 435 dependent loads for the 30
                //  dense rows of a stacked q/k/v layer - on every CTA, before its first mailbox row went out)
                const int topX = p.topX;
                if (bt == 0) sts_u32(sdn_a, 0u);
                sts_u32(sden + 4 * bt, 0u);
                sts_u32(sden + 4 * (bt + NBT), 0u);
                named_bar_sync(3, NBT);
                if (topX <= 32) {
                    if (bt < 32) {
                        const int cc = bt < topX ? __ldg(p.fri + bt) : -1 - bt;
                        bool first = true;  // rows on the same channel were combined by the contributors: the first of them carries the sum
                        for (int j2 = 0; j2 < topX; ++j2) {
                            const int c2 = __shfl_sync(0xffffffffu, cc, j2);
                            if (c2 == cc && j2 < bt) first = false;
                        }
                        const bool mine = bt < topX && first && cc >= 0 && cc < N && cc / STRIP >= so0 && cc / STRIP < so1;
                        const unsigned m = __ballot_sync(0xffffffffu, mine);
                        if (mine) sdj[__popc(m & ((1u << bt) - 1u))] = bt;
                        if (bt == 0) sts_u32(sdn_a, (uint32_t)__popc(m));
                    }
                } else {
                    for (int j = bt; j < topX; j += NBT) {
                        const int cc = __ldg(p.fri + j);
                        if (cc >= 0 && cc < N && cc / STRIP >= so0 && cc / STRIP < so1) {
                            uint32_t at;
                            asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(at) : "r"(sdn_a) : "memory");
                            sdj[at] = j;
                        }
                    }
                }
                named_bar_sync(3, NBT);
            }
            const int sdn = p.full_rows ? (int)lds_u32(sdn_a) : 0;
            for (int s = max(0, nseg - NTB); s < nseg - 1; ++s) {
                tfree_wait(s);
                flush(s);
            }
            TRACE(13, bt == 0);
            {
                unsigned long long cw[FAST], hw[3];
#pragma unroll
                for (int u = 0; u < FAST; ++u) {
                    const int col = (so0 + u) * STRIP + bt;
                    cw[u] = (p.rows && u < nown && col < N) ? ld_relaxed_u64(p.ws_cbox + col) : box_word(0.f, boxtag);
                }
#pragma unroll
                for (int h = 0; h < 3; ++h)
                    hw[h] = h < nh ? ld_relaxed_u64(p.ws_hbox + ((size_t)blockIdx.x + 1 + h) * STRIP + bt) : box_word(0.f, boxtag);
                // OPS residual: one word per owned column, issued with the mailbox words.  An external vector's element is given the token's
                // tag here; an earlier item's word is taken like x (read again until it carries the tag, bounded).  Column col reads the
                // element of the full-length vector that store_y writes: col on one GPU, e below on several.
                const uint32_t *res_tag = nullptr;
                const XT *res_ext = nullptr;
                if constexpr (OPS) {
                    res_tag = c.ops[g].res_tag;
                    res_ext = static_cast<const XT *>(c.ops[g].res_ext);
                }
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
                uint32_t rw[FAST], rlast = 0u;
                if constexpr (OPS) {
                    if (res_tag || res_ext) {
#pragma unroll
                        for (int u = 0; u < FAST; ++u) {
                            const int col = (so0 + u) * STRIP + bt;
                            rw[u] = u < nown && u != lidx && col < N ? res_word(col) : 0u;   // (the last owned strip's word: rlast)
                        }
                        const int lcol = (so0 + lidx) * STRIP + bt;
                        if (lidx >= 0 && lcol < N) rlast = res_word(lcol);
                    }
                }
                // dense rows: hc tagged words per listed row (one from every contributing CTA), four loads in flight per thread; row sums are
                // collected in shared memory and added to the column they belong to by the thread that owns that column
                float last_dense = 0.f;
                if (sdn > 0) {
                    const int hc = p.hc;
                    unsigned long long *const dbox = p.ws_dbox;
                    for (int j0 = 0; j0 < sdn; j0 += 4) {  // four rows x up to four words per thread in flight (hc <= MAX_GRID_V2 = 4 x NBT)
                        unsigned long long dw[4][4];
                        int row[4];
#pragma unroll
                        for (int a = 0; a < 4; ++a) {
                            row[a] = j0 + a < sdn ? sdj[j0 + a] : -1;
#pragma unroll
                            for (int b = 0; b < 4; ++b)
                                if (row[a] >= 0 && bt + b * NBT < hc) dw[a][b] = ld_relaxed_u64(dbox + (size_t)row[a] * MAX_GRID_V2 + bt + b * NBT);
                        }
#pragma unroll
                        for (int a = 0; a < 4; ++a) {
                            if (row[a] < 0) continue;  // (uniform)
                            float v = 0.f;
#pragma unroll
                            for (int b = 0; b < 4; ++b)
                                if (bt + b * NBT < hc) v += box_take(dw[a][b], dbox + (size_t)row[a] * MAX_GRID_V2 + bt + b * NBT, err, boxtag, true);
                            v = warp_sum(v);
                            if (lane == 0) asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(sden + 4u * (uint32_t)(j0 + a)), "f"(v) : "memory");
                        }
                    }
                    named_bar_sync(3, NBT);
                    for (int i = 0; i < sdn; ++i) {
                        const int cc = __ldg(p.fri + sdj[i]);
                        if ((cc & (STRIP - 1)) == bt) {
                            const int u = cc / STRIP - so0;
                            const float v = lds_f32(sden + 4u * (uint32_t)i);
                            if (u == lidx) last_dense += v;
                            else if (u < SOWN) {
                                const uint32_t a = sown + 4u * (uint32_t)(u * STRIP + bt);
                                sts_u32(a, __float_as_uint(lds_f32(a) + v));
                            } else atomicAdd(acc_out + cc, v);
                        }
                    }
                    named_bar_sync(3, NBT);  // (the list and the sums are reused by the next item; an idle CTA has no other barrier before that)
                }
                const int w = MULTI ? N / p.xw_members : 0;
                auto store_y = [&](int col, float yv, uint32_t rword = 0u) {
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
                                    if (t1 - t0 > 2000000000ull) { *reinterpret_cast<volatile int *>(err) = 1; break; }
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
                // per owned strip but the last segment's: [our own sums (+ dense rows), from shared memory] + [the column's outlier sum]
                TRACE(14, bt == 0);
                float last_others = last_dense;
#pragma unroll
                for (int u = 0; u < FAST; ++u) {
                    const int col = (so0 + u) * STRIP + bt;
                    if (u < nown && col < N) {
                        float yv = 0.f;
                        if (u != lidx && u < SOWN) yv = lds_f32(sown + 4u * (uint32_t)(u * STRIP + bt));
                        if (p.rows) yv += box_take(cw[u], p.ws_cbox + col, err, boxtag, true);
                        if (u == lidx) last_others += yv;
                        else store_y(col, yv, OPS ? rw[u] : 0u);
                    }
                }
                for (int i = FAST; i < nown; ++i) {  // (more owned strips than FAST; beyond SOWN the sums went through the global accumulator)
                    const int col = (so0 + i) * STRIP + bt;
                    if (col < N) {
                        float yv = 0.f;
                        if (i >= SOWN) { yv = __ldcg(p.ws_acc + col); p.ws_acc[col] = 0.f; }
                        else if (i != lidx) yv = lds_f32(sown + 4u * (uint32_t)(i * STRIP + bt));
                        if (p.rows) yv += box_take(0ull, p.ws_cbox + col, err, boxtag, true);
                        if (i == lidx) last_others += yv;
                        else store_y(col, yv, OPS ? res_word(col) : 0u);
                    }
                }
                TRACE(15, bt == 0);
#pragma unroll
                for (int h = 0; h < 3; ++h)
                    if (h < nh) last_others += box_take(hw[h], p.ws_hbox + ((size_t)blockIdx.x + 1 + h) * STRIP + bt, err, boxtag, true);
                // (a strip that spans many CTAs - narrow column shards: 18 CTAs per strip for a 512-column shard of down_proj - has many such
                //  words: eight reads in flight, not one round trip after the other)
                for (int h0 = 3; h0 < nh; h0 += 8) {
                    unsigned long long mw[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (h0 + k < nh) mw[k] = ld_relaxed_u64(p.ws_hbox + ((size_t)blockIdx.x + 1 + h0 + k) * STRIP + bt);
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (h0 + k < nh) last_others += box_take(mw[k], p.ws_hbox + ((size_t)blockIdx.x + 1 + h0 + k) * STRIP + bt, err, boxtag, true);
                }
                TRACE(8, bt == 0);
                if (nseg > 0) {
                    const int s = nseg - 1;
                    tfree_wait(s);
                    if (last_owned) {
                        const uint32_t a = sacc_of(s);
                        const float own = lds_f32(a);
                        sts_u32(a, 0u);
                        const int lcol = (s0 + s) * STRIP + bt;
                        if (lcol < N) store_y(lcol, last_others + own, rlast);
                    } else {
                        flush(s);
                    }
                }
            }
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
        constexpr int XB = C::XU * 2;
        constexpr int XBS = SU2 * XB;
        int slot = 0, q0 = 0;
        uint32_t par = 0;
        auto stage_of = [&](int sl) { return (sl < n_lo ? lo_base : hi_base) + sl * C::STAGE + lane_in_stage; };
        auto advance = [&]() { if (++slot == nstage) { slot = 0; par ^= 1u; } };
        for (int g = 0; g < ngemv; ++g) {
            const SeqDesc &d = c.descs[g];
            const P2 &p = d.p;
            SEQ_GEOMETRY(p)
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
            for (int seg = 0; seg < nseg; ++seg) {
                const int q = q0 + seg, b = q % NTB;
                const uint32_t tab = tab0 + b * C::TAB;
                const uint32_t tb_hi = (MODE == 1 && BITS == 4) ? tab : (BITS == 4 ? (tab & 0xFFFF0000u) : tab);
                uint32_t l[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    l[t] = tb_hi | slotb[t];
                    asm volatile("mov.u32 %0, %0;" : "+r"(l[t]));
                }
                const uint32_t segc = ((tab >> 8) & 0xF0u) * 0x01010101u;
                const int sstart = seg == 0 ? 0 : seg * R - r0, send = min(len, (seg + 1) * R - r0);
                const int seglen = send - sstart;
                const int u0 = r0 + sstart - seg * R;
                uint32_t xaddr = xs_u32 + (uint32_t)((u0 + 2 * warp + jsel) * XB);
                const int nstg = (seglen + SU2 - 1) / SU2;
                const int mine = 2 * warp < seglen ? (seglen - 2 * warp + SU2 - 1) / SU2 : 0;
                mbar_wait(bar_u32 + 256 + 8 * b, (uint32_t)((q / NTB) & 1));
                TRACE(16 + (seg < 7 ? seg : 7), tid == 0);
                for (int k = 0; k < nstg; ++k) {
                    mbar_wait(bar_u32 + 8 * slot, par);
                    if (k < mine) {
                        Fetch<BITS, XT> F;
                        fetch2<BITS, XT>(F, stage_of(slot), xaddr);
                        math2<BITS, MODE, XT>(F, jsel, l, segc, xaddr, A);
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_u32 + 128 + 8 * slot);
                    advance();
                    xaddr += XBS;
                }
                {
                    float s[4];
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        s[t] = MODE == 0 ? sum2(A.a[t]) : A.f[t] + A.f[t + 4];
                        A.a[t] = 0ull;
                        A.f[t] = 0.f;
                        A.f[t + 4] = 0.f;
                    }
                    const float v0 = __shfl_xor_sync(0xffffffffu, s[1], 16);
                    const float v1 = __shfl_xor_sync(0xffffffffu, s[0], 16);
                    const float v2 = __shfl_xor_sync(0xffffffffu, s[3], 16);
                    const float v3 = __shfl_xor_sync(0xffffffffu, s[2], 16);
                    if (jsel == 0 && mine > 0) {
                        const uint32_t a = sacc0 + (uint32_t)(b * STRIP + 4 * i16) * 4u;
                        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a), "f"(s[0] + v0) : "memory");
                        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a + 4), "f"(s[1] + v1) : "memory");
                        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a + 8), "f"(s[2] + v2) : "memory");
                        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a + 12), "f"(s[3] + v3) : "memory");
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_u32 + 288 + 8 * b);
                }
                TRACE(24 + (seg < 7 ? seg : 7), tid == 0);
            }
            TRACE(6, tid == 0);
            q0 += nseg;
        }
        // exports: plain 16-bit copies of the vectors the caller asked for (on several GPUs this is also where the last exchange completes)
        for (int e = (int)blockIdx.x; e < c.nexport; e += (int)gridDim.x) {
            const SeqExport ex = c.exports[e];
            poll_tagged<MULTI>(ex.src, ex.n / 4, tid, NCT, xwant, c.err, [&](int i, uint32_t lo, uint32_t hi) {
                *reinterpret_cast<uint2 *>(reinterpret_cast<unsigned char *>(ex.dst) + 8 * (size_t)i) = make_uint2(lo, hi);
            });
        }
    }
#undef SEQ_GEOMETRY
}

}  // namespace seq

}  // namespace
