// lutgemv.cu - H100 (sm_90a) dense-and-sparse LUT GEMV, written from scratch: the one-vector GEMVs with their plans and launches,
// the sequence objects, the workspace symbols and the 12 launchers of the reference.
//
// Replaces (behaviour, not code) squeezellm/quant_cuda_kernel.cu of SqueezeAILab/SqueezeLLM:
//   VecQuant{3,4}MatMulKernelNUQPerChannel[Batched]  (:741-1038)   LUT GEMV
//   SPMV_ATOMIC[_BATCHED]                            (:1040-1089)  CSR outliers
//   DenseMatVecKernel[Batched]                       (:1092-1164)  topX dense rows
// and the 12 host launchers (:132-738), behind the C ABI of include/sqllm_b200.h.
//
// lutgemv2_kernel (lutgemv_v2.cuh) runs every one-vector GEMV in the accumulate and the default (fast) fused mode, the sequence
// kernel (lutgemv_seq.cuh) a list of dependent GEMVs in one persistent launch, and lutgemv_kernel (lutgemv_v1.cuh) the deterministic
// fused mode.  The other kernel families have translation units of their own: lutgemv_rows.cu (the batched symbols and a few
// fp16 / bf16 rows on the CUDA cores), lutgemm_tc.cu (prefill-sized batches on the tensor cores), backward.cu (input and codebook
// gradients, Fisher information) and tools.cu (dequantize, k-means, pack); host.cu holds the process-wide state.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <unordered_map>
#include <vector>

#include "host.h"
#include "lutgemv_seq.cuh"
#include "lutgemv_v1.cuh"

using namespace sqllm;

namespace {

// shared-window address at which a kernel without static shared memory sees its dynamic shared memory (the v2 carve-up aligns
// tables to their own size - up to 64 KB - so the host needs the real address, not a worst case; the kernel re-checks it)
__global__ void smem_base_probe(unsigned *out) {
    extern __shared__ unsigned char probe_smem[];
    *out = smem_u32(probe_smem);
}

// the (x, y) dtype pairs of the one-GEMV entry points (sqllm_lutgemv_fused_dt, sqllm_lutgemv_fused_exchange_dt): y is fp32 or the
// 16-bit type of x, and that is fp16 for fp32 x
bool fused_dt_pair(int x_dt, int y_dt) {
    const int y16 = x_dt == SQLLM_DT_BF16 ? SQLLM_DT_BF16 : SQLLM_DT_F16;
    return dt_valid(x_dt) && (y_dt == SQLLM_DT_F32 || y_dt == y16);
}
int fused_dt_fail(int x_dt, int y_dt) {
    return fail(SQLLM_EINVAL, "x_dtype=%d, y_dtype=%d: x must be SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16, y SQLLM_DT_F32 or the "
                              "16-bit type of x (SQLLM_DT_F16 for fp32 x)", x_dt, y_dt);
}

struct Plan {
    int R, strips, T, chunk, G, maxc, hc, hrows, smem, maxseg, x_direct, xfloats;
    size_t ws_cnt_off, ws_hyb_off, ws_part_off, ws_csr_off, ws_bytes;
    int csr_rpc, has_stage;
};

// stage: bytes of the shared-memory staging buffer when the layer has CSR outliers or dense rows: STAGE for a launch (smaller only
// in sqllm_workspace_bytes)
int make_plan(int bits, int K, int N, int topX, bool has_csr_in, int stage, Plan &pl) {
    std::lock_guard<std::recursive_mutex> state_lock(g_state_mu);  // lazily initialised statics below
    const bool has_csr = has_csr_in || topX > 0;  // from here on: "a staging buffer is needed"
    pl.has_stage = has_csr ? stage : 0;
    int sm = 0;
    const int rc = dev_setup({{lutgemv_kernel<4>, 227 * 1024}, {lutgemv_kernel<3>, 227 * 1024}}, &sm);
    if (rc) return rc;
    const int XU = bits == 4 ? 8 : 32;
    pl.R = bits == 4 ? K / 8 : K / 32;
    pl.strips = (N + STRIP - 1) / STRIP;
    const long long T = (long long)pl.strips * pl.R;
    if (T > 0x3fffffff) return fail(SQLLM_EINVAL, "problem too large");
    pl.T = (int)T;
    if (pl.strips > MAX_STRIPS || N > MAX_N_FUSED) return fail(SQLLM_EINVAL, "out_features=%d exceeds the workspace header (max %d)", N, MAX_N_FUSED);

    // One wave: a plan whose shared memory lets fewer than CTAS_PER_SM CTAs onto an SM would run a second one.  Plan for
    // CTAS_PER_SM, ask the occupancy calculator, and fall back to fewer CTAs per SM if it disagrees.
    int use_cps = CTAS_PER_SM;
replan:
    const int G0 = sm * use_cps;
    int chunk = (int)(2 * ((T + 2LL * G0 - 1) / (2LL * G0)));  // an even number of units: a consumer warp's pair never straddles the end
    if (chunk > 3 * pl.R) chunk = 3 * pl.R;  // a CTA may touch at most MAXSEG strips
    if (chunk < 2) chunk = 2;
    int maxseg = (chunk - 2) / pl.R + 2;      // worst case over start offsets (even offsets, even R)
    if (maxseg > MAXSEG) maxseg = MAXSEG;
    const bool direct = (long long)chunk * XU >= K;
    const int xfl = direct ? K : chunk * XU;
    pl.x_direct = direct ? 1 : 0;
    const int smem = bits == 4 ? Cfg<4>::total(maxseg, xfl, pl.has_stage) : Cfg<3>::total(maxseg, xfl, pl.has_stage);
    if (smem > 227 * 1024) return fail(SQLLM_EINVAL, "in_features=%d needs %d B of shared memory (> 227 KB)", K, smem);
    {
        static std::unordered_map<unsigned long long, int> occ_cache;
        const unsigned long long key = ((unsigned long long)smem << 8) | (unsigned long long)bits;
        int occ = -1;
        auto it = occ_cache.find(key);
        if (it != occ_cache.end()) occ = it->second;
        if (occ < 0) {
            const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bits == 4 ? lutgemv_kernel<4> : lutgemv_kernel<3>, THREADS, smem);
            if (e != cudaSuccess) return fail(SQLLM_ECUDA, "occupancy query failed: %s", cudaGetErrorString(e));
            occ_cache[key] = occ;
        }
        if (occ < 1) return fail(SQLLM_EINVAL, "kernel does not fit an SM (shared memory %d B)", smem);
        if (occ < use_cps) { use_cps = occ; goto replan; }
    }
    pl.smem = smem;
    pl.maxseg = maxseg;
    pl.xfloats = xfl;
    pl.chunk = chunk;
    pl.G = (int)((T + chunk - 1) / chunk);
    pl.maxc = (pl.R - 1) / chunk + 2;
    pl.hc = 0;
    pl.hrows = 0;
    int hc = 0;
    if (topX > 0) {
        // dense-row contributors: as few k-rows per CTA as the grid allows, down to what one warp requests before the dependency
        // wait (HYB_R steps of 32/topX rows), and no more partials (hc*topX floats) than the 2*CSR_CH-float staging buffer of the
        // finisher holds
        const int rows_pre = HYB_R * (topX <= 32 ? 32 / topX : 1);
        hc = std::min({pl.G, (K + rows_pre - 1) / rows_pre, 2 * CSR_CH / topX});
        if (hc < 1) hc = 1;
        pl.hrows = (K + hc - 1) / hc;
        pl.hc = (K + pl.hrows - 1) / pl.hrows;
    }
    pl.csr_rpc = (N + pl.G - 1) / pl.G;
    if (pl.csr_rpc < 1) pl.csr_rpc = 1;
    // Fixed header: [256, 256+4*MAX_STRIPS) per-strip tickets.  Tickets must never share bytes with data regions of ANY shape
    // (the workspace is reused across layers of different sizes).
    size_t off = WS_HEADER;
    pl.ws_cnt_off = 256;
    pl.ws_hyb_off = off; off += (size_t)hc * topX * 4;
    off = (off + 255) & ~(size_t)255;
    pl.ws_part_off = off; off += (size_t)pl.strips * pl.maxc * STRIP * 4;
    off = (off + 255) & ~(size_t)255;
    pl.ws_csr_off = off; off += (size_t)N * 4;
    pl.ws_bytes = off;
    return SQLLM_OK;
}

int launch(const sqllm_lutgemv_args *a, const Plan &pl, Params &p, cudaStream_t st) {
    std::lock_guard<std::recursive_mutex> state_lock(g_state_mu);
    set_layer(p, *a);
    p.K = a->in_features; p.N = a->out_features;
    p.R = pl.R; p.strips = pl.strips; p.T = pl.T; p.chunk = pl.chunk;
    p.maxseg = pl.maxseg; p.x_direct = pl.x_direct; p.xfloats = pl.xfloats;
    p.hc = p.topX > 0 ? pl.hc : 0; p.hrows = pl.hrows; p.maxc = pl.maxc;
    p.has_stage = pl.has_stage;
    p.csr_rpc = pl.csr_rpc;
    p.csr_al16 = (a->rows && ((reinterpret_cast<uintptr_t>(a->cols) | reinterpret_cast<uintptr_t>(a->vals)) & 15) == 0) ? 1 : 0;
    p.trace = g_trace;
    if (g_trace) g_trace += g_trace_stride;
    g_last_grid = pl.G;
    const cudaError_t e = launch_ex(a->bits == 4 ? lutgemv_kernel<4> : lutgemv_kernel<3>, pl.G, THREADS, pl.smem, st, PDL, p);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

// =================================================================================================
// v2 (lutgemv_v2.cuh): plan + launch.  One CTA per SM; all process-wide state behind one mutex / atomics.
// =================================================================================================
typedef void (*K2)(const v2::P2, const CUtensorMap, const CUtensorMap);
struct K2Info { K2 fn; int tab, stage; };
// fused: variant 0: exact, fp32 x ; 1: exact, fp16 x ; 2: fp16 pair table, fp16 x ; 3: exact, bf16 x.  Accumulate mode (the 12
// symbols): variant 0 only.
constexpr int K2_VARIANTS = 4;
K2Info k2_lookup(int bits, int variant, bool fused) {
#define K2E(B, M, XT, F) K2Info{v2::lutgemv2_kernel<B, M, XT, F>, v2::C2<B, M>::TAB, v2::C2<B, M>::STAGE}
    if (bits == 4) {
        if (!fused) return K2E(4, 0, float, false);
        if (variant == 0) return K2E(4, 0, float, true);
        if (variant == 1) return K2E(4, 0, __half, true);
        if (variant == 3) return K2E(4, 0, __nv_bfloat16, true);
        return K2E(4, 1, __half, true);
    }
    if (!fused) return K2E(3, 0, float, false);
    if (variant == 0) return K2E(3, 0, float, true);
    if (variant == 1) return K2E(3, 0, __half, true);
    if (variant == 3) return K2E(3, 0, __nv_bfloat16, true);
    return K2E(3, 1, __half, true);
#undef K2E
}

// Stream-K plan of one layer for the v2 and sequence kernels, on a grid of at most `sm` CTAs, and the layer's buffers: fills the
// shape and buffer fields of p and returns the grid in G.
int plan_layer(const sqllm_lutgemv_args &a, int sm, v2::P2 &p, int &G) {
    const int K = a.in_features, N = a.out_features;
    set_layer(p, a);
    p.K = K; p.N = N;
    p.R = a.bits == 4 ? K / 8 : K / 32;
    p.strips = (N + STRIP - 1) / STRIP;
    const long long T = (long long)p.strips * p.R;
    if (T > 0x3fffffff) return fail(SQLLM_EINVAL, "problem too large");
    p.T = (int)T;
    p.chunk = std::max(2, (int)(2 * ((T + 2LL * sm - 1) / (2LL * sm))));
    G = (int)((T + p.chunk - 1) / p.chunk);
    p.csr_rpc = (N + G - 1) / G;
    p.hc = p.hrows = 0;
    if (p.topX > 0) {
        p.hrows = (K + G - 1) / G;
        p.hc = (K + p.hrows - 1) / p.hrows;
    }
    return SQLLM_OK;
}

// The two tensor maps over the packed matrix: 64 columns x (32 units | 2 units) boxes.
int tensor_maps(const sqllm_lutgemv_args &a, CUtensorMap &big, CUtensorMap &small) {
    const int rows_per_unit = a.bits == 4 ? 1 : 3, qrows = a.in_features / 32 * a.bits;
    // (a matrix shorter than one full stage never issues the big box; its map is clamped so that the encoder accepts it)
    const int rc = get_tensor_map(a.qweight, qrows, a.out_features, qrows < v2::SU2 * rows_per_unit ? 2 * rows_per_unit : v2::SU2 * rows_per_unit, big);
    return rc ? rc : get_tensor_map(a.qweight, qrows, a.out_features, 2 * rows_per_unit, small);
}

int launch2(const sqllm_lutgemv_args *a, int variant, bool fused, v2::P2 &p, cudaStream_t st) {
    const K2Info ki = k2_lookup(a->bits, variant, fused);
    KernelSmem all[2 * (1 + K2_VARIANTS)];  // every v2 kernel: accumulate mode and each fused variant, both widths
    int nk = 0;
    for (int b = 3; b <= 4; ++b) {
        all[nk++] = {k2_lookup(b, 0, false).fn, 227 * 1024};
        for (int v = 0; v < K2_VARIANTS; ++v) all[nk++] = {k2_lookup(b, v, true).fn, 227 * 1024};
    }
    int sm = 0;
    unsigned raw = 0;
    int rc = dev_setup(all, &sm, &raw);
    if (rc) return rc;
    int G = 0;
    if ((rc = plan_layer(*a, sm, p, G))) return rc;
    if (fused && p.N > MAX_N_FUSED) return fail(SQLLM_EINVAL, "out_features=%d exceeds the fused accumulator (max %d)", p.N, MAX_N_FUSED);
    if (fused && G > MAX_GRID_V2) return fail(SQLLM_EINVAL, "grid of %d CTAs exceeds the mailbox area (%d)", G, MAX_GRID_V2);
    const unsigned base = (raw + 127u) & ~127u;
    const unsigned xbytes = (unsigned)((p.K * (variant == 0 ? 4 : 2) + 127) & ~127);  // this layer's x, in its own dtype
    // one GEMV: the ring needs no more stages than the CTA's chunk fills
    const int n = v2::Carve(base, xbytes, 0u, ki.tab, 2, ki.stage, 0).depth(raw, 227 * 1024, ki.stage, (p.chunk + v2::SU2 - 1) / v2::SU2 + 1);
    if (n < 0) return fail(SQLLM_EINVAL, "in_features=%d does not fit the shared-memory carve-up of this table mode", p.K);
    if (n < 2) return fail(SQLLM_EINVAL, "in_features=%d leaves no room for a weight ring in shared memory", p.K);
    const int smem = (int)(v2::Carve(base, xbytes, 0u, ki.tab, 2, ki.stage, n).end - raw);
    p.nstage = n;
    p.smem_raw = raw;
    p.nown_ctas = 0;
    if (p.xw_world)
        for (int b = 0; b < G; ++b) {  // CTAs in whose range at least one strip starts
            const long long c0 = (long long)b * p.chunk, c1 = std::min<long long>(p.T, c0 + p.chunk);
            if ((c0 + p.R - 1) / p.R < (c1 + p.R - 1) / p.R) ++p.nown_ctas;
        }
    {
        std::lock_guard<std::recursive_mutex> lk(g_state_mu);
        p.trace = g_trace;
        if (g_trace) g_trace += g_trace_stride;
        g_last_grid = G;
    }
    CUtensorMap tm_big, tm_small;
    if ((rc = tensor_maps(*a, tm_big, tm_small))) return rc;
    const cudaError_t e = launch_ex(ki.fn, G, v2::THREADS2, smem, st, PDL, p, tm_big, tm_small);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}


// ---- sequences (lutgemv_seq.cuh): plan + descriptors at create time, two launches per run -----------------------------
typedef void (*KSeq)(const seq::SeqCfg);
struct KSeqInfo { KSeq fn; int tab, stage, ntb; };
// bf16 x always takes the exact table (the pair table multiplies fp16 by fp16), whatever `mode` says
// ops: the instance that also runs the items' RMSNorm / SiLU gating / residual (sqllm_sequence_create_ops with at least one op)
KSeqInfo kseq_lookup_ops(int bits, int mode, bool multi, bool bf16) {
#define KSO(B, M, X, T) KSeqInfo{seq::lutgemv_seq_kernel<B, M, X, T, true>, v2::C2<B, M>::TAB, v2::C2<B, M>::STAGE, v2::C2<B, M>::NTB}
    if (bf16) {
        if (bits == 4) return multi ? KSO(4, 0, true, __nv_bfloat16) : KSO(4, 0, false, __nv_bfloat16);
        return multi ? KSO(3, 0, true, __nv_bfloat16) : KSO(3, 0, false, __nv_bfloat16);
    }
    if (bits == 4) {
        if (mode == 0) return multi ? KSO(4, 0, true, __half) : KSO(4, 0, false, __half);
        return multi ? KSO(4, 1, true, __half) : KSO(4, 1, false, __half);
    }
    if (mode == 0) return multi ? KSO(3, 0, true, __half) : KSO(3, 0, false, __half);
    return multi ? KSO(3, 1, true, __half) : KSO(3, 1, false, __half);
#undef KSO
}
KSeqInfo kseq_lookup(int bits, int mode, bool multi, bool bf16) {
#define KSE(B, M, X) KSeqInfo{seq::lutgemv_seq_kernel<B, M, X>, v2::C2<B, M>::TAB, v2::C2<B, M>::STAGE, v2::C2<B, M>::NTB}
#define KSB(B, X) KSeqInfo{seq::lutgemv_seq_kernel<B, 0, X, __nv_bfloat16>, v2::C2<B, 0>::TAB, v2::C2<B, 0>::STAGE, v2::C2<B, 0>::NTB}
    if (bf16) {
        if (bits == 4) return multi ? KSB(4, true) : KSB(4, false);
        return multi ? KSB(3, true) : KSB(3, false);
    }
    if (bits == 4) {
        if (mode == 0) return multi ? KSE(4, 0, true) : KSE(4, 0, false);
        return multi ? KSE(4, 1, true) : KSE(4, 1, false);
    }
    if (mode == 0) return multi ? KSE(3, 0, true) : KSE(3, 0, false);
    return multi ? KSE(3, 1, true) : KSE(3, 1, false);
#undef KSB
#undef KSE
}
constexpr int SEQ_MAX_ITEMS = 1023;  // the mailbox tag keeps 10 bits for the item

size_t seq_item_len(const sqllm_seq_item &it) {  // elements of the item's full-length output vector
    const int members = it.members > 0 ? it.members : 1;
    const int nfull = it.out_features_full > 0 ? it.out_features_full : it.a.out_features / members;
    return (size_t)members * nfull;
}
}  // namespace

namespace __attribute__((visibility("hidden"))) sqllm {

// d.smem_raw from smem_base_probe, once per device.  The probe is synchronous and refused during stream capture: only v2 and sequence
// plans ask for it, and the first of them on a device must come before any capture - any warm-up does.  Caller holds g_state_mu.
int smem_window(DevInfo &d) {
    if (d.smem_raw) return SQLLM_OK;
    unsigned *d_out = nullptr, h_out = 0;
    cudaError_t pe = cudaMalloc(&d_out, sizeof(unsigned));
    if (pe == cudaSuccess) {
        smem_base_probe<<<1, 1, 1024>>>(d_out);
        pe = cudaMemcpy(&h_out, d_out, sizeof(unsigned), cudaMemcpyDeviceToHost);
        cudaFree(d_out);
    }
    if (pe != cudaSuccess || h_out == 0) {
        cudaGetLastError();
        return fail(SQLLM_ECUDA, "shared-memory probe failed (first call inside a stream capture? run one call before capturing): %s", cudaGetErrorString(pe));
    }
    d.smem_raw = h_out;
    return SQLLM_OK;
}

}  // namespace sqllm

struct sqllm_sequence {
    int n = 0, bits = 0, mode = 0, world = 1, rank = 0, grid = 0, smem = 0;
    seq::SeqCfg cfg;
    KSeq fn = nullptr;
    void *d_descs = nullptr, *d_exports = nullptr, *d_ws = nullptr, *d_arena = nullptr, *d_ops = nullptr;
    bool own_arena = false;
};

namespace {
int seq_fail_free(sqllm_sequence *s, int rc) {
    if (s) sqllm_sequence_destroy(s);
    return rc;
}
}  // namespace

extern "C" size_t sqllm_sequence_arena_bytes(const sqllm_seq_item *items, int n_items) {
    if (!items || n_items <= 0) return 0;
    size_t off = 0;
    for (int i = 0; i < n_items; ++i) off += (seq_item_len(items[i]) * 4 + 127) / 128 * 128;
    return off;
}

extern "C" int sqllm_sequence_create(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, sqllm_sequence **out) {
    return sqllm_sequence_create_dt(items, n_items, opt, SQLLM_DT_F16, out);
}

extern "C" int sqllm_sequence_create_dt(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, int dtype, sqllm_sequence **out) {
    return sqllm_sequence_create_ops(items, nullptr, n_items, opt, dtype, out);
}

namespace {
bool seq_op_active(const sqllm_seq_op &o) { return o.x_op != SQLLM_SEQ_X_PLAIN || o.res_from >= 0 || o.res_ext; }

// the checks of one item's op (items[i], ops[i]); the item's own checks have passed
int check_seq_op(const sqllm_seq_item *items, const sqllm_seq_op &o, int i, const char *tn) {
    const sqllm_lutgemv_args &a = items[i].a;
    const uintptr_t ga = reinterpret_cast<uintptr_t>(o.norm_weight), ra = reinterpret_cast<uintptr_t>(o.res_ext);
    if (o.x_op != SQLLM_SEQ_X_PLAIN && o.x_op != SQLLM_SEQ_X_RMSNORM && o.x_op != SQLLM_SEQ_X_SILU_MUL)
        return fail(SQLLM_EINVAL, "sequence: item %d: unknown x_op=%d", i, o.x_op);
    if (o.x_op == SQLLM_SEQ_X_RMSNORM) {
        if (!o.norm_weight || (ga & 15)) return fail(SQLLM_EINVAL, "sequence: item %d: norm_weight must be a 16-byte aligned %s vector", i, tn);
        if (!std::isfinite(o.eps) || o.eps < 0.f) return fail(SQLLM_EINVAL, "sequence: item %d: eps=%g must be finite and >= 0", i, (double)o.eps);
    }
    if (o.x_op == SQLLM_SEQ_X_SILU_MUL) {
        if (o.x2_from < 0 || o.x2_from >= i) return fail(SQLLM_EINVAL, "sequence: item %d: x2_from=%d must name an earlier item", i, o.x2_from);
        if (o.x2_offset < 0 || o.x2_offset % 4 || (size_t)o.x2_offset + a.in_features > seq_item_len(items[o.x2_from]))
            return fail(SQLLM_EINVAL, "sequence: item %d: x2 reads [%d, %d) of item %d's %zu outputs", i, o.x2_offset, o.x2_offset + a.in_features,
                        o.x2_from, seq_item_len(items[o.x2_from]));
    }
    if (o.res_from >= 0 && o.res_ext) return fail(SQLLM_EINVAL, "sequence: item %d: one residual source: res_from=%d or res_ext, not both", i, o.res_from);
    if (o.res_from >= i || o.res_from < -1) return fail(SQLLM_EINVAL, "sequence: item %d: residual source res_from=%d must name an earlier item (or -1)", i, o.res_from);
    if (o.res_from >= 0) {
        const size_t n = seq_item_len(items[i]), m = seq_item_len(items[o.res_from]);
        if (o.res_offset < 0 || o.res_offset % 4 || (size_t)o.res_offset + n > m)
            return fail(SQLLM_EINVAL, "sequence: item %d: residual reads [%d, %zu) of item %d's %zu outputs (the item's full length is %zu)",
                        i, o.res_offset, (size_t)std::max(0, o.res_offset) + n, o.res_from, m, n);
    }
    if (ra & 15) return fail(SQLLM_EINVAL, "sequence: item %d: res_ext must be a 16-byte aligned %s vector", i, tn);
    return SQLLM_OK;
}
}  // namespace

extern "C" int sqllm_sequence_create_ops(const sqllm_seq_item *items, const sqllm_seq_op *ops, int n_items, const sqllm_seq_options *opt, int dtype,
                                         sqllm_sequence **out) {
    if (dtype != SQLLM_DT_F16 && dtype != SQLLM_DT_BF16) return fail(SQLLM_EINVAL, "sequence: dtype=%d is not SQLLM_DT_F16 or SQLLM_DT_BF16", dtype);
    const bool bf = dtype == SQLLM_DT_BF16;
    const char *const tn = bf ? "bf16" : "fp16";
    if (!items || !opt || !out || n_items <= 0) return fail(SQLLM_EINVAL, "sequence: null / empty arguments");
    if (n_items > SEQ_MAX_ITEMS) return fail(SQLLM_EINVAL, "sequence: at most %d items (got %d)", SEQ_MAX_ITEMS, n_items);
    const int world = opt->world > 0 ? opt->world : 1, rank = opt->rank;
    if (world > 64 || rank < 0 || rank >= world) return fail(SQLLM_EINVAL, "sequence: bad world / rank (%d / %d)", world, rank);
    if (world > 1 && (!opt->arena || !opt->peer_base)) return fail(SQLLM_EINVAL, "sequence: several GPUs need a peer-visible arena and peer_base");
    // bf16 x keeps the exact table in the fp16 table mode, as sqllm_lutgemv_fused_dt does
    const int bits = items[0].a.bits, mode = opt->lut_mode == SQLLM_LUT_FP16_PAIR && !bf ? 1 : 0;
    int kmax = 0;
    for (int i = 0; i < n_items; ++i) {
        const sqllm_seq_item &it = items[i];
        const sqllm_lutgemv_args &a = it.a;
        const int rc = check_common(&a);
        if (rc) return rc;
        if (a.bits != bits) return fail(SQLLM_EINVAL, "sequence: item %d has bits=%d, item 0 has %d (one sequence, one width)", i, a.bits, bits);
        if (a.out_features < STRIP) return fail(SQLLM_EINVAL, "sequence: item %d: out_features=%d < %d", i, a.out_features, STRIP);
        if (a.out_features > MAX_N_FUSED) return fail(SQLLM_EINVAL, "sequence: item %d: out_features=%d exceeds %d", i, a.out_features, MAX_N_FUSED);
        if (a.full_rows && a.topX > MAX_TOPX_FUSED) return fail(SQLLM_EINVAL, "sequence: topX <= %d", MAX_TOPX_FUSED);
        const int members = it.members > 0 ? it.members : 1;
        if (a.out_features % members || (a.out_features / members) % 4) return fail(SQLLM_EINVAL, "sequence: item %d: %d columns are not %d members of a multiple of 4", i, a.out_features, members);
        if (world == 1 && seq_item_len(it) != (size_t)a.out_features) return fail(SQLLM_EINVAL, "sequence: item %d: members * out_features_full must equal out_features on one GPU", i);
        if (world > 1 && seq_item_len(it) < (size_t)world * a.out_features) return fail(SQLLM_EINVAL, "sequence: item %d: full length %zu < world * shard columns", i, seq_item_len(it));
        if (world > 1 && it.y) return fail(SQLLM_EINVAL, "sequence: item %d: plain y copies exist on one GPU only (use exports)", i);
        if (seq_item_len(it) % 4) return fail(SQLLM_EINVAL, "sequence: item %d: output length must be a multiple of 4", i);
        if (it.x_from >= i || it.x_from < -1) return fail(SQLLM_EINVAL, "sequence: item %d: x_from=%d must name an earlier item (or -1)", i, it.x_from);
        if (it.x_from < 0) {
            if (!it.x_ext || (reinterpret_cast<uintptr_t>(it.x_ext) & 15)) return fail(SQLLM_EINVAL, "sequence: item %d: x_ext must be a 16-byte aligned %s vector", i, tn);
        } else {
            if (it.x_offset < 0 || it.x_offset % 4 || (size_t)it.x_offset + a.in_features > seq_item_len(items[it.x_from]))
                return fail(SQLLM_EINVAL, "sequence: item %d reads [%d, %d) of item %d's %zu outputs", i, it.x_offset, it.x_offset + a.in_features, it.x_from, seq_item_len(items[it.x_from]));
        }
        if ((reinterpret_cast<uintptr_t>(it.y) & 1) || (reinterpret_cast<uintptr_t>(it.bias) & 3)) return fail(SQLLM_EINVAL, "sequence: item %d: misaligned y / bias", i);
        kmax = std::max(kmax, a.in_features);
    }
    for (int e = 0; e < opt->n_export; ++e) {
        if (!opt->export_items || !opt->export_dst) return fail(SQLLM_EINVAL, "sequence: export arrays missing");
        const int it = opt->export_items[e];
        if (it < 0 || it >= n_items || !opt->export_dst[e] || (reinterpret_cast<uintptr_t>(opt->export_dst[e]) & 7))
            return fail(SQLLM_EINVAL, "sequence: export %d: bad item %d or destination (8-byte aligned %s vector)", e, it, tn);
    }
    bool any_op = false;
    for (int i = 0; ops && i < n_items; ++i) {
        const int rc = check_seq_op(items, ops[i], i, tn);
        if (rc) return rc;
        any_op = any_op || seq_op_active(ops[i]);
    }
    const KSeqInfo ki = any_op ? kseq_lookup_ops(bits, mode, world > 1, bf) : kseq_lookup(bits, mode, world > 1, bf);
    int sm = 0;
    unsigned raw = 0;
    const int rc = dev_setup({{ki.fn, 227 * 1024}}, &sm, &raw);
    if (rc) return rc;
    const unsigned base = (raw + 127u) & ~127u;
    const int xbytes = (kmax * 2 + 127) & ~127;  // every item's x is staged in the 16-bit dtype in one buffer, and ntb strip-sum rows follow it
    // no cap from the chunk: the weight stream runs on across items
    const int nst = v2::Carve(base, xbytes, ki.ntb * STRIP * 4, ki.tab, ki.ntb, ki.stage, 0).depth(raw, 227 * 1024, ki.stage, v2::MAXD);
    if (nst < 0) return fail(SQLLM_EINVAL, "sequence: in_features=%d does not fit the shared-memory carve-up of this table mode", kmax);
    if (nst < 2) return fail(SQLLM_EINVAL, "sequence: in_features=%d leaves no room for a weight ring in shared memory", kmax);
    const int smem = (int)(v2::Carve(base, xbytes, ki.ntb * STRIP * 4, ki.tab, ki.ntb, ki.stage, nst).end - raw);

    sqllm_sequence *s = new sqllm_sequence();
    s->n = n_items; s->bits = bits; s->mode = mode; s->world = world; s->rank = rank; s->grid = sm; s->smem = smem; s->fn = ki.fn;
    // workspace: [0,4) token counter, [64,68) error word, per parity {flags [64 + MAX_STRIPS] ints, accumulator [MAX_N_FUSED] floats} (only
    // used by CTAs that own more than 8 strips), then EVERY item's own mailboxes: outlier row sums [N], partial strip sums [grid][64],
    // dense-row parts [topX][MAX_GRID_V2].  Mailboxes are not shared between items: an item may read only a slice of its predecessor's
    // output, so "x of item g+1 is complete" does not mean that every strip owner of item g has already taken its words.
    const size_t cnt_bytes = (size_t)(64 + MAX_STRIPS) * 4, acc_bytes = (size_t)MAX_N_FUSED * 4;
    const size_t par_off = 256, par_bytes = (cnt_bytes + acc_bytes + 255) / 256 * 256;
    std::vector<size_t> cbox_off(n_items), hbox_off(n_items), dbox_off(n_items);
    size_t ws_bytes = par_off + 2 * par_bytes;
    for (int i = 0; i < n_items; ++i) {
        const bool hyb = items[i].a.full_rows && items[i].a.topX > 0;
        cbox_off[i] = ws_bytes; ws_bytes += ((size_t)items[i].a.out_features * 8 + 255) / 256 * 256;
        hbox_off[i] = ws_bytes; ws_bytes += (size_t)MAX_GRID_V2 * 64 * 8;
        dbox_off[i] = ws_bytes; ws_bytes += hyb ? (size_t)items[i].a.topX * MAX_GRID_V2 * 8 : 0;
    }
    if (cudaMalloc(&s->d_ws, ws_bytes) != cudaSuccess || cudaMemset(s->d_ws, 0, ws_bytes) != cudaSuccess)
        return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: workspace allocation failed"));
    unsigned char *ws = static_cast<unsigned char *>(s->d_ws);
    const size_t arena_need = sqllm_sequence_arena_bytes(items, n_items);
    if (opt->arena) {
        if (opt->arena_bytes < arena_need || (reinterpret_cast<uintptr_t>(opt->arena) & 127))
            return seq_fail_free(s, fail(SQLLM_EINVAL, "sequence: arena of %zu bytes (128-byte aligned) needed, got %zu", arena_need, opt->arena_bytes));
        s->d_arena = opt->arena;
    } else {
        if (cudaMalloc(&s->d_arena, arena_need) != cudaSuccess || cudaMemset(s->d_arena, 0, arena_need) != cudaSuccess)
            return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: arena allocation failed"));
        s->own_arena = true;
    }
    std::vector<seq::SeqDesc> descs(n_items);
    std::vector<size_t> yoff(n_items);
    size_t off = 0;
    for (int i = 0; i < n_items; ++i) {
        yoff[i] = off;
        off += (seq_item_len(items[i]) * 4 + 127) / 128 * 128;
    }
    for (int i = 0; i < n_items; ++i) {
        const sqllm_seq_item &it = items[i];
        const sqllm_lutgemv_args &a = it.a;
        seq::SeqDesc &d = descs[i];
        memset(&d, 0, sizeof(d));
        v2::P2 &p = d.p;
        int G = 0;
        int rc = plan_layer(a, sm, p, G);
        if (rc) return seq_fail_free(s, rc);
        if (G > MAX_GRID_V2) return seq_fail_free(s, fail(SQLLM_EINVAL, "sequence: grid of %d CTAs exceeds the mailbox area", G));
        p.nstage = nst; p.smem_raw = raw;
        p.y_is_half = 1;
        p.bias = it.bias;
        p.out = it.y;
        p.x = it.x_from < 0 ? it.x_ext : nullptr;
        unsigned char *par = ws + par_off + (size_t)(i & 1) * par_bytes;
        p.ws_cnt = reinterpret_cast<int *>(par);
        p.ws_acc = reinterpret_cast<float *>(par + cnt_bytes);
        p.ws_hbox = reinterpret_cast<unsigned long long *>(ws + hbox_off[i]);
        p.ws_cbox = reinterpret_cast<unsigned long long *>(ws + cbox_off[i]);
        p.ws_dbox = reinterpret_cast<unsigned long long *>(ws + dbox_off[i]);
        p.xw_world = world > 1 ? world : 0; p.xw_rank = rank;
        p.xw_members = it.members > 0 ? it.members : 1;
        p.xw_nfull = it.out_features_full > 0 ? it.out_features_full : p.N / p.xw_members;
        p.trace = opt->trace ? reinterpret_cast<unsigned long long *>(opt->trace) + (size_t)i * 1024 * 32 : nullptr;
        d.x_tag = it.x_from < 0 ? nullptr : reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[it.x_from]) + it.x_offset;
        d.y_off = yoff[i];
        if ((rc = tensor_maps(a, d.tm_big, d.tm_small))) return seq_fail_free(s, rc);
    }
    std::vector<seq::SeqExport> ex(std::max(1, opt->n_export));
    for (int e = 0; e < opt->n_export; ++e) {
        const int it = opt->export_items[e];
        ex[e].src = reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[it]);
        ex[e].dst = opt->export_dst[e];
        ex[e].n = (int)seq_item_len(items[it]);
    }
    if (cudaMalloc(&s->d_descs, descs.size() * sizeof(seq::SeqDesc)) != cudaSuccess ||
        cudaMemcpy(s->d_descs, descs.data(), descs.size() * sizeof(seq::SeqDesc), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMalloc(&s->d_exports, ex.size() * sizeof(seq::SeqExport)) != cudaSuccess ||
        cudaMemcpy(s->d_exports, ex.data(), ex.size() * sizeof(seq::SeqExport), cudaMemcpyHostToDevice) != cudaSuccess)
        return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: descriptor upload failed: %s", cudaGetErrorString(cudaGetLastError())));
    if (any_op) {
        std::vector<seq::SeqOp> so(n_items);
        for (int i = 0; i < n_items; ++i) {
            const sqllm_seq_op &o = ops[i];
            seq::SeqOp &q = so[i];
            memset(&q, 0, sizeof(q));
            q.x_op = o.x_op;
            q.eps = o.eps;
            q.gamma = o.x_op == SQLLM_SEQ_X_RMSNORM ? o.norm_weight : nullptr;
            if (o.x_op == SQLLM_SEQ_X_SILU_MUL)
                q.x2_tag = reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[o.x2_from]) + o.x2_offset;
            if (o.res_from >= 0) q.res_tag = reinterpret_cast<const uint32_t *>(static_cast<unsigned char *>(s->d_arena) + yoff[o.res_from]) + o.res_offset;
            q.res_ext = o.res_ext;
        }
        if (cudaMalloc(&s->d_ops, so.size() * sizeof(seq::SeqOp)) != cudaSuccess ||
            cudaMemcpy(s->d_ops, so.data(), so.size() * sizeof(seq::SeqOp), cudaMemcpyHostToDevice) != cudaSuccess)
            return seq_fail_free(s, fail(SQLLM_ECUDA, "sequence: op upload failed: %s", cudaGetErrorString(cudaGetLastError())));
    }
    seq::SeqCfg &c = s->cfg;
    memset(&c, 0, sizeof(c));
    c.descs = static_cast<const seq::SeqDesc *>(s->d_descs);
    c.ngemv = n_items;
    c.epoch = reinterpret_cast<const unsigned *>(ws);
    c.err = reinterpret_cast<int *>(ws + 64);
    c.smem_raw = raw; c.xbytes = xbytes; c.nstage = nst;
    c.world = world; c.rank = rank;
    c.peer_base = reinterpret_cast<const unsigned long long *>(opt->peer_base);
    c.arena_base = reinterpret_cast<unsigned long long>(s->d_arena);
    c.exports = static_cast<const seq::SeqExport *>(s->d_exports);
    c.nexport = opt->n_export;
    c.ops = static_cast<const seq::SeqOp *>(s->d_ops);
    *out = s;
    return SQLLM_OK;
}

extern "C" int sqllm_sequence_run(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    seq::seq_bump_epoch<<<1, 1, 0, st>>>(reinterpret_cast<unsigned *>(s->d_ws));
    const cudaError_t e = launch_ex(s->fn, s->grid, v2::THREADS2, s->smem, st, COOPERATIVE, s->cfg);
    if (e != cudaSuccess) return fail(SQLLM_ECUDA, "sequence launch failed: %s", cudaGetErrorString(e));
    return SQLLM_OK;
}

extern "C" int sqllm_sequence_error(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    int h = 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (cudaMemcpyAsync(&h, static_cast<unsigned char *>(s->d_ws) + 64, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return fail(SQLLM_ECUDA, "sequence: reading the error word failed: %s", cudaGetErrorString(cudaGetLastError()));
    return h != 0;
}

extern "C" int sqllm_sequence_reset_error(sqllm_sequence *s, void *stream) {
    if (!s) return fail(SQLLM_EINVAL, "sequence: null handle");
    if (cudaMemsetAsync(static_cast<unsigned char *>(s->d_ws) + 64, 0, 4, static_cast<cudaStream_t>(stream)) != cudaSuccess)
        return fail(SQLLM_ECUDA, "sequence: clearing the error word failed: %s", cudaGetErrorString(cudaGetLastError()));
    return SQLLM_OK;
}

extern "C" void sqllm_sequence_destroy(sqllm_sequence *s) {
    if (!s) return;
    cudaFree(s->d_descs);
    cudaFree(s->d_exports);
    cudaFree(s->d_ops);
    cudaFree(s->d_ws);
    if (s->own_arena) cudaFree(s->d_arena);
    delete s;
}

namespace {

// ---- fused GEMV: v2, or v1 in the deterministic mode; with an exchange descriptor (v2 only) the result goes to every rank's
// arena instead of y ---------------------------------------------------------------------------------------------------------------
// x_dt / y_dt: SQLLM_DT_* codes, a pair sqllm_lutgemv_fused_dt accepts
int lutgemv_fused(const sqllm_lutgemv_args *a, const void *x, int x_dt, void *y, int y_dt, const float *bias,
                  void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, cudaStream_t st) {
    int rc = check_common(a);
    if (rc) return rc;
    if (!x || (!xc && !y)) return fail(SQLLM_EINVAL, xc ? "x / exchange descriptor must not be null" : "x / y must not be null");
    if (reinterpret_cast<uintptr_t>(x) & 15) return fail(SQLLM_EINVAL, "x must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(bias) & 15))
        return fail(SQLLM_EINVAL, xc ? "bias must be 16-byte aligned" : "y and bias must be 16-byte aligned");
    const int det = det_mode();
    if (xc) {
        if (det == 1) return fail(SQLLM_EINVAL, "the exchange path needs the default (non-deterministic) fused mode");
        if (xc->world < 1 || xc->world > 64 || xc->rank < 0 || xc->rank >= xc->world) return fail(SQLLM_EINVAL, "bad world / rank (%d / %d)", xc->world, xc->rank);
        if (xc->members < 1 || a->out_features % xc->members) return fail(SQLLM_EINVAL, "out_features=%d is not %d equal members", a->out_features, xc->members);
        const int w = a->out_features / xc->members;
        if (w % 4) return fail(SQLLM_EINVAL, "shard width %d must be a multiple of 4", w);
        if (xc->out_features_full < xc->world * w) return fail(SQLLM_EINVAL, "out_features_full=%d < world * shard width = %d", xc->out_features_full, xc->world * w);
        if (!xc->peer_base) return fail(SQLLM_EINVAL, "peer_base must not be null");
        if ((xc->out_offset & 15) || (xc->flag_offset & 7) || (xc->state_offset & 7) || (xc->error_offset & 3)) return fail(SQLLM_EINVAL, "misaligned arena offsets");
        const int yb = y_dt == SQLLM_DT_F32 ? 4 : 2;
        if ((xc->out_features_full * yb) % 16 || (w * yb) % 8) return fail(SQLLM_EINVAL, "vector sizes must keep 8/16-byte store alignment");
    }
    const bool hyb = a->full_rows && a->topX > 0;
    if (hyb && a->topX > MAX_TOPX_FUSED) return fail(SQLLM_EINVAL, "fused path supports topX <= %d", MAX_TOPX_FUSED);
    unsigned char *ws = static_cast<unsigned char *>(workspace);
    if (det == 0) {
        if (!workspace || workspace_bytes < WS_HEADER) return fail(SQLLM_EWORKSPACE, "workspace too small: need %zu bytes, got %zu", (size_t)WS_HEADER, workspace_bytes);
        v2::P2 q;
        memset(&q, 0, sizeof(q));
        q.ws_cnt = reinterpret_cast<int *>(ws);
        q.ws_acc = reinterpret_cast<float *>(ws + WS_ACC_OFF);
        q.ws_hbox = reinterpret_cast<unsigned long long *>(ws + WS_HBOX_OFF);
        q.ws_cbox = reinterpret_cast<unsigned long long *>(ws + WS_CBOX_OFF);
        q.ws_dbox = reinterpret_cast<unsigned long long *>(ws + WS_DBOX_OFF);
        q.x = x; q.out = y; q.y_is_half = y_dt != SQLLM_DT_F32; q.bias = bias;
        if (xc) {
            q.xw_world = xc->world; q.xw_rank = xc->rank; q.xw_members = xc->members; q.xw_nfull = xc->out_features_full;
            q.xw_base = reinterpret_cast<const unsigned long long *>(xc->peer_base);
            q.xw_out_off = xc->out_offset; q.xw_flag_off = xc->flag_offset; q.xw_state_off = xc->state_offset; q.xw_err_off = xc->error_offset;
        }
        // layers narrower than one strip keep the exact codebook in the fp16 table mode: their results do not depend on the mode;
        // bf16 x always does (the pair table multiplies fp16 by fp16)
        const int variant = x_dt == SQLLM_DT_F16 ? (lut_mode() == 1 && a->out_features >= STRIP ? 2 : 1) : x_dt == SQLLM_DT_BF16 ? 3 : 0;
        return launch2(a, variant, true, q, st);
    }
    Plan pl;
    rc = make_plan(a->bits, a->in_features, a->out_features, hyb ? a->topX : 0, a->rows != nullptr, STAGE, pl);
    if (rc) return rc;
    if (!workspace || workspace_bytes < pl.ws_bytes)
        return fail(SQLLM_EWORKSPACE, "workspace too small: need %zu bytes, got %zu", pl.ws_bytes, workspace_bytes);
    Params p;
    memset(&p, 0, sizeof(p));
    p.ws_cnt = reinterpret_cast<int *>(ws + pl.ws_cnt_off);
    p.ws_hyb = reinterpret_cast<float *>(ws + pl.ws_hyb_off);
    p.ws_part = reinterpret_cast<float *>(ws + pl.ws_part_off);
    p.ws_csr = reinterpret_cast<float *>(ws + pl.ws_csr_off);
    p.x = x; p.x_dt = x_dt; p.out = y; p.y_dt = y_dt; p.bias = bias;
    return launch(a, pl, p, st);
}

}  // namespace

extern "C" {

int sqllm_workspace_error(const void *workspace, void *stream) {
    if (!workspace) return fail(SQLLM_EINVAL, "null workspace");
    int flag = 0;
    if (cudaMemcpyAsync(&flag, static_cast<const unsigned char *>(workspace) + 64, 4, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)) != cudaSuccess ||
        cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess)
        return fail(SQLLM_ECUDA, "cannot read the workspace error word: %s", cudaGetErrorString(cudaGetLastError()));
    return flag ? 1 : 0;
}

size_t sqllm_workspace_bytes(int bits, int in_features, int out_features, int topX) {
    Plan pl;
    if (bits != 3 && bits != 4) return 0;
    if (in_features <= 0 || in_features % 64 || out_features <= 0) return 0;
    // CSR staging changes the shared-memory footprint, hence occupancy, grid and chunk: take the max of both plans.  The
    // deterministic mode gets exactly what its kernel needs.  The default mode plans with the CSR cols / vals alone in the staging
    // buffer: less shared memory, at least as many CTAs and strip partials, so a workspace sized in either mode serves both.
    const int stage = det_mode() == 1 ? STAGE : CSR_CH * 8;
    size_t b = 0;
    for (int csr = 0; csr < 2; ++csr)
        if (make_plan(bits, in_features, out_features, topX, csr != 0, stage, pl) == SQLLM_OK && pl.ws_bytes > b) b = pl.ws_bytes;
    return b;
}

int sqllm_lutgemv(const sqllm_lutgemv_args *a, void *stream) {
    int rc = check_common(a);
    if (rc) return rc;
    if (!a->vec || !a->mul) return fail(SQLLM_EINVAL, "vec / mul must not be null");
    if (a->batch < 1) return fail(SQLLM_EINVAL, "batch must be >= 1");
    if (reinterpret_cast<uintptr_t>(a->vec) & 15) return fail(SQLLM_EINVAL, "vec must be 16-byte aligned");
    if (a->batch >= 2) return launch_batched(a, static_cast<cudaStream_t>(stream));
    v2::P2 q;
    memset(&q, 0, sizeof(q));
    q.x = a->vec;
    q.out = a->mul;
    return launch2(a, 0, false, q, static_cast<cudaStream_t>(stream));
}

int sqllm_lutgemv_fused(const sqllm_lutgemv_args *a, const void *x, int x_is_half, void *y, int y_is_half,
                        const float *bias, void *workspace, size_t workspace_bytes, void *stream) {
    return sqllm_lutgemv_fused_dt(a, x, x_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, y, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias,
                                  workspace, workspace_bytes, stream);
}

int sqllm_lutgemv_fused_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *workspace, size_t workspace_bytes, void *stream) {
    if (!fused_dt_pair(x_dtype, y_dtype)) return fused_dt_fail(x_dtype, y_dtype);
    return lutgemv_fused(a, x, x_dtype, y, y_dtype, bias, workspace, workspace_bytes, nullptr, static_cast<cudaStream_t>(stream));
}

int sqllm_lutgemv_fused_exchange(const sqllm_lutgemv_args *a, const void *x, int x_is_half, int y_is_half, const float *bias,
                                 void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, void *stream) {
    return sqllm_lutgemv_fused_exchange_dt(a, x, x_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, y_is_half ? SQLLM_DT_F16 : SQLLM_DT_F32, bias,
                                           workspace, workspace_bytes, xc, stream);
}

int sqllm_lutgemv_fused_exchange_dt(const sqllm_lutgemv_args *a, const void *x, int x_dtype, int y_dtype, const float *bias,
                                    void *workspace, size_t workspace_bytes, const sqllm_exchange *xc, void *stream) {
    if (!fused_dt_pair(x_dtype, y_dtype)) return fused_dt_fail(x_dtype, y_dtype);
    if (!xc) {
        const int rc = check_common(a);
        return rc ? rc : fail(SQLLM_EINVAL, "x / exchange descriptor must not be null");
    }
    return lutgemv_fused(a, x, x_dtype, nullptr, y_dtype, bias, workspace, workspace_bytes, xc, static_cast<cudaStream_t>(stream));
}

// ---- the reference's 12 launchers -----------------------------------------------------------------
static int run12(int bits, const float *vec, const int32_t *mat, float *mul, const float *lut, int height, int width,
                 int batch, int vec_height, const int32_t *rows, const int32_t *cols, const float *vals, int num_rows,
                 const float *full_rows, const int32_t *fri, int fr_height, int fr_width, void *stream) {
    sqllm_lutgemv_args a;
    memset(&a, 0, sizeof(a));
    a.bits = bits;
    if (height <= 0 || height % bits) return fail(SQLLM_EINVAL, "height=%d is not a multiple of bits=%d", height, bits);
    a.in_features = height / bits * 32;
    a.out_features = width;
    a.batch = batch;
    if (vec_height >= 0 && vec_height != a.in_features)
        return fail(SQLLM_EINVAL, "vec has %d features, packed matrix implies %d", vec_height, a.in_features);
    if (rows && num_rows != width) return fail(SQLLM_EINVAL, "num_rows=%d must equal the matrix width %d", num_rows, width);
    if (full_rows && fr_height != a.in_features)
        return fail(SQLLM_EINVAL, "full_rows has %d rows, expected in_features=%d", fr_height, a.in_features);
    a.qweight = mat; a.lookup_table = lut; a.vec = vec; a.mul = mul;
    a.rows = rows; a.cols = cols; a.vals = vals;
    a.full_rows = full_rows; a.full_row_indices = fri; a.topX = full_rows ? fr_width : 0;
    return sqllm_lutgemv(&a, stream);
}

int sqllm_vecquant3matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul, const float *lut, int height,
                                         int width, void *stream) {
    return run12(3, vec, mat, mul, lut, height, width, 1, -1, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul, const float *lut, int height,
                                         int width, void *stream) {
    return run12(4, vec, mat, mul, lut, height, width, 1, -1, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul, const float *lut,
                                                 int height, int width, int batch, int vec_height, void *stream) {
    return run12(3, vec, mat, mul, lut, height, width, batch, vec_height, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul, const float *lut,
                                                 int height, int width, int batch, int vec_height, void *stream) {
    return run12(4, vec, mat, mul, lut, height, width, batch, vec_height, 0, 0, 0, 0, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat, const float *vec,
                                              float *mul, int num_rows, const int32_t *mat3, const float *lut, int height,
                                              int width, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat, const float *vec,
                                              float *mul, int num_rows, const int32_t *mat4, const float *lut, int height,
                                              int width, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows, const int32_t *mat3,
                                                      const float *lut, int height, int width, int batch, int vec_height,
                                                      void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant4matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows, const int32_t *mat4,
                                                      const float *lut, int height, int width, int batch, int vec_height,
                                                      void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, 0, 0, 0, 0, stream);
}
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows, const int32_t *fri,
                                                     float *mul, int num_rows, const int32_t *mat3, const float *lut,
                                                     int height, int width, int fr_height, int fr_width, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows, const int32_t *fri,
                                                     float *mul, int num_rows, const int32_t *mat4, const float *lut,
                                                     int height, int width, int fr_height, int fr_width, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, 1, -1, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                             const float *vec, const float *full_rows, const int32_t *fri,
                                                             float *mul, int num_rows, const int32_t *mat3, const float *lut,
                                                             int height, int width, int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream) {
    return run12(3, vec, mat3, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                             const float *vec, const float *full_rows, const int32_t *fri,
                                                             float *mul, int num_rows, const int32_t *mat4, const float *lut,
                                                             int height, int width, int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream) {
    return run12(4, vec, mat4, mul, lut, height, width, batch, vec_height, rows, cols, mat, num_rows, full_rows, fri, fr_height, fr_width, stream);
}

}  // extern "C"
