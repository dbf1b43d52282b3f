// dequant.cuh - the dense weight of a layer, W[c][k] = codebook + CSR outliers + dense rows, written as fp32, fp16 or bf16 [n][K]
// (nn.Linear.weight's [out, in] layout) for the column range [c0, c0 + n): sqllm_dequantize.  Included by lutgemv_kernels.cu
// inside its anonymous namespace, after lutgemm_tc.cuh (whose index decoders it shares).
//
// Every element is defined exactly:
//   w  = lookup_table[c][idx(k, c)]                                        (fp32)
//   w += vals[e]          for each CSR entry e of row c with cols[e] == k, in storage order
//   w += full_rows[k][j]  for each j with full_row_indices[j] == c, in ascending j
//   W[c - c0][k] = w rounded once (to nearest even) to the output type
// CSR columns outside [0, K) and dense-row channels outside [0, N) are ignored; duplicates add up.  The codebook is the stored
// fp32 table whatever sqllm_set_lut_mode says.
//
// The packed words are [K/32*bits][N] (contiguous along c) and W is contiguous along k, so a CTA decodes a BN x BK tile (BN
// output channels, BK inputs) into an fp32 tile in shared memory and writes it out transposed:
//   * thread (c, h) reads the packed words of column c for the 32 inputs of group h (coalesced along c) and decodes them through
//     the tile's codebook, staged [value][column] with lutgemm_tc.cuh's row stride (tc::dec3 / tc::dec4);
//   * CSR: one warp per column scans the column's row 32 entries at a time and adds the entries that fall in the tile's k range,
//     in storage order (a ballot, then one lane after the other);
//   * dense rows: the j whose channel lies in the tile, listed in ascending j; one thread per k adds them in that order;
//   * W: each thread rounds 4 (fp32) or 8 (fp16 / bf16) consecutive k of one row and writes them with one 16-byte store.
// Every output element is written once by one thread: no atomics, no workspace, bit-reproducible.
#pragma once

namespace dq {

constexpr int BN = 64;         // output channels per CTA
constexpr int BK = 128;        // inputs per CTA (4 groups of 32)
constexpr int THREADS = 256;   // (column, group) pairs: BN x BK / 32
constexpr int PITCH = BK + 4;  // floats per tile row: the 16-byte stores of 8 consecutive columns hit distinct banks
constexpr int LUT_ROW = tc::BN;  // floats per codebook row: the stride tc::dec3 / tc::dec4 decode with (BN of them are used)
constexpr int TILE = 0;
constexpr int LUT = TILE + BN * PITCH * 4;   // fp32 [16][LUT_ROW]
constexpr int LIST = LUT + 16 * LUT_ROW * 4;  // int [THREADS] dense rows j of one pass, then int [THREADS] their channels in the tile
constexpr int WCNT = LIST + 2 * THREADS * 4;  // int [THREADS / 32] listed per warp
constexpr int SMEM = WCNT + THREADS / 32 * 4;

struct PD {
    const uint32_t *qw;
    const float *lut;
    const int *rows, *cols;
    const float *vals;
    const float *full_rows;
    const int *fri;
    int topX, K, N;
    int c0, n;  // column range [c0, c0 + n)
    void *w;    // [n][K], OT
};

// two fp32 values rounded (to nearest even) to a 16-bit type, packed low then high
template <typename OT>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
    const OT a = f32_to<OT>(lo), b = f32_to<OT>(hi);
    unsigned short ua, ub;
    memcpy(&ua, &a, 2);
    memcpy(&ub, &b, 2);
    return (uint32_t)ua | ((uint32_t)ub << 16);
}

template <int BITS, typename OT>
__global__ void __launch_bounds__(THREADS) dequant_kernel(const PD p) {
    constexpr int LV = 1 << BITS;
    constexpr int WROWS = BITS == 4 ? 4 : 3;  // packed words per (column, 32 k)
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *tile = reinterpret_cast<float *>(smem_raw + TILE);
    float *lut_s = reinterpret_cast<float *>(smem_raw + LUT);
    int *list_j = reinterpret_cast<int *>(smem_raw + LIST), *list_c = list_j + THREADS;
    int *wcnt = reinterpret_cast<int *>(smem_raw + WCNT);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t0 = blockIdx.x * BN;            // first output row of the tile
    const int n0 = p.c0 + t0;                  // ... its channel
    const int nt = min(BN, p.n - t0);          // channels in the tile
    const int k0 = blockIdx.y * BK;
    const int kt = min(BK, p.K - k0);          // inputs in the tile: a multiple of 32
    const int K = p.K;
    const int c = tid & (BN - 1), h = tid >> 6;  // decode role: tile column, group of 32 inputs
    const int kb = 32 * h;

    uint32_t q[WROWS];
    {
        const int r0 = BITS == 4 ? (k0 + kb) / 8 : 3 * ((k0 + kb) / 32);
        const bool ok = c < nt && kb < kt;
#pragma unroll
        for (int r = 0; r < WROWS; ++r) q[r] = ok ? __ldg(p.qw + (size_t)(r0 + r) * p.N + n0 + c) : 0u;
    }
    for (int e = tid; e < BN * LV; e += THREADS) {
        const int cc = e / LV, v = e % LV;
        lut_s[v * LUT_ROW + cc] = cc < nt ? __ldg(p.lut + (size_t)(n0 + cc) * LV + v) : 0.f;
    }
    __syncthreads();

    // ---- codebook ----
    {
        float w[32];
        const uint32_t lb = smem_u32(lut_s) + c * 4;
        if constexpr (BITS == 4) tc::dec4(w, q, lb);
        else tc::dec3<0>(w, q[0], q[1], q[2], lb);
        const uint32_t dst = smem_u32(tile + c * PITCH + kb);
#pragma unroll
        for (int i = 0; i < 8; ++i)
            asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + 16 * i), "f"(w[4 * i]), "f"(w[4 * i + 1]), "f"(w[4 * i + 2]),
                         "f"(w[4 * i + 3]) : "memory");
    }
    __syncthreads();

    // ---- CSR outliers: one warp per column, entries in storage order ----
    if (p.rows) {
        for (int cc = warp; cc < nt; cc += THREADS / 32) {
            const int e1 = __ldg(p.rows + n0 + cc + 1);
            float *trow = tile + cc * PITCH;
            for (int eb = __ldg(p.rows + n0 + cc); eb < e1; eb += 32) {
                const int e = eb + lane;
                const int k = e < e1 ? __ldg(p.cols + e) : -1;
                const bool hit = k >= k0 && k < k0 + kt;
                const float v = hit ? __ldg(p.vals + e) : 0.f;
                for (unsigned m = __ballot_sync(0xffffffffu, hit); m; m &= m - 1) {
                    if (lane == __ffs(m) - 1) trow[k - k0] += v;
                    __syncwarp();
                }
            }
        }
        __syncthreads();
    }

    // ---- dense rows: the j on the tile's channels in ascending j, one thread per k ----
    for (int jb = 0; jb < p.topX; jb += THREADS) {
        const int j = jb + tid;
        const int f = j < p.topX ? __ldg(p.fri + j) : -1;
        const bool in = f >= n0 && f < n0 + nt;
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) wcnt[warp] = __popc(m);
        __syncthreads();
        int base = 0, total = 0;
#pragma unroll
        for (int i = 0; i < THREADS / 32; ++i) {
            base += i < warp ? wcnt[i] : 0;
            total += wcnt[i];
        }
        if (in) {
            const int at = base + __popc(m & ((1u << lane) - 1u));
            list_j[at] = j;
            list_c[at] = f - n0;
        }
        __syncthreads();
        for (int kk = tid; kk < kt; kk += THREADS) {
            const float *fr = p.full_rows + (size_t)(k0 + kk) * p.topX;
            for (int i = 0; i < total; ++i) tile[list_c[i] * PITCH + kk] += __ldg(fr + list_j[i]);
        }
        __syncthreads();  // the list and the counts are rewritten by the next pass; the tile is read below
    }

    // ---- W rows: one rounding, 16-byte stores ----
    constexpr int EPV = 16 / (int)sizeof(OT);  // elements per store
    const int vpr = kt / EPV;                  // stores per row
    for (int i = tid; i < nt * vpr; i += THREADS) {
        const int cc = i / vpr, kv = i - cc * vpr;
        const uint32_t src = smem_u32(tile + cc * PITCH + kv * EPV);
        uint4 o;
        if constexpr (std::is_same<OT, float>::value) {
            o = lds_u4(src);
        } else {
            const float4 a = lds_v4(src), b = lds_v4(src + 16);
            o = make_uint4(pack16x2<OT>(a.x, a.y), pack16x2<OT>(a.z, a.w), pack16x2<OT>(b.x, b.y), pack16x2<OT>(b.z, b.w));
        }
        *reinterpret_cast<uint4 *>(reinterpret_cast<OT *>(p.w) + (size_t)(t0 + cc) * K + k0 + kv * EPV) = o;
    }
}

}  // namespace dq
