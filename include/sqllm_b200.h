/*
 * sqllm_b200.h - C ABI of the H100-native (sm_90a) dense-and-sparse LUT GEMV library
 *                (libsqllm_b200.so), a from-scratch replacement for the hot path of
 *                SqueezeAILab/SqueezeLLM:  squeezellm/quant_cuda_kernel.cu + quant_cuda.cpp.
 *
 * Boundary.  The reference exposes this path as a pybind11 C++ module `quant_cuda` whose 12
 * functions take torch::Tensor by value (squeezellm/quant_cuda.cpp:257-270) - there is no C ABI in
 * the reference.  This header is the C ABI that module sits on in our build: plain device
 * pointers, sizes and a stream; no torch types.  Each of the 12 entry points below replaces the
 * reference launcher named in its comment (same argument meaning, same accumulate-into-`mul`
 * contract); squeezellm_b200/csrc/quant_cuda_pybind.cpp is the thin torch::Tensor wrapper that
 * re-exports them under the reference's Python names.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer on the current CUDA device unless said otherwise;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - calls are asynchronous; nothing is retained after the call returns except `workspace`
 *     contents, which belong to the library between calls on the same stream;
 *   - return value: 0 on success, a negative SQLLM_E* code otherwise; sqllm_last_error() gives a
 *     thread-local human readable message.  (The reference performs no checks at all:
 *     squeezellm/quant_cuda_kernel.cu has no TORCH_CHECK / cudaGetLastError - SURVEY.md 8(b).)
 *   - shapes (reference: squeezellm/quant.py:48-95):
 *       vec           fp32 [batch, in]            (batch = 1 for the non-batched entry points)
 *       mat3 / mat4   int32 [in/32*bits, out]     packed indices, row-major
 *       lookup_table  fp32 [out, 2^bits]
 *       mul           fp32 [batch, out]           ACCUMULATED INTO (caller pre-fills zeros or bias)
 *       rows          int32 [out+1]   CSR row pointers, row = output channel
 *       cols          int32 [nnz]     input index of each non-zero
 *       vals          fp32  [nnz]
 *       full_rows     fp32 [in, topX] ; full_row_indices int32 [topX]  (output channel of column j)
 *     `height` = in/32*bits (rows of mat), `width` = out, as in the reference launchers.
 *   - requirements (checked, SQLLM_EINVAL otherwise): in % 64 == 0, out % 4 == 0, 16-byte aligned
 *     mat / vec, 1 <= batch.  The reference silently requires in % 128 == 0 and out % 128 == 0.
 */
#ifndef SQLLM_B200_H
#define SQLLM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SQLLM_OK 0
#define SQLLM_EINVAL (-1)   /* bad argument (shape, alignment, null pointer) */
#define SQLLM_ECUDA (-2)    /* a CUDA runtime call or launch failed */
#define SQLLM_EWORKSPACE (-3) /* workspace missing or too small */

#define SQLLM_ABI_VERSION 4   /* 2: + sqllm_lutgemv_fused_exchange, sqllm_set_deterministic ; 3: + sqllm_set_lut_mode, sqllm_workspace_error ; 4: + sqllm_sequence_*,
                                 later + sqllm_lutgemm_fused, sqllm_lutgemv_rows, sqllm_lutgemm_t, sqllm_lut_grad,
                                 sqllm_lutgemm_fused_dt, sqllm_lutgemv_fused_dt, sqllm_lutgemv_rows_dt, sqllm_dequantize,
                                 sqllm_fisher_accumulate, sqllm_sequence_create_dt, sqllm_lutgemv_fused_exchange_dt,
                                 sqllm_lutgemm_fused_f32, sqllm_sequence_create_ops
                                 (backward compatible, same version) */

int sqllm_abi_version(void);
const char *sqllm_last_error(void);

/* Number of SMs of the current device, the grid of the one-GEMV and sequence kernels
 * (informational; also used by bench.py to report the grid). */
int sqllm_device_sm_count(void);

/* ---------------------------------------------------------------------------------------------
 * Workspace.  Used only by the *_fused entry point (cross-CTA accumulator, counters, deterministic-mode partials).
 * Must be zero-filled once after allocation (cudaMemset); the library keeps it consistent afterwards.  One
 * workspace serves layers of any shape, but must not be used by two streams concurrently.  A size returned in either
 * summation mode serves both.
 * ------------------------------------------------------------------------------------------- */
size_t sqllm_workspace_bytes(int bits, int in_features, int out_features, int topX);

/* ---------------------------------------------------------------------------------------------
 * Generic descriptor entry point (what all 12 wrappers below call).
 * ------------------------------------------------------------------------------------------- */
typedef struct sqllm_lutgemv_args {
    int bits;                 /* 3 or 4 */
    int in_features;          /* K */
    int out_features;         /* N */
    int batch;                /* rows of vec / mul */
    const int32_t *qweight;   /* [K/32*bits, N] */
    const float *lookup_table;/* [N, 2^bits] */
    const float *vec;         /* [batch, K] fp32 */
    float *mul;               /* [batch, N] fp32, accumulated into */
    /* optional CSR outliers (rows == NULL -> none) */
    const int32_t *rows;
    const int32_t *cols;
    const float *vals;
    /* optional dense rows (full_rows == NULL or topX == 0 -> none) */
    const float *full_rows;
    const int32_t *full_row_indices;
    int topX;
} sqllm_lutgemv_args;

int sqllm_lutgemv(const sqllm_lutgemv_args *args, void *stream);

/* Fused-path summation mode (process-wide).
 *   0 (default; env SQLLM_DETERMINISTIC unset): contributions are added in the order they arrive (red.add.f32), like the
 *     reference's atomicAdd - results can differ in the last bits from run to run.
 *   1: per-strip partials reduced in a fixed order by the last-arriving contributor - bit-reproducible, 1.3-2x slower on
 *     layers with outliers. */
void sqllm_set_deterministic(int on);

/* Look-up-table precision of the fused path (process-wide; the 12 reference launchers below always use the exact table).
 *   SQLLM_LUT_EXACT (default): the per-channel codebook is used as stored, fp32 (squeezellm/quant_cuda_kernel.cu:779,866).
 *   SQLLM_LUT_FP16_PAIR      : north_star's "per-channel fp16 LUT" - centroids are rounded to fp16 (round-to-nearest-even) when a
 *     CTA builds its shared-memory table, which then holds PAIRS of centroids: one shared-memory read serves two weights and
 *     the products run as fp16 x fp16 -> fp32 FMAs (exact products, fp32 accumulation).  Only taken when x is fp16 (an fp32 x
 *     silently keeps the exact table); centroids must be finite in fp16 (|v| <= 65504).  Error against the exact result is that
 *     of the centroid rounding alone: <= 2^-11 relative per weight, ~2.5e-4 of max|y| on 4096-wide layers (tests/test_lut_fp16.py
 *     states and checks the bounds).  Environment: SQLLM_LUT_MODE=fp16.  Do not switch while other threads launch. */
#define SQLLM_LUT_EXACT 0
#define SQLLM_LUT_FP16_PAIR 1
void sqllm_set_lut_mode(int mode);
int sqllm_get_lut_mode(void);

/* Reads the workspace's error word (synchronises `stream`): 1 if a bounded in-kernel wait (2 s) ever gave up on this workspace -
 * the result of that call, and possibly later ones, is incomplete - else 0; negative on failure. */
int sqllm_workspace_error(const void *workspace, void *stream);

/* Fused module path behind QuantLinearLUT.forward (squeezellm/quant.py:211-312), batch-1 decode:
 *   y[c] = bias[c] + LUT-GEMV + CSR + dense rows, written (not accumulated) as fp16 or fp32,
 * from an fp16 or fp32 x, in ONE launch: replaces torch.zeros (quant.py:218), x.float() (:223,267),
 * the 1-3 reference launches and y.to(dtype) (:311).  Summation order: see sqllm_set_deterministic.
 * x_is_half / y_is_half select the element type of x / y.  bias may be NULL.  x, y and bias must be 16-byte aligned;
 * out_features <= SQLLM_FUSED_MAX_OUT and topX <= SQLLM_FUSED_MAX_TOPX on this path (and on the sequence and exchange
 * entry points); larger layers go through sqllm_lutgemv / the 12 launchers.  args->vec / args->mul / args->batch are ignored. */
#define SQLLM_FUSED_MAX_TOPX 128
#define SQLLM_FUSED_MAX_OUT 262144
int sqllm_lutgemv_fused(const sqllm_lutgemv_args *args,
                        const void *x, int x_is_half, void *y, int y_is_half, const float *bias,
                        void *workspace, size_t workspace_bytes, void *stream);

/* Fused module path for M >= 1 rows (prefill, evaluation) on the tensor cores (wgmma):
 *   y[m][c] = bias[c] + LUT-GEMM + CSR + dense rows, written (not accumulated), from fp16 x [M][in_features] (row-major),
 * in ONE launch.  args->batch = M; args->vec / args->mul are ignored.  y is fp16 (y_is_half) or fp32 [M][out_features].
 * The outliers and dense rows are folded into the dequantized weight tiles, so there is no limit on topX or on the outliers per
 * row; CSR column indices need not be ascending (ascending rows are cheaper).  Every weight is split into two fp16 parts of a
 * per-column power-of-two scale and both are multiplied in (exact products, fp32 accumulation): the codebook is always used as
 * stored, sqllm_set_lut_mode does not apply.  Every output is written once by one CTA in a fixed order: bit-reproducible.
 * Requirements (checked, SQLLM_EINVAL otherwise): in_features % 32 == 0, batch >= 1, x and y 16-byte aligned, qweight,
 * lookup_table and bias 4-byte aligned.  No workspace, no allocation, no host synchronisation: CUDA-graph capturable. */
int sqllm_lutgemm_fused(const sqllm_lutgemv_args *args, const void *x_half, void *y, int y_is_half, const float *bias,
                        void *stream);

/* Fused module path for a few fp16 rows (decode of several sequences, speculative-decoding verification, short prompts) on the
 * CUDA cores: y[m][c] = bias[c] + LUT-GEMV + CSR + dense rows, written (not accumulated), from fp16 x [M][in_features]
 * (row-major), in ONE launch.  args->batch = M >= 1 (any M is correct; QuantLinearLUT sends 2 to 63 rows here); args->vec /
 * args->mul are ignored.  y is fp16 (y_is_half) or fp32 [M][out_features].  The exact fp32 codebook and fp32 sums are always
 * used: sqllm_set_lut_mode does not apply.  Every output is written once by one CTA in a fixed order (thread-block clusters
 * split K; the leader adds the peers' partial sums over distributed shared memory), so results are bit-reproducible and a
 * row's result does not depend on M or on the other rows: sqllm_set_deterministic does not apply either.  No limit on topX or on
 * the outliers per row; duplicate dense-row channels add up; dense-row channels outside [0, out_features) and CSR columns
 * outside [0, in_features) are ignored.  in_features <= SQLLM_ROWS_MAX_IN (the slab of x each CTA stages must fit its shared
 * memory); out_features <= 65535 * 64.  Requirements (checked, SQLLM_EINVAL otherwise): in_features % 32 == 0,
 * out_features % 4 == 0, batch >= 1, non-null qweight / lookup_table / x / y, x and y 16-byte aligned, qweight, lookup_table
 * and bias 4-byte aligned, topX >= 0, full_row_indices present with full_rows.  No workspace, no allocation, no host
 * synchronisation: CUDA-graph capturable and safe on several streams at once. */
#define SQLLM_ROWS_MAX_IN 49152
int sqllm_lutgemv_rows(const sqllm_lutgemv_args *args, const void *x_half, void *y, int y_is_half, const float *bias,
                       void *stream);

/* Element types of the tensors of sqllm_lutgemm_fused_dt, sqllm_lutgemv_fused_dt, sqllm_lutgemv_rows_dt, sqllm_lutgemm_t,
 * sqllm_lut_grad and sqllm_dequantize. */
#define SQLLM_DT_F32 0
#define SQLLM_DT_F16 1
#define SQLLM_DT_BF16 2

/* sqllm_lutgemm_fused for fp16 or bf16 x: the same tensor-core LUT-GEMM, y[m][c] = bias[c] + LUT-GEMM + CSR + dense rows, written
 * (not accumulated), from x [M][in_features] (row-major) of x_dtype = SQLLM_DT_F16 or SQLLM_DT_BF16 into y [M][out_features] of
 * y_dtype = SQLLM_DT_F32 or x's dtype.  fp16 x is computed exactly as by sqllm_lutgemm_fused (which calls this).  bf16 x: every
 * folded weight (codebook + CSR + dense rows, over the column's power-of-two scale) is split exactly into three bf16 parts,
 * hi = bf16(w), mid = bf16(w - hi), lo = bf16(w - hi - mid), which carry the fp32 value down to bf16's subnormal range; x is
 * exact in bf16, so every product on the tensor cores is exact and the sums are fp32.  The codebook is always used as stored:
 * sqllm_set_lut_mode does not apply.  Every output is written once by one CTA in a fixed order: results are bit-reproducible,
 * and a row's bits do not depend on M or on the other rows.  Requirements (checked, SQLLM_EINVAL otherwise): those of
 * sqllm_lutgemm_fused, and the two dtype codes above.  No workspace, no allocation, no host synchronisation: CUDA-graph
 * capturable and safe on several streams at once. */
int sqllm_lutgemm_fused_dt(const sqllm_lutgemv_args *args, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *stream);

/* sqllm_lutgemm_fused for fp32 x: the same tensor-core LUT-GEMM, y[m][c] = bias[c] + LUT-GEMM + CSR + dense rows, written (not
 * accumulated), from fp32 x [M][in_features] (row-major) into fp32 y [M][out_features].  fp32 x is not exact in a 16-bit operand, so
 * both sides are split exactly into three bf16 parts with the same rule: x = x_h + x_m + x_l with x_h = bf16(x),
 * x_m = bf16(x - x_h), x_l = bf16(x - x_h - x_m), and each folded weight w (codebook + CSR + dense rows, over the column's
 * power-of-two scale) = w_h + w_m + w_l as for bf16 x.  Per 64-k chunk the tensor cores multiply the six part pairs whose orders
 * sum to at most 2, smallest first: x_l.w_h, x_m.w_m, x_h.w_l, then x_m.w_h, x_h.w_m, then x_h.w_h (each over the chunk's four
 * k16 steps), into one fp32 accumulator that starts from zero and is added into the fp32 running sum once per chunk.  Every
 * product is exact; the dropped terms x_m.w_l + x_l.w_m + x_l.w_l are below 2^-23 |x||w| per product (about 2 u, u = 2^-24), so
 * each output is within a few u of sum_k |x_k||w_kc| of the exact result, as for fp16 and bf16 x.  Below |x| of about 2^-110
 * (1e-33) the lower parts of x fall into bf16's subnormal range and the split keeps x only to within 2^-133 absolute.  The codebook
 * is always used as stored: sqllm_set_lut_mode does not apply.  Every output is written once by one CTA in a fixed order: results
 * are bit-reproducible, and a row's bits do not depend on M or on the other rows.  Any topX and any number of outliers.
 * Requirements (checked, SQLLM_EINVAL otherwise, before any device access): those of sqllm_lutgemm_fused (in_features % 32 == 0,
 * batch >= 1, non-null x and y, x and y 16-byte aligned, qweight, lookup_table and bias 4-byte aligned).  No workspace, no
 * allocation, no host synchronisation: CUDA-graph capturable and safe on several streams at once. */
int sqllm_lutgemm_fused_f32(const sqllm_lutgemv_args *args, const float *x, float *y, const float *bias, void *stream);

/* sqllm_lutgemv_fused with the element types as codes, and bf16 x besides fp32 and fp16: the same one-vector LUT-GEMV,
 * y[c] = bias[c] + LUT-GEMV + CSR + dense rows, written (not accumulated).  Pairs (x_dtype, y_dtype):
 *   SQLLM_DT_F32  x: y SQLLM_DT_F32 or SQLLM_DT_F16;   SQLLM_DT_F16 x: y SQLLM_DT_F32 or SQLLM_DT_F16;
 *   SQLLM_DT_BF16 x: y SQLLM_DT_F32 or SQLLM_DT_BF16;  any other pair: SQLLM_EINVAL (the message names both codes).
 * fp32 and fp16 x are computed exactly as by sqllm_lutgemv_fused (which calls this).  bf16 x is staged in its own type and every
 * value is widened to fp32 exactly before its product: the exact fp32 codebook and fp32 sums, in both summation modes
 * (sqllm_set_deterministic).  SQLLM_LUT_FP16_PAIR applies to fp16 x only: bf16 x keeps the exact table, as fp32 x does.  Every
 * other requirement (alignment, SQLLM_FUSED_MAX_*, the workspace) is that of sqllm_lutgemv_fused; CUDA-graph capturable, one
 * workspace per stream. */
int sqllm_lutgemv_fused_dt(const sqllm_lutgemv_args *args, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                           void *workspace, size_t workspace_bytes, void *stream);

/* sqllm_lutgemv_rows for fp16 or bf16 x: the same multi-row LUT-GEMV from x [M][in_features] of x_dtype = SQLLM_DT_F16 or
 * SQLLM_DT_BF16 into y [M][out_features] of y_dtype = SQLLM_DT_F32 or x's dtype; any other pair: SQLLM_EINVAL (the message names
 * both codes).  fp16 x is computed exactly as by sqllm_lutgemv_rows (which calls this).  bf16 x is widened to fp32 exactly as the
 * CTA stages it; from there on both types run the same code: exact fp32 codebook, fp32 sums, bit-reproducible, a row's result
 * independent of M and of the other rows.  Every other requirement is that of sqllm_lutgemv_rows (in_features <=
 * SQLLM_ROWS_MAX_IN, out_features % 4 == 0, alignment); no workspace, CUDA-graph capturable, safe on several streams at once. */
int sqllm_lutgemv_rows_dt(const sqllm_lutgemv_args *args, const void *x, int x_dtype, void *y, int y_dtype, const float *bias,
                          void *stream);

/* Input gradient of the layer (backpropagation through QuantLinearLUT): the transposed LUT-GEMM
 *   dx[m][k] = sum_c dy[m][c] W[k][c],   W[k][c] = LUT[c][idx(k,c)] + CSR(c,k) + sum_j full_rows[k][j] [full_row_indices[j] == c]
 * from dy [M][out_features] (row-major; fp32, fp16 or bf16: dy_dtype) into dx [M][in_features] (written, not accumulated; fp32
 * or dy's dtype: dx_dtype).  args->batch = M; args->vec / args->mul are ignored; there is no bias term.  The outlier rules are
 * those of the forward entry points: duplicate dense-row channels add up, CSR columns outside [0, in_features) and dense-row
 * channels outside [0, out_features) are ignored, no limit on topX or on the entries per CSR row, CSR columns need not be
 * ascending.  Every output is written once by one CTA in a fixed order: bit-reproducible.
 *   path 1 = tensor cores (fp16 / bf16 dy only): 128 x 128 dx tiles on wgmma, the reduction axis in chunks of 64 columns; every
 *     folded weight is split exactly (fp16 dy: hi + lo fp16 parts of a per-chunk power-of-two scale; bf16 dy: three bf16 parts),
 *     products are exact and sums fp32.  A weight more than about 2^20 below the largest weight of its 64-column chunk is kept
 *     to about 2^-40 of that largest weight (fp16 dy).
 *   path 2 = CUDA cores (any dy dtype): exact fp32 codebook and fp32 sums; thread-block clusters split out_features and the
 *     leader adds the peers' partial sums over distributed shared memory; a row's result does not depend on M or on the other
 *     rows.
 *   path 0 = path 1 for fp16 / bf16 dy of at least SQLLM_BWD_TC_MIN_ROWS rows, else path 2.
 * Requirements (checked, SQLLM_EINVAL otherwise): in_features % 32 == 0, out_features >= 1, batch >= 1, non-null qweight /
 * lookup_table / dy / dx, qweight and lookup_table 4-byte aligned, dy aligned to its element size, dx 16-byte aligned,
 * topX >= 0, full_row_indices present with full_rows.  No workspace, no allocation, no host synchronisation: CUDA-graph
 * capturable and safe on several streams at once. */
#define SQLLM_BWD_TC_MIN_ROWS 96
int sqllm_lutgemm_t(const sqllm_lutgemv_args *args, const void *dy, int dy_dtype, void *dx, int dx_dtype, int path,
                    void *stream);

/* Gradients of the layer's continuous parameters (fine-tuning the codebook with the indices fixed), from G = x^T . dy:
 *   G[k][c]          = sum_m x[m][k] dy[m][c]
 *   dlut[c][v]       = sum_{k : idx(k,c) = v} G[k][c]                              [out_features][2^bits]
 *   dvals[e]         = G[cols[e]][c] for e in CSR row c and 0 <= cols[e] < K, else 0    [nnz]
 *   dfull_rows[k][j] = G[k][full_row_indices[j]] if 0 <= full_row_indices[j] < N, else 0 [in_features][topX]
 * x [M][in_features] and dy [M][out_features] are row-major (x_dtype, dy_dtype: SQLLM_DT_*, any pair); args->batch = M.  The outputs
 * are fp32, written (not accumulated); a NULL output is not computed.  dvals needs args->rows / cols (the entries of CSR rows
 * [rows[0], rows[out_features]) are written; args->vals is not read), dfull_rows needs args->full_row_indices and topX >= 1
 * (args->full_rows is not read); the lookup table is not read either.  Duplicate CSR entries and duplicate dense-row channels each
 * get the full G of their position.  The gradient is that of the exact codebook whatever sqllm_set_lut_mode says.
 *   path 1 = tensor cores (x and dy both fp16 or both bf16): wgmma m64n128k16 on the operands as given, exact products, fp32 sums.
 *   path 2 = CUDA cores (any dtype pair): fp32 products and sums of the values as given.
 *   path 0 = path 1 when x and dy are both fp16 or both bf16 and M >= SQLLM_LUT_GRAD_TC_MIN_ROWS, else path 2.
 * Both reduce each 128 x 128 tile of G over M in fixed chunks, bucket it in ascending k, and add the bins of the CTAs of a
 * thread-block cluster (which split in_features) in rank order: every output is written once in a fixed order, bit-reproducible.
 * Requirements (checked, SQLLM_EINVAL otherwise): in_features % 32 == 0, out_features >= 1, batch >= 1, non-null qweight / x / dy,
 * at least one output, qweight and the outputs 4-byte aligned, x and dy aligned to their element size, topX >= 0.  No workspace,
 * no allocation, no host synchronisation: CUDA-graph capturable and safe on several streams at once. */
#define SQLLM_LUT_GRAD_TC_MIN_ROWS 8
int sqllm_lut_grad(const sqllm_lutgemv_args *args, const void *x, int x_dtype, const void *dy, int dy_dtype, float *dlut, float *dvals,
                   float *dfull_rows, int path, void *stream);

/* The dense weight of the layer's output channels [col0, col0 + ncols): W [ncols][in_features] (row-major: nn.Linear.weight's
 * [out, in] layout) of w_dtype = SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16, written (not accumulated).  Every element is
 *   w  = lookup_table[c][idx(k, c)]                                        (fp32)
 *   w += vals[e]          for each CSR entry e of row c with cols[e] == k, in storage order          (fp32 adds)
 *   w += full_rows[k][j]  for each j with full_row_indices[j] == c, in ascending j                  (fp32 adds)
 *   W[c - col0][k] = w rounded once, to nearest even, to w_dtype
 * CSR columns outside [0, in_features) and dense-row channels outside [0, out_features) are ignored; duplicates add up; no limit
 * on topX or on the entries per CSR row.  The codebook is the stored fp32 table: sqllm_set_lut_mode does not apply.  The column
 * range lets a caller dequantize one member of stacked sibling layers without copying the packed weights.  args->vec, mul and
 * batch are ignored.  Every output is written once by one thread: bit-reproducible.  Requirements (checked, SQLLM_EINVAL
 * otherwise): in_features % 32 == 0, out_features >= 1, 0 <= col0, ncols >= 1, col0 + ncols <= out_features, non-null qweight /
 * lookup_table / w, full_row_indices present with full_rows, topX >= 0, qweight and
 * lookup_table 4-byte aligned, w 16-byte aligned.  No workspace, no allocation, no host synchronisation: CUDA-graph capturable
 * and safe on several streams at once. */
int sqllm_dequantize(const sqllm_lutgemv_args *args, int col0, int ncols, void *w, int w_dtype, void *stream);

/* The diagonal of the empirical Fisher information of a linear layer, accumulated into fisher [out_features][in_features] (fp32,
 * row-major: nn.Linear.weight's [out, in] layout).  x [rows][in_features] and dy [rows][out_features] (the layer's input and the
 * gradient of its output) are row-major, both of dtype = SQLLM_DT_F16 or SQLLM_DT_BF16; sample s is rows [s seq_len, (s + 1)
 * seq_len).  Every element is
 *   g_s   = sum_{t in sample s} dy[t][n] x[t][k]    per 64-row chunk of the sample, in ascending order: the chunk's exact products
 *                                                   summed in the tensor core's fp32 accumulator, the chunk sums added in fp32
 *   f     = fmaf(g_s, g_s, f)                       for s = 0, 1, ... in ascending order, from f = 0 (fp32)
 *   fisher[n][k] = fisher[n][k] + f                 (one fp32 add)
 * so fisher gains sum_s g_s^2: the squares of the per-sample weight gradients, not the square of their sum.  Every element is read
 * once and written once by one thread: bit-reproducible.  Requirements (checked, SQLLM_EINVAL otherwise): rows, seq_len >= 1,
 * rows % seq_len == 0, in_features and out_features positive multiples of 8, out_features <= 8388480, non-null x / dy / fisher,
 * all three 16-byte aligned.
 * No workspace, no atomics, no host synchronisation: CUDA-graph capturable and safe on several streams at once. */
int sqllm_fisher_accumulate(const void *x, const void *dy, int dtype, int rows, int seq_len, int in_features, int out_features,
                            float *fisher, void *stream);

/* Fused forward of a COLUMN SHARD with the exchange built in (multi-GPU; the reference has none - north_star's
 * "column-shard each QuantLinear + all-reduce on the output vector", done by the kernel instead of a separate collective).
 * Every rank calls this with its shard (args->out_features = members * w columns: `members` sibling layers stacked, each
 * contributing this rank's w columns [rank*w, (rank+1)*w) of its out_features_full).  The CTAs that finish the GEMV store
 * their slice of y straight into EVERY rank's arena over NVLink peer memory - member m, column rank*w + j goes to element
 * [m][rank*w + j] of a [members][out_features_full] vector at out_offset - publish with a system-scope release on a
 * counter in each arena, and wait (bounded: 2 s, then *error_offset = 1) until all ranks' finishers have published on the
 * local one.  When the call's grid completes, the local vector is whole: the next stream-ordered consumer may read it.
 *   peer_base    device array [world] of the arenas' base addresses (e.g. torch symmetric memory's buffer_ptrs_dev)
 *   *_offset     byte offsets inside every arena: the destination vector, a u64 arrival counter (zero-initialised, only
 *                ever incremented), this rank's u64 expected-arrivals word (zero-initialised, local use), a u32 error word.
 * All ranks must issue the same sequence of exchange calls; consecutive calls must not target the same destination
 * (a fast rank may deliver call k+1 while a slow one still reads the result of call k).  Default summation mode only. */
typedef struct sqllm_exchange {
    int world, rank;
    int members;
    int out_features_full;
    const uint64_t *peer_base;
    size_t out_offset, flag_offset, state_offset, error_offset;
} sqllm_exchange;

int sqllm_lutgemv_fused_exchange(const sqllm_lutgemv_args *args,
                                 const void *x, int x_is_half, int y_is_half, const float *bias,
                                 void *workspace, size_t workspace_bytes, const sqllm_exchange *xchg, void *stream);

/* sqllm_lutgemv_fused_exchange with dtype codes: x of x_dtype, the destination vectors of y_dtype, exactly the pairs of
 * sqllm_lutgemv_fused_dt (SQLLM_DT_BF16 x: SQLLM_DT_F32 or SQLLM_DT_BF16 vectors, each element rounded once with the bias inside
 * the fp32 sum); any other pair: SQLLM_EINVAL with sqllm_lutgemv_fused_dt's message.  sqllm_lutgemv_fused_exchange calls this. */
int sqllm_lutgemv_fused_exchange_dt(const sqllm_lutgemv_args *args, const void *x, int x_dtype, int y_dtype, const float *bias,
                                    void *workspace, size_t workspace_bytes, const sqllm_exchange *xchg, void *stream);

/* ---------------------------------------------------------------------------------------------
 * The reference's 12 launchers, one C entry point each.
 * ------------------------------------------------------------------------------------------- */
/* vecquant3matmul_nuq_perchannel_cuda  - squeezellm/quant_cuda_kernel.cu:132-154 */
int sqllm_vecquant3matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul,
                                         const float *lookup_table, int height, int width, void *stream);
/* vecquant4matmul_nuq_perchannel_cuda  - squeezellm/quant_cuda_kernel.cu:157-179 */
int sqllm_vecquant4matmul_nuq_perchannel(const float *vec, const int32_t *mat, float *mul,
                                         const float *lookup_table, int height, int width, void *stream);
/* vecquant3matmul_nuq_perchannel_batched_cuda - :182-207 ; batch = vec.size(0), vec_height = vec.size(1) */
int sqllm_vecquant3matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul,
                                                 const float *lookup_table, int height, int width,
                                                 int batch, int vec_height, void *stream);
/* vecquant4matmul_nuq_perchannel_batched_cuda - :210-235 */
int sqllm_vecquant4matmul_nuq_perchannel_batched(const float *vec, const int32_t *mat, float *mul,
                                                 const float *lookup_table, int height, int width,
                                                 int batch, int vec_height, void *stream);
/* vecquant3matmul_spmv_nuq_perchannel_cuda - :238-282  (mat = CSR values, mat3 = packed weights) */
int sqllm_vecquant3matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                              const float *vec, float *mul, int num_rows,
                                              const int32_t *mat3, const float *lookup_table,
                                              int height, int width, void *stream);
/* vecquant4matmul_spmv_nuq_perchannel_cuda - :285-327 */
int sqllm_vecquant4matmul_spmv_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                              const float *vec, float *mul, int num_rows,
                                              const int32_t *mat4, const float *lookup_table,
                                              int height, int width, void *stream);
/* vecquant3matmul_spmv_nuq_perchannel_batched_cuda - :331-381 */
int sqllm_vecquant3matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows,
                                                      const int32_t *mat3, const float *lookup_table,
                                                      int height, int width, int batch, int vec_height,
                                                      void *stream);
/* vecquant4matmul_spmv_nuq_perchannel_batched_cuda - :385-435 */
int sqllm_vecquant4matmul_spmv_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols, const float *mat,
                                                      const float *vec, float *mul, int num_rows,
                                                      const int32_t *mat4, const float *lookup_table,
                                                      int height, int width, int batch, int vec_height,
                                                      void *stream);
/* vecquant3matmul_spmv_hybrid_nuq_perchannel_cuda - :439-507 ; full_rows is [fr_height=in, fr_width=topX] */
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows,
                                                     const int32_t *full_row_indices, float *mul, int num_rows,
                                                     const int32_t *mat3, const float *lookup_table,
                                                     int height, int width, int fr_height, int fr_width,
                                                     void *stream);
/* vecquant4matmul_spmv_hybrid_nuq_perchannel_cuda - :511-577 */
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel(const int32_t *rows, const int32_t *cols, const float *mat,
                                                     const float *vec, const float *full_rows,
                                                     const int32_t *full_row_indices, float *mul, int num_rows,
                                                     const int32_t *mat4, const float *lookup_table,
                                                     int height, int width, int fr_height, int fr_width,
                                                     void *stream);
/* vecquant3matmul_spmv_hybrid_nuq_perchannel_batched_cuda - :580-657 */
int sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols,
                                                             const float *mat, const float *vec,
                                                             const float *full_rows,
                                                             const int32_t *full_row_indices, float *mul,
                                                             int num_rows, const int32_t *mat3,
                                                             const float *lookup_table, int height, int width,
                                                             int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream);
/* vecquant4matmul_spmv_hybrid_nuq_perchannel_batched_cuda - :660-738 */
int sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(const int32_t *rows, const int32_t *cols,
                                                             const float *mat, const float *vec,
                                                             const float *full_rows,
                                                             const int32_t *full_row_indices, float *mul,
                                                             int num_rows, const int32_t *mat4,
                                                             const float *lookup_table, int height, int width,
                                                             int fr_height, int fr_width, int batch,
                                                             int vec_height, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Sequences: ONE persistent launch for a whole list of dependent matvecs.
 * Replaces the reference's per-layer launch loop during decode (squeezellm/llama.py:226-234 calls
 * QuantLinearLUT.forward once per layer; each forward is quant.py:212-312, i.e. 1-3 launches of
 * quant_cuda_kernel.cu:132-738).  Every item is one fused matvec (as sqllm_lutgemv_fused, fp16 in
 * and out, or bf16 in and out with sqllm_sequence_create_dt); its input is either an external
 * vector or a slice of an earlier item's output.
 * The kernel keeps the weight stream running across item boundaries and hands results from one
 * item to the next as self-validating tagged words in an arena (csrc/lutgemv_seq.cuh) - no
 * launch, no grid-wide barrier, no fence between two matvecs.  All items share `bits`.
 *
 * Several GPUs (column shards, one process per GPU): every rank creates the same sequence over
 * its own shards (items[i].a.out_features = members * shard width) and passes the peer-visible
 * arena of every rank; owners store their slice of each result into every rank's arena over
 * NVLink, the next item's input poll is the exchange.  All ranks must call sqllm_sequence_run the
 * same number of times.
 * ------------------------------------------------------------------------------------------- */
typedef struct sqllm_sequence sqllm_sequence;

typedef struct sqllm_seq_item {
    sqllm_lutgemv_args a;    /* the matrix: bits, in/out features, qweight, lookup_table, CSR, dense rows (vec/mul/batch ignored) */
    const float *bias;       /* optional, [out_features] */
    int x_from;              /* -1: x_ext ; i >= 0: the (full-length) output vector of item i < this item's index */
    int x_offset;            /* first element of that vector this item reads (multiple of 4); it reads in_features elements */
    const void *x_ext;       /* [in_features] of the sequence's dtype (fp16 unless sqllm_sequence_create_dt says bf16), read by every run (x_from == -1) */
    void *y;                 /* optional plain [out_features] copy of this item's own output columns, of the sequence's dtype */
    int members;             /* several GPUs: the item stacks `members` column shards of equal width (else 1) */
    int out_features_full;   /* several GPUs: full length of one member's output vector (else out_features) */
} sqllm_seq_item;

typedef struct sqllm_seq_options {
    int lut_mode;            /* SQLLM_LUT_EXACT / SQLLM_LUT_FP16_PAIR */
    int world, rank;         /* 1, 0 on a single GPU */
    void *arena;             /* world > 1: this rank's peer-visible arena (zero-filled once); NULL on one GPU: allocated here */
    size_t arena_bytes;
    const uint64_t *peer_base; /* world > 1: DEVICE array of `world` arena base addresses as seen from this rank */
    int n_export;            /* results wanted as plain vectors of the sequence's dtype: item indices and destinations (full length) */
    const int *export_items;
    void *const *export_dst;
    uint64_t *trace;         /* debug builds (-DSQLLM_TRACE): [n_items][1024][32] time stamps, else NULL */
} sqllm_seq_options;

/* bytes of arena a sequence over these items needs (0 on error) */
size_t sqllm_sequence_arena_bytes(const sqllm_seq_item *items, int n_items);
int sqllm_sequence_create(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, sqllm_sequence **out);
/* The same for the activation type `dtype`: SQLLM_DT_F16 (what sqllm_sequence_create makes) or SQLLM_DT_BF16.  It is the type of
 * every x_ext, of the values the items hand over (the low half of each tagged word), of the items' y copies and of the export
 * destinations; every item's output is rounded to it once, with the bias inside the fp32 sum.  A bf16 sequence uses the exact
 * table whatever opt->lut_mode says (the pair table multiplies fp16 by fp16).  Any other code: SQLLM_EINVAL (the message names
 * it), checked before any device access like the other arguments. */
int sqllm_sequence_create_dt(const sqllm_seq_item *items, int n_items, const sqllm_seq_options *opt, int dtype, sqllm_sequence **out);

/* What a decoder layer puts between two matvecs, inside the same launch: per item, a transform of its input and a residual added to
 * its output.  Every op rounds to the sequence's dtype once:
 *   SQLLM_SEQ_X_RMSNORM   x'_k = round(w_k (x_k r)), r = 1 / sqrt(S / K + eps), S = sum x_k^2 in fp32 in one fixed order (every CTA
 *                         computes the same bits); w = norm_weight [in_features] of the sequence's dtype.  (HF's RMSNorm rounds x r to
 *                         the dtype before multiplying by w: one rounding more.)
 *   SQLLM_SEQ_X_SILU_MUL  x'_k = round(silu(g_k) u_k), silu(g) = g / (1 + exp(-g)) in fp32; g = the item's input (x_from, x_offset),
 *                         u = in_features elements of item x2_from's output from x2_offset (an earlier item, possibly the same as x_from)
 *   residual              y = round(sum + bias + r): r = element res_offset + e of item res_from's full-length output (res_from earlier
 *                         than the item; e = the element of the item's own full-length output), or element e of res_ext, a plain vector
 *                         of the item's full length; res_from = -1 and res_ext = NULL: none.
 * On several GPUs every vector involved is full length, as the items' outputs are. */
#define SQLLM_SEQ_X_PLAIN 0
#define SQLLM_SEQ_X_RMSNORM 1
#define SQLLM_SEQ_X_SILU_MUL 2
typedef struct sqllm_seq_op {
    int x_op;                /* SQLLM_SEQ_X_* */
    const void *norm_weight; /* RMSNorm: [in_features] of the sequence's dtype, 16-byte aligned */
    float eps;               /* RMSNorm: finite, >= 0 */
    int x2_from, x2_offset;  /* SiLU gating: the up slice (earlier item, offset a multiple of 4) */
    int res_from, res_offset; /* residual: earlier item and first element (a multiple of 4), or -1 */
    const void *res_ext;     /* residual: external vector (16-byte aligned), or NULL */
} sqllm_seq_op;

/* sqllm_sequence_create_dt with one op per item (ops[i] for items[i]); ops == NULL: exactly sqllm_sequence_create_dt, and so is a
 * list of ops that do nothing (x_op plain, res_from -1, res_ext NULL).  Bad ops (unknown x_op; null or misaligned norm_weight; eps not
 * finite or < 0; an x2 slice out of range; a residual source not earlier or too short; misaligned res_ext) give SQLLM_EINVAL with a
 * message naming the item, before any device access. */
int sqllm_sequence_create_ops(const sqllm_seq_item *items, const sqllm_seq_op *ops, int n_items, const sqllm_seq_options *opt, int dtype,
                              sqllm_sequence **out);
/* two launches on `stream` (token counter, then the persistent kernel); CUDA-graph capturable */
int sqllm_sequence_run(sqllm_sequence *s, void *stream);
/* synchronises `stream`; 1 if a bounded in-kernel wait ever gave up (results incomplete), 0 if not, < 0 on error */
int sqllm_sequence_error(sqllm_sequence *s, void *stream);
/* clears the error word on `stream` (after a start-up skew between ranks has been dealt with: barrier, then reset on every rank) */
int sqllm_sequence_reset_error(sqllm_sequence *s, void *stream);
void sqllm_sequence_destroy(sqllm_sequence *s);

/* Test hook: unpack the packed indices on the GPU exactly as the GEMV kernels do
 * (idx uint8 [in, out]); lets tests prove the integer path bit-exact on its own. */
int sqllm_unpack_indices(int bits, const int32_t *qweight, int in_features, int out_features,
                         uint8_t *idx, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Quantizer: exact weighted 1-D k-means per row (the codebook fit of reference quantization/nuq.py:50-58,
 * solved exactly by dynamic programming instead of sklearn's seeded Lloyd; DESIGN.md section 3.13).
 *   w, s        fp32 [rows, n]   values and sample weights (s >= 0 and finite, w finite: not checked on the device);
 *                                a row whose weights are all zero is weighted uniformly (nuq.py:174-175)
 *   centroids   fp32 [rows, k]   the optimal centroids, non-decreasing; a cluster with no weight repeats its neighbour's
 *   labels      uint8 [rows, n]  nearest centroid of every element, ties to the lower index:
 *                                label(w) = #{j in 1..k-1 : w > fl32(0.5f * (c[j-1] + c[j]))}
 *   requirements (SQLLM_EINVAL otherwise, checked before any device access): rows >= 1, 2 <= k <= 16, k <= n <= 65535,
 *   non-null 4-byte aligned w / s / centroids, non-null labels, a 256-byte aligned workspace.
 * The workspace (no initialisation needed) holds one chunk of rows; sqllm_kmeans1d_workspace_bytes gives its size for
 * (rows, n, k) (it queries the sort's temporary storage, so it needs a current device).  Results are bit-reproducible and a
 * row's result depends on that row alone; no atomics; capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------- */
int sqllm_kmeans1d_workspace_bytes(int rows, int n, int k, size_t *bytes);
int sqllm_kmeans1d(const float *w, const float *s, int rows, int n, int k, float *centroids, uint8_t *labels,
                   void *workspace, size_t workspace_bytes, void *stream);

/* labels uint8 [out, in] (one row per output channel, as sqllm_kmeans1d gives them) -> qweight int32 [in/32*bits, out],
 * bit-identical to the reference's pack2 (quant.py:171-208).  in % 32 == 0; each label is taken modulo 2^bits. */
int sqllm_pack_indices(int bits, const uint8_t *labels, int in_features, int out_features, int32_t *qweight, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SQLLM_B200_H */
