// quant_cuda_pybind.cpp - the Python module `quant_cuda`: same 12 function names, positional
// signatures and accumulate-into-`mul` semantics as the reference's pybind module
// (squeezellm/quant_cuda.cpp:112-270), implemented as a thin torch::Tensor -> C ABI adapter over
// libsqllm_b200.so (include/sqllm_b200.h).  No kernels live here.
//
// Deliberate differences from the reference wrapper (all "more defined", none changes results):
//   * arguments are validated (device, dtype, contiguity, shapes) and violations raise RuntimeError;
//     the reference has no checks (SURVEY.md section 8(b));
//   * kernels are launched on PyTorch's CURRENT stream (the reference uses the legacy default
//     stream, quant_cuda_kernel.cu:147,172,...), so the calls are CUDA-graph capturable;
//   * `*_balanced_*` is not exported, exactly as in the reference (quant.py:238,282 reference a
//     symbol that quant_cuda.cpp never defines).
// Extra, not in the reference: `lutgemv_fused`, `lutgemm_fused`, `lutgemv_rows`, `lutgemv_rows_bf16`, `lutgemm_t`, `lut_grad`, `dequantize`, `fisher_accumulate`, `attn_decode`, `attn_decode_batch`, `attn_extend`, `attn_verify`, `attn_decode_paged`, `attn_extend_paged`, `attn_extend_batch`, `attn_extend_batch_paged`, `sample`, `unpack_indices`, `abi_version`,
// `fused_limits`.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cuda_runtime.h>

#include <cmath>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "sqllm_b200.h"

namespace {

void check_status(int rc, const char *what) { TORCH_CHECK(rc == SQLLM_OK, what, ": ", sqllm_last_error()); }

void need(const torch::Tensor &t, const char *name, c10::ScalarType dt, const torch::Tensor &like) {
    TORCH_CHECK(t.defined(), name, " is undefined");
    TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
    TORCH_CHECK(t.device() == like.device(), name, " is on ", t.device(), " but vec is on ", like.device());
    TORCH_CHECK(t.scalar_type() == dt, name, " must have dtype ", dt, " (got ", t.scalar_type(), ")");
    TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

void *cur_stream() { return static_cast<void *>(at::cuda::getCurrentCUDAStream().stream()); }

struct Dense {
    const float *vec;
    const int32_t *mat;
    float *mul;
    const float *lut;
    int height, width, batch, vec_height;
};

Dense check_dense(int bits, const torch::Tensor &vec, const torch::Tensor &mat, const torch::Tensor &mul,
                  const torch::Tensor &lut, bool batched) {
    need(vec, "vec", torch::kFloat32, vec);
    need(mat, "mat", torch::kInt32, vec);
    need(mul, "mul", torch::kFloat32, vec);
    need(lut, "lookup_table", torch::kFloat32, vec);
    TORCH_CHECK(mat.dim() == 2, "mat must be 2-D [in/32*bits, out]");
    Dense d;
    d.height = (int)mat.size(0);
    d.width = (int)mat.size(1);
    TORCH_CHECK(d.height % bits == 0, "mat has ", d.height, " rows, not a multiple of bits=", bits);
    const int64_t K = (int64_t)d.height / bits * 32;
    if (batched) {
        TORCH_CHECK(vec.dim() == 2, "batched vec must be 2-D [batch, in]");
        d.batch = (int)vec.size(0);
        d.vec_height = (int)vec.size(1);
        TORCH_CHECK(mul.numel() == (int64_t)d.batch * d.width, "mul must have batch*out = ", (int64_t)d.batch * d.width, " elements");
    } else {
        d.batch = 1;
        d.vec_height = (int)vec.numel();
        TORCH_CHECK(mul.numel() == d.width, "mul must have out = ", d.width, " elements (got ", mul.numel(), ")");
    }
    TORCH_CHECK(d.vec_height == K, "vec has ", d.vec_height, " features but mat implies ", K);
    TORCH_CHECK(lut.numel() == (int64_t)d.width * (1 << bits), "lookup_table must be [out, 2^bits]");
    d.vec = vec.data_ptr<float>();
    d.mat = mat.data_ptr<int32_t>();
    d.mul = mul.data_ptr<float>();
    d.lut = lut.data_ptr<float>();
    return d;
}

void check_csr(const torch::Tensor &rows, const torch::Tensor &cols, const torch::Tensor &vals, const torch::Tensor &vec,
               int num_rows, int width) {
    need(rows, "rows", torch::kInt32, vec);
    need(cols, "cols", torch::kInt32, vec);
    need(vals, "mat (CSR values)", torch::kFloat32, vec);
    TORCH_CHECK(num_rows == width, "num_rows=", num_rows, " must equal the packed matrix width ", width);
    TORCH_CHECK(rows.numel() == (int64_t)num_rows + 1, "rows must have num_rows+1 entries");
    TORCH_CHECK(cols.numel() == vals.numel(), "cols and vals differ in length");
}

void check_full(const torch::Tensor &full_rows, const torch::Tensor &fri, const torch::Tensor &vec, int64_t K) {
    need(full_rows, "full_rows", torch::kFloat32, vec);
    need(fri, "full_row_indices", torch::kInt32, vec);
    TORCH_CHECK(full_rows.dim() == 2 && full_rows.size(0) == K, "full_rows must be [in, topX]");
    TORCH_CHECK(fri.numel() == full_rows.size(1), "full_row_indices must have topX entries");
}

// ---- dense ------------------------------------------------------------------------------------
template <int BITS, bool BATCHED>
void dense(torch::Tensor vec, torch::Tensor mat, torch::Tensor mul, torch::Tensor lookup_table) {
    const at::cuda::OptionalCUDAGuard guard(device_of(vec));
    const Dense d = check_dense(BITS, vec, mat, mul, lookup_table, BATCHED);
    int rc;
    if (BITS == 3) rc = BATCHED ? sqllm_vecquant3matmul_nuq_perchannel_batched(d.vec, d.mat, d.mul, d.lut, d.height, d.width, d.batch, d.vec_height, cur_stream())
                                : sqllm_vecquant3matmul_nuq_perchannel(d.vec, d.mat, d.mul, d.lut, d.height, d.width, cur_stream());
    else rc = BATCHED ? sqllm_vecquant4matmul_nuq_perchannel_batched(d.vec, d.mat, d.mul, d.lut, d.height, d.width, d.batch, d.vec_height, cur_stream())
                      : sqllm_vecquant4matmul_nuq_perchannel(d.vec, d.mat, d.mul, d.lut, d.height, d.width, cur_stream());
    check_status(rc, "quant_cuda dense LUT matmul");
}

// ---- dense + CSR ------------------------------------------------------------------------------
template <int BITS, bool BATCHED>
void spmv(torch::Tensor rows, torch::Tensor cols, torch::Tensor mat, torch::Tensor vec, torch::Tensor mul, int num_rows,
          torch::Tensor matq, torch::Tensor lookup_table) {
    const at::cuda::OptionalCUDAGuard guard(device_of(vec));
    const Dense d = check_dense(BITS, vec, matq, mul, lookup_table, BATCHED);
    check_csr(rows, cols, mat, vec, num_rows, d.width);
    const int32_t *r = rows.data_ptr<int32_t>(), *c = cols.data_ptr<int32_t>();
    const float *v = mat.data_ptr<float>();
    int rc;
    if (BITS == 3) rc = BATCHED ? sqllm_vecquant3matmul_spmv_nuq_perchannel_batched(r, c, v, d.vec, d.mul, num_rows, d.mat, d.lut, d.height, d.width, d.batch, d.vec_height, cur_stream())
                                : sqllm_vecquant3matmul_spmv_nuq_perchannel(r, c, v, d.vec, d.mul, num_rows, d.mat, d.lut, d.height, d.width, cur_stream());
    else rc = BATCHED ? sqllm_vecquant4matmul_spmv_nuq_perchannel_batched(r, c, v, d.vec, d.mul, num_rows, d.mat, d.lut, d.height, d.width, d.batch, d.vec_height, cur_stream())
                      : sqllm_vecquant4matmul_spmv_nuq_perchannel(r, c, v, d.vec, d.mul, num_rows, d.mat, d.lut, d.height, d.width, cur_stream());
    check_status(rc, "quant_cuda LUT matmul + spmv");
}

// ---- dense + CSR + topX dense rows ------------------------------------------------------------
template <int BITS, bool BATCHED>
void hybrid(torch::Tensor rows, torch::Tensor cols, torch::Tensor mat, torch::Tensor vec, torch::Tensor full_rows,
            torch::Tensor full_row_indices, torch::Tensor mul, int num_rows, torch::Tensor matq, torch::Tensor lookup_table) {
    const at::cuda::OptionalCUDAGuard guard(device_of(vec));
    const Dense d = check_dense(BITS, vec, matq, mul, lookup_table, BATCHED);
    check_csr(rows, cols, mat, vec, num_rows, d.width);
    check_full(full_rows, full_row_indices, vec, d.vec_height);
    const int32_t *r = rows.data_ptr<int32_t>(), *c = cols.data_ptr<int32_t>(), *fi = full_row_indices.data_ptr<int32_t>();
    const float *v = mat.data_ptr<float>(), *fr = full_rows.data_ptr<float>();
    const int frh = (int)full_rows.size(0), frw = (int)full_rows.size(1);
    int rc;
    if (BITS == 3) rc = BATCHED ? sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel_batched(r, c, v, d.vec, fr, fi, d.mul, num_rows, d.mat, d.lut, d.height, d.width, frh, frw, d.batch, d.vec_height, cur_stream())
                                : sqllm_vecquant3matmul_spmv_hybrid_nuq_perchannel(r, c, v, d.vec, fr, fi, d.mul, num_rows, d.mat, d.lut, d.height, d.width, frh, frw, cur_stream());
    else rc = BATCHED ? sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel_batched(r, c, v, d.vec, fr, fi, d.mul, num_rows, d.mat, d.lut, d.height, d.width, frh, frw, d.batch, d.vec_height, cur_stream())
                      : sqllm_vecquant4matmul_spmv_hybrid_nuq_perchannel(r, c, v, d.vec, fr, fi, d.mul, num_rows, d.mat, d.lut, d.height, d.width, frh, frw, cur_stream());
    check_status(rc, "quant_cuda LUT matmul + spmv + dense rows");
}

// ---- fused module path ------------------------------------------------------------------------
// Workspace of the fused path: one per (device, stream), allocated on first use (so: before any graph capture on that stream -
// GraphedDecodeStep warms up for exactly this reason), at least 8 MB - every supported shape fits, it is never regrown in
// practice; if it ever is, the old one is kept alive for graphs that captured its address.  A workspace serialises the launches
// that use it: graphs captured on the SAME stream must not be replayed concurrently on different streams (they share it);
// capture them on different streams if they have to overlap.
std::mutex g_ws_mutex;
std::map<std::pair<int, void *>, torch::Tensor> g_ws;  // (device, stream) -> zero-initialised workspace
std::vector<torch::Tensor> g_ws_retired;               // outgrown workspaces: never freed, a captured CUDA graph may still point at them

// the workspace of the current (device, stream) for the fused call of layer a, on like's device
torch::Tensor workspace_for(const torch::Tensor &like, const sqllm_lutgemv_args &a) {
    const size_t bytes = sqllm_workspace_bytes(a.bits, a.in_features, a.out_features, a.topX);
    TORCH_CHECK(bytes > 0, "sqllm_workspace_bytes failed: ", sqllm_last_error());
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    const auto key = std::make_pair((int)like.get_device(), cur_stream());
    auto it = g_ws.find(key);
    if (it == g_ws.end() || (size_t)it->second.numel() < bytes) {
        // grow generously so that the allocation happens once (and never during graph capture of a later call)
        const size_t cap = std::max<size_t>(bytes, 8u << 20);
        torch::Tensor ws = torch::zeros({(int64_t)cap}, torch::TensorOptions().dtype(torch::kUInt8).device(like.device()));
        if (it != g_ws.end()) g_ws_retired.push_back(it->second);
        g_ws[key] = ws;
        return ws;
    }
    return it->second;
}

// shared argument checking / descriptor filling of the fused entry points: everything but the dtype and the shape of x (each
// binding checks those)
void fill_layer_args(sqllm_lutgemv_args &a, const float *&bias_p, const torch::Tensor &x, const torch::Tensor &qweight,
                     const torch::Tensor &lookup_table, int bits, const c10::optional<torch::Tensor> &bias,
                     const c10::optional<torch::Tensor> &rows, const c10::optional<torch::Tensor> &cols,
                     const c10::optional<torch::Tensor> &vals, const c10::optional<torch::Tensor> &full_rows,
                     const c10::optional<torch::Tensor> &full_row_indices) {
    TORCH_CHECK(x.is_cuda() && x.is_contiguous(), "x must be a contiguous CUDA tensor");
    TORCH_CHECK(bits == 3 || bits == 4, "bits must be 3 or 4");
    need(qweight, "qweight", torch::kInt32, x);
    need(lookup_table, "lookup_table", torch::kFloat32, x);
    TORCH_CHECK(qweight.dim() == 2 && qweight.size(0) % bits == 0, "qweight must be [in/32*bits, out]");
    memset(&a, 0, sizeof(a));
    a.bits = bits;
    a.in_features = (int)(qweight.size(0) / bits * 32);
    a.out_features = (int)qweight.size(1);
    a.batch = 1;
    TORCH_CHECK(lookup_table.numel() == (int64_t)a.out_features * (1 << bits), "lookup_table must be [out, 2^bits]");
    a.qweight = qweight.data_ptr<int32_t>();
    a.lookup_table = lookup_table.data_ptr<float>();
    bias_p = nullptr;
    if (bias.has_value() && bias->defined()) {
        need(*bias, "bias", torch::kFloat32, x);
        TORCH_CHECK(bias->numel() == a.out_features, "bias must have out_features elements");
        bias_p = bias->data_ptr<float>();
    }
    if (rows.has_value() && rows->defined()) {
        TORCH_CHECK(cols.has_value() && vals.has_value(), "rows given without cols / vals");
        check_csr(*rows, *cols, *vals, x, a.out_features, a.out_features);
        a.rows = rows->data_ptr<int32_t>();
        a.cols = cols->data_ptr<int32_t>();
        a.vals = vals->data_ptr<float>();
    }
    if (full_rows.has_value() && full_rows->defined() && full_rows->numel() > 0) {
        TORCH_CHECK(full_row_indices.has_value(), "full_rows given without full_row_indices");
        check_full(*full_rows, *full_row_indices, x, a.in_features);
        a.full_rows = full_rows->data_ptr<float>();
        a.full_row_indices = full_row_indices->data_ptr<int32_t>();
        a.topX = (int)full_rows->size(1);
    }
}

// ... of the matvec entry points: x holds one input vector
void fill_fused_args(sqllm_lutgemv_args &a, const float *&bias_p, const torch::Tensor &x, const torch::Tensor &qweight,
                     const torch::Tensor &lookup_table, int bits, const c10::optional<torch::Tensor> &bias,
                     const c10::optional<torch::Tensor> &rows, const c10::optional<torch::Tensor> &cols,
                     const c10::optional<torch::Tensor> &vals, const c10::optional<torch::Tensor> &full_rows,
                     const c10::optional<torch::Tensor> &full_row_indices) {
    fill_layer_args(a, bias_p, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices);
    TORCH_CHECK(x.numel() == a.in_features, "x has ", x.numel(), " elements, expected in_features=", a.in_features);
}

// SQLLM_DT_* of an fp32 / fp16 / bf16 tensor
int dtype_code(const torch::Tensor &t, const char *what) {
    switch (t.scalar_type()) {
        case torch::kFloat32: return SQLLM_DT_F32;
        case torch::kFloat16: return SQLLM_DT_F16;
        case torch::kBFloat16: return SQLLM_DT_BF16;
        default: TORCH_CHECK(false, what, " must be fp16, bf16 or fp32 (got ", t.scalar_type(), ")");
    }
    return -1;
}

// "path" of lutgemm_t and lut_grad -> the path code of sqllm_lutgemm_t / sqllm_lut_grad
int path_code(const std::string &path, const char *name) {
    TORCH_CHECK(path == "auto" || path == "tc" || path == "cuda", name, ": path must be 'auto', 'tc' or 'cuda' (got '", path, "')");
    return path == "auto" ? 0 : path == "tc" ? 1 : 2;
}

// The bindings x [M, in] -> y [M, out] in x's dtype: the shape checks, y and the call of `entry` (sqllm_lutgemm_fused_dt or
// sqllm_lutgemv_rows_dt, or sqllm_lutgemm_fused_f32 through lutgemm_f32_entry).  The binding `name` has checked x's dtype.
typedef int (*RowsEntry)(const sqllm_lutgemv_args *, const void *, int, void *, int, const float *, void *);
torch::Tensor layer_rows(const char *name, RowsEntry entry, const torch::Tensor &x, const torch::Tensor &qweight,
                         const torch::Tensor &lookup_table, int bits, const c10::optional<torch::Tensor> &bias,
                         const c10::optional<torch::Tensor> &rows, const c10::optional<torch::Tensor> &cols,
                         const c10::optional<torch::Tensor> &vals, const c10::optional<torch::Tensor> &full_rows,
                         const c10::optional<torch::Tensor> &full_row_indices) {
    const at::cuda::OptionalCUDAGuard guard(device_of(x));
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_layer_args(a, bias_p, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices);
    TORCH_CHECK(x.dim() == 2 && x.size(1) == a.in_features, name, ": x must be [M, in_features=", a.in_features, "]");
    TORCH_CHECK(x.size(0) >= 1 && x.size(0) <= INT32_MAX, name, ": x must have 1 to 2^31-1 rows");
    a.batch = (int)x.size(0);
    torch::Tensor y = torch::empty({x.size(0), (int64_t)a.out_features}, x.options());
    const int dt = dtype_code(x, "x");
    const int rc = entry(&a, x.data_ptr(), dt, y.data_ptr(), dt, bias_p, cur_stream());
    TORCH_CHECK(rc == SQLLM_OK, "quant_cuda.", name, ": ", sqllm_last_error());
    return y;
}

// y [M, out] = bias + LUT-GEMM(x) [+ CSR] [+ dense rows] from fp16 or bf16 x [M, in], in x's dtype, on the tensor cores
// (sqllm_lutgemm_fused_dt): QuantLinearLUT.forward's batched branch (squeezellm/quant.py:314-379) in one launch.
torch::Tensor lutgemm_fused(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                            c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                            c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                            c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices) {
    TORCH_CHECK(x.scalar_type() == torch::kFloat16 || x.scalar_type() == torch::kBFloat16,
                "lutgemm_fused: x must be fp16 or bf16 (got ", x.scalar_type(), ")");
    return layer_rows("lutgemm_fused", sqllm_lutgemm_fused_dt, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows,
                      full_row_indices);
}

// sqllm_lutgemm_fused_f32 behind layer_rows' entry signature (the dtype codes are SQLLM_DT_F32: lutgemm_fused_f32 checked x)
int lutgemm_f32_entry(const sqllm_lutgemv_args *a, const void *x, int, void *y, int, const float *bias, void *stream) {
    return sqllm_lutgemm_fused_f32(a, static_cast<const float *>(x), static_cast<float *>(y), bias, stream);
}

// The same for fp32 x [M, in] -> fp32 y [M, out] (sqllm_lutgemm_fused_f32: x split exactly into three bf16 parts, six part
// products per k-step): QuantLinearLUT.forward's batched branch for QuantLinearLUT.FP32_TC_MIN_ROWS or more fp32 rows.  A symbol
// of its own, so that lutgemm_fused keeps meaning "16-bit x".
torch::Tensor lutgemm_fused_f32(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                                c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                                c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                                c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices) {
    TORCH_CHECK(x.scalar_type() == torch::kFloat32, "lutgemm_fused_f32: x must be fp32 (got ", x.scalar_type(), ")");
    return layer_rows("lutgemm_fused_f32", lutgemm_f32_entry, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows,
                      full_row_indices);
}

// y [M, out] fp16 = bias + LUT-GEMV(x) [+ CSR] [+ dense rows] from fp16 x [M, in], a few rows on the CUDA cores (sqllm_lutgemv_rows_dt):
// QuantLinearLUT.forward's batched branch for 2 to QuantLinearLUT.ROWS_MAX rows in one launch.  bf16 x: lutgemv_rows_bf16.
torch::Tensor lutgemv_rows(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                           c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                           c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                           c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices) {
    // bf16 x is refused with the message of the fp16 / fp32 decode bindings (it has lutgemv_rows_bf16), fp32 x with its own
    TORCH_CHECK(x.scalar_type() == torch::kFloat16 || x.scalar_type() == torch::kFloat32, "x must be fp16 or fp32");
    TORCH_CHECK(x.scalar_type() == torch::kFloat16, "lutgemv_rows: x must be fp16");
    return layer_rows("lutgemv_rows", sqllm_lutgemv_rows_dt, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows,
                      full_row_indices);
}

// The same for bf16 x [M, in] -> bf16 y [M, out] (sqllm_lutgemv_rows_dt): QuantLinearLUT.forward's batched branch for 2 to
// QuantLinearLUT.BF16_ROWS_MAX bf16 rows.  A symbol of its own, so that lutgemv_rows keeps meaning "the fp16 rows route".
torch::Tensor lutgemv_rows_bf16(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                                c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                                c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                                c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices) {
    TORCH_CHECK(x.scalar_type() == torch::kBFloat16, "lutgemv_rows_bf16: x must be bf16 (got ", x.scalar_type(), ")");
    return layer_rows("lutgemv_rows_bf16", sqllm_lutgemv_rows_dt, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows,
                      full_row_indices);
}

// dx [M, in] = dy [M, out] . W^T (LUT + CSR + dense rows), in dy's dtype (fp16, bf16 or fp32): the input gradient of
// QuantLinearLUT (sqllm_lutgemm_t).  path: "auto" (the library picks), "tc" (tensor cores) or "cuda" (CUDA cores).
torch::Tensor lutgemm_t(torch::Tensor dy, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                        c10::optional<torch::Tensor> rows, c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                        c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices,
                        const std::string &path) {
    const at::cuda::OptionalCUDAGuard guard(device_of(dy));
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_layer_args(a, bias_p, dy, qweight, lookup_table, bits, c10::nullopt, rows, cols, vals, full_rows, full_row_indices);
    const int dt = dtype_code(dy, "lutgemm_t: dy");
    const int pc = path_code(path, "lutgemm_t");
    TORCH_CHECK(dy.dim() == 2 && dy.size(1) == a.out_features, "lutgemm_t: dy must be [M, out_features=", a.out_features, "]");
    TORCH_CHECK(dy.size(0) >= 1 && dy.size(0) <= INT32_MAX, "lutgemm_t: dy must have 1 to 2^31-1 rows");
    a.batch = (int)dy.size(0);
    torch::Tensor dx = torch::empty({dy.size(0), (int64_t)a.in_features}, dy.options());
    check_status(sqllm_lutgemm_t(&a, dy.data_ptr(), dt, dx.data_ptr(), dt, pc, cur_stream()), "quant_cuda.lutgemm_t");
    return dx;
}

// (dlut [out, 2^bits], dvals [nnz], dfull_rows [in, topX]) fp32 from x [M, in] and dy [M, out] (sqllm_lut_grad): the gradients of
// QuantLinearLUT's codebook, CSR values and dense rows, one launch; None for an output not asked for.  path: "auto", "tc" or "cuda".
py::tuple lut_grad(torch::Tensor x, torch::Tensor dy, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                   c10::optional<torch::Tensor> rows, c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                   c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices, bool want_lut, bool want_vals,
                   bool want_full_rows, const std::string &path) {
    const at::cuda::OptionalCUDAGuard guard(device_of(x));
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_layer_args(a, bias_p, x, qweight, lookup_table, bits, c10::nullopt, rows, cols, vals, full_rows, full_row_indices);
    const int xdt = dtype_code(x, "lut_grad: x"), dydt = dtype_code(dy, "lut_grad: dy");
    TORCH_CHECK(dy.is_cuda() && dy.is_contiguous() && dy.device() == x.device(), "lut_grad: dy must be a contiguous CUDA tensor on x's device");
    const int pc = path_code(path, "lut_grad");
    TORCH_CHECK(x.dim() == 2 && x.size(1) == a.in_features, "lut_grad: x must be [M, in_features=", a.in_features, "]");
    TORCH_CHECK(dy.dim() == 2 && dy.size(1) == a.out_features && dy.size(0) == x.size(0),
                "lut_grad: dy must be [M=", x.size(0), ", out_features=", a.out_features, "]");
    TORCH_CHECK(x.size(0) >= 1 && x.size(0) <= INT32_MAX, "lut_grad: x must have 1 to 2^31-1 rows");
    TORCH_CHECK(want_lut || want_vals || want_full_rows, "lut_grad: nothing requested (want_lut, want_vals and want_full_rows are all False)");
    TORCH_CHECK(!want_vals || a.rows, "lut_grad: want_vals needs the CSR arrays rows / cols / vals");
    TORCH_CHECK(!want_full_rows || a.topX > 0, "lut_grad: want_full_rows needs full_rows / full_row_indices");
    a.batch = (int)x.size(0);
    const auto f32 = x.options().dtype(torch::kFloat32);
    torch::Tensor dlut, dvals, dfull;
    if (want_lut) dlut = torch::empty({(int64_t)a.out_features, (int64_t)1 << bits}, f32);
    if (want_vals) dvals = torch::zeros({vals->numel()}, f32);  // entries outside the CSR rows' range [rows[0], rows[out]) stay 0
    if (want_full_rows) dfull = torch::empty({(int64_t)a.in_features, (int64_t)a.topX}, f32);
    float *pl = want_lut ? dlut.data_ptr<float>() : nullptr, *pv = want_vals && dvals.numel() ? dvals.data_ptr<float>() : nullptr;
    float *pf = want_full_rows ? dfull.data_ptr<float>() : nullptr;
    if (pl || pv || pf)  // else only an empty dvals was asked for
        check_status(sqllm_lut_grad(&a, x.data_ptr(), xdt, dy.data_ptr(), dydt, pl, pv, pf, pc, cur_stream()), "quant_cuda.lut_grad");
    auto opt = [](const torch::Tensor &t) -> py::object { return t.defined() ? py::cast(t) : py::none(); };
    return py::make_tuple(opt(dlut), opt(dvals), opt(dfull));
}

// y = bias + LUT-GEMV(x) [+ CSR] [+ dense rows]; x fp16 / bf16 / fp32 with numel == in; returns [out] in x's dtype
// (QuantLinearLUT.forward's matvec branch, squeezellm/quant.py:212-312, in one launch).
torch::Tensor lutgemv_fused(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                            c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                            c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                            c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices) {
    const at::cuda::OptionalCUDAGuard guard(device_of(x));
    TORCH_CHECK(x.scalar_type() == torch::kFloat16 || x.scalar_type() == torch::kFloat32 || x.scalar_type() == torch::kBFloat16,
                "x must be fp16, bf16 or fp32");
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_fused_args(a, bias_p, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices);
    torch::Tensor ws = workspace_for(x, a);
    torch::Tensor y = torch::empty({(int64_t)a.out_features}, x.options());
    const int dt = dtype_code(x, "lutgemv_fused: x");
    const int rc = sqllm_lutgemv_fused_dt(&a, x.data_ptr(), dt, y.data_ptr(), dt, bias_p, ws.data_ptr(), (size_t)ws.numel(), cur_stream());
    check_status(rc, "quant_cuda.lutgemv_fused");
    return y;
}

// Column shard with the exchange built in (include/sqllm_b200.h, sqllm_lutgemv_fused_exchange_dt): the result is written into every
// rank's symmetric arena in x's dtype; nothing is returned.  The binding `name` has checked x's dtype.  peer_base: address of the device array of arena base addresses.
void exchange_call(const char *name, torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                   c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows, c10::optional<torch::Tensor> cols,
                   c10::optional<torch::Tensor> vals, c10::optional<torch::Tensor> full_rows,
                   c10::optional<torch::Tensor> full_row_indices, int64_t peer_base, int64_t out_offset, int64_t flag_offset,
                   int64_t state_offset, int64_t error_offset, int world, int rank, int members, int out_features_full) {
    const at::cuda::OptionalCUDAGuard guard(device_of(x));
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_fused_args(a, bias_p, x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices);
    torch::Tensor ws = workspace_for(x, a);
    sqllm_exchange xc;
    memset(&xc, 0, sizeof(xc));
    xc.world = world; xc.rank = rank; xc.members = members; xc.out_features_full = out_features_full;
    xc.peer_base = reinterpret_cast<const uint64_t *>(peer_base);
    xc.out_offset = (size_t)out_offset; xc.flag_offset = (size_t)flag_offset; xc.state_offset = (size_t)state_offset; xc.error_offset = (size_t)error_offset;
    const int dt = dtype_code(x, name);  // the arena vectors are in x's dtype
    const int rc = sqllm_lutgemv_fused_exchange_dt(&a, x.data_ptr(), dt, dt, bias_p, ws.data_ptr(), (size_t)ws.numel(), &xc, cur_stream());
    check_status(rc, (std::string("quant_cuda.") + name).c_str());
}

// fp16 or fp32 x; the vectors in x's dtype.  bf16 x: lutgemv_fused_exchange_bf16.
void lutgemv_fused_exchange(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                            c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                            c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                            c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices,
                            int64_t peer_base, int64_t out_offset, int64_t flag_offset, int64_t state_offset, int64_t error_offset,
                            int world, int rank, int members, int out_features_full) {
    TORCH_CHECK(x.scalar_type() == torch::kFloat16 || x.scalar_type() == torch::kFloat32, "x must be fp16 or fp32");
    exchange_call("lutgemv_fused_exchange", x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices,
                  peer_base, out_offset, flag_offset, state_offset, error_offset, world, rank, members, out_features_full);
}

// The same for bf16 x, bf16 vectors in the arenas.  A symbol of its own, so that lutgemv_fused_exchange keeps its fp16 / fp32 contract
// (as lutgemv_rows / lutgemv_rows_bf16).
void lutgemv_fused_exchange_bf16(torch::Tensor x, torch::Tensor qweight, torch::Tensor lookup_table, int bits,
                                 c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> rows,
                                 c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals,
                                 c10::optional<torch::Tensor> full_rows, c10::optional<torch::Tensor> full_row_indices,
                                 int64_t peer_base, int64_t out_offset, int64_t flag_offset, int64_t state_offset, int64_t error_offset,
                                 int world, int rank, int members, int out_features_full) {
    TORCH_CHECK(x.scalar_type() == torch::kBFloat16, "lutgemv_fused_exchange_bf16: x must be bf16 (got ", x.scalar_type(), ")");
    exchange_call("lutgemv_fused_exchange_bf16", x, qweight, lookup_table, bits, bias, rows, cols, vals, full_rows, full_row_indices,
                  peer_base, out_offset, flag_offset, state_offset, error_offset, world, rank, members, out_features_full);
}


// ---- sequences (include/sqllm_b200.h, sqllm_sequence_*): one persistent launch for a list of dependent fused matvecs -----------
// items: list of tuples (qweight, lookup_table, bits, bias|None, rows|None, cols|None, vals|None, full_rows|None, full_row_indices|None,
//                        x_from, x_offset, x_ext|None, members, out_features_full)
// exports: list of (item index, destination tensor of the item's full output length).  dtype: the activation type, torch.float16 or
// torch.bfloat16 (sqllm_sequence_create_dt): every x_ext and every export destination has it.  The caller keeps every tensor alive for
// the life of the handle (squeezellm_b200.runtime.DecodeSequence does).  peer_base / arena: several GPUs only (0 / None otherwise).
// ops (keyword, sqllm_sequence_create_ops): None, or one entry per item: None (nothing) or a tuple
//     (x_op, norm_weight|None, eps, x2_from, x2_offset, res_from, res_offset, res_ext|None)
// with x_op 0 plain, 1 RMSNorm, 2 SiLU gating; norm_weight and res_ext contiguous CUDA tensors of the sequence's dtype.  The op checks
// that need no item (x_op, eps, which items the sources name, the tensors) come first; the rest are the C entry point's.
std::vector<sqllm_seq_op> sequence_ops(const py::object &ops, int n, at::ScalarType dtype, const char *tn) {
    std::vector<sqllm_seq_op> v;
    if (ops.is_none()) return v;
    py::list l = ops.cast<py::list>();
    TORCH_CHECK((int)l.size() == n, "sequence_create: ", l.size(), " ops for ", n, " items");
    v.resize(n);
    for (int i = 0; i < n; ++i) {
        sqllm_seq_op &o = v[i];
        memset(&o, 0, sizeof(o));
        o.x2_from = o.res_from = -1;
        if (l[i].is_none()) continue;
        py::tuple t = l[i].cast<py::tuple>();
        TORCH_CHECK(t.size() == 8, "sequence op ", i, ": expected None or an 8-tuple (x_op, norm_weight, eps, x2_from, x2_offset, res_from, res_offset, res_ext)");
        o.x_op = t[0].cast<int>();
        o.eps = t[2].cast<float>();
        o.x2_from = t[3].cast<int>(); o.x2_offset = t[4].cast<int>();
        o.res_from = t[5].cast<int>(); o.res_offset = t[6].cast<int>();
        TORCH_CHECK(o.x_op == SQLLM_SEQ_X_PLAIN || o.x_op == SQLLM_SEQ_X_RMSNORM || o.x_op == SQLLM_SEQ_X_SILU_MUL, "sequence item ", i, ": unknown x_op=", o.x_op);
        auto vec = [&](int k, const char *name) -> const void * {
            if (t[k].is_none()) return nullptr;
            torch::Tensor w = t[k].cast<torch::Tensor>();
            TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.scalar_type() == dtype, "sequence item ", i, ": ", name, " must be a contiguous ", tn,
                        " CUDA tensor (the sequence's dtype; got ", w.scalar_type(), w.is_cuda() ? "" : " on the CPU", ")");
            return w.data_ptr();
        };
        o.norm_weight = vec(1, "norm_weight");
        o.res_ext = vec(7, "res_ext");
        if (o.x_op == SQLLM_SEQ_X_RMSNORM) {
            TORCH_CHECK(o.norm_weight, "sequence item ", i, ": RMSNorm needs norm_weight");
            TORCH_CHECK(std::isfinite(o.eps) && o.eps >= 0.f, "sequence item ", i, ": eps=", o.eps, " must be finite and >= 0");
        }
        if (o.x_op == SQLLM_SEQ_X_SILU_MUL)
            TORCH_CHECK(o.x2_from >= 0 && o.x2_from < i, "sequence item ", i, ": x2_from=", o.x2_from, " must name an earlier item");
        TORCH_CHECK(o.res_from >= -1 && o.res_from < i, "sequence item ", i, ": residual source res_from=", o.res_from, " must name an earlier item (or -1)");
    }
    return v;
}

int64_t sequence_create(py::list items, py::list exports, const std::string &lut_mode, int world, int rank,
                        c10::optional<torch::Tensor> arena, int64_t peer_base, at::ScalarType dtype, py::object ops) {
    TORCH_CHECK(lut_mode == "exact" || lut_mode == "fp16", "lut mode must be 'exact' or 'fp16'");
    TORCH_CHECK(dtype == torch::kFloat16 || dtype == torch::kBFloat16, "sequence_create: dtype must be torch.float16 or torch.bfloat16 (got ", dtype, ")");
    const bool bf = dtype == torch::kBFloat16;
    const char *const tn = bf ? "bf16" : "fp16";
    const int n = (int)items.size();
    TORCH_CHECK(n > 0, "sequence_create: no items");
    const std::vector<sqllm_seq_op> sops = sequence_ops(ops, n, dtype, tn);
    std::vector<sqllm_seq_item> its(n);
    c10::optional<torch::Tensor> first;
    for (int i = 0; i < n; ++i) {
        py::tuple t = items[i].cast<py::tuple>();
        TORCH_CHECK(t.size() == 14, "sequence item ", i, ": expected a 14-tuple");
        auto opt = [&](int k) -> c10::optional<torch::Tensor> {
            if (t[k].is_none()) return c10::nullopt;
            return t[k].cast<torch::Tensor>();
        };
        torch::Tensor qweight = t[0].cast<torch::Tensor>(), lut = t[1].cast<torch::Tensor>();
        const int bits = t[2].cast<int>();
        sqllm_seq_item &it = its[i];
        memset(&it, 0, sizeof(it));
        it.x_from = t[9].cast<int>();
        it.x_offset = t[10].cast<int>();
        it.members = t[12].cast<int>();
        it.out_features_full = t[13].cast<int>();
        TORCH_CHECK(qweight.is_cuda() && qweight.dim() == 2 && (bits == 3 || bits == 4), "sequence item ", i, ": qweight must be a packed CUDA matrix");
        const int K = (int)(qweight.size(0) / bits * 32);
        torch::Tensor xs;  // what the shared checks look at (device, numel): the external input, or a stand-in of the right length
        if (it.x_from < 0) {
            TORCH_CHECK(!t[11].is_none(), "sequence item ", i, ": x_from = -1 needs x_ext");
            xs = t[11].cast<torch::Tensor>();
            TORCH_CHECK(xs.scalar_type() == dtype, "sequence item ", i, ": x_ext must be ", tn, " (the sequence's dtype; got ", xs.scalar_type(), ")");
        } else {
            xs = torch::empty({(int64_t)K}, torch::TensorOptions().dtype(dtype).device(qweight.device()));
        }
        const float *bias_p = nullptr;
        fill_fused_args(it.a, bias_p, xs, qweight, lut, bits, opt(3), opt(4), opt(5), opt(6), opt(7), opt(8));
        if (it.x_from < 0) it.x_ext = xs.data_ptr();
        it.bias = bias_p;
        if (!first.has_value()) first = qweight;
    }
    const at::cuda::OptionalCUDAGuard guard(device_of(*first));
    const int ne = (int)exports.size();
    std::vector<int> ex_items(std::max(1, ne));
    std::vector<void *> ex_dst(std::max(1, ne));
    for (int e = 0; e < ne; ++e) {
        py::tuple t = exports[e].cast<py::tuple>();
        ex_items[e] = t[0].cast<int>();
        torch::Tensor d = t[1].cast<torch::Tensor>();
        TORCH_CHECK(d.is_cuda() && d.is_contiguous() && d.scalar_type() == dtype, "export ", e, ": destination must be a contiguous ", tn,
                    " CUDA tensor (the sequence's dtype; got ", d.scalar_type(), ")");
        TORCH_CHECK(ex_items[e] >= 0 && ex_items[e] < n, "export ", e, ": bad item index");
        const sqllm_seq_item &it = its[ex_items[e]];
        const int64_t len = (int64_t)(it.members > 0 ? it.members : 1) * (it.out_features_full > 0 ? it.out_features_full : it.a.out_features / std::max(1, it.members));
        TORCH_CHECK(d.numel() == len, "export ", e, ": destination has ", d.numel(), " elements, the item's output has ", len);
        ex_dst[e] = d.data_ptr();
    }
    sqllm_seq_options o;
    memset(&o, 0, sizeof(o));
    o.lut_mode = lut_mode == "fp16" ? SQLLM_LUT_FP16_PAIR : SQLLM_LUT_EXACT;
    o.world = world; o.rank = rank;
    if (arena.has_value() && arena->defined()) {
        o.arena = arena->data_ptr();
        o.arena_bytes = (size_t)arena->numel() * arena->element_size();
    }
    o.peer_base = reinterpret_cast<const uint64_t *>(peer_base);
    o.n_export = ne; o.export_items = ex_items.data(); o.export_dst = ex_dst.data();
    sqllm_sequence *h = nullptr;
    check_status(sqllm_sequence_create_ops(its.data(), sops.empty() ? nullptr : sops.data(), n, &o, bf ? SQLLM_DT_BF16 : SQLLM_DT_F16, &h),
                 "quant_cuda.sequence_create");
    return reinterpret_cast<int64_t>(h);
}

// W [ncols, in] in `dtype` (fp32, fp16 or bf16) = the dense weight of output channels [col0, col0 + ncols) (codebook + CSR + dense
// rows, sqllm_dequantize): QuantLinearLUT.dequantize.  ncols = -1: to the last channel.  A new tensor on qweight's device.
torch::Tensor dequantize(torch::Tensor qweight, torch::Tensor lookup_table, int bits, c10::optional<torch::Tensor> rows,
                         c10::optional<torch::Tensor> cols, c10::optional<torch::Tensor> vals, c10::optional<torch::Tensor> full_rows,
                         c10::optional<torch::Tensor> full_row_indices, at::ScalarType dtype, int64_t col0, int64_t ncols) {
    TORCH_CHECK(qweight.defined() && qweight.is_cuda() && qweight.is_contiguous(), "dequantize: qweight must be a contiguous CUDA tensor");
    const at::cuda::OptionalCUDAGuard guard(device_of(qweight));
    sqllm_lutgemv_args a;
    const float *bias_p;
    fill_layer_args(a, bias_p, qweight, qweight, lookup_table, bits, c10::nullopt, rows, cols, vals, full_rows, full_row_indices);
    TORCH_CHECK(dtype == torch::kFloat32 || dtype == torch::kFloat16 || dtype == torch::kBFloat16,
                "dequantize: dtype must be torch.float32, torch.float16 or torch.bfloat16 (got ", dtype, ")");
    if (ncols == -1) ncols = a.out_features - col0;
    TORCH_CHECK(col0 >= 0 && ncols >= 1 && col0 + ncols <= a.out_features, "dequantize: columns [col0=", col0, ", col0 + ncols=",
                col0 + ncols, ") must be non-empty and lie in [0, out_features=", a.out_features, ")");
    torch::Tensor w = torch::empty({ncols, (int64_t)a.in_features}, qweight.options().dtype(dtype));
    const int dt = dtype == torch::kFloat32 ? SQLLM_DT_F32 : dtype == torch::kFloat16 ? SQLLM_DT_F16 : SQLLM_DT_BF16;
    check_status(sqllm_dequantize(&a, (int)col0, (int)ncols, w.data_ptr(), dt, cur_stream()), "quant_cuda.dequantize");
    return w;
}

// fisher [out, in] fp32 += sum_s (dy_s^T x_s)^2 over the samples of seq_len rows of x [rows, in] and dy [rows, out], both fp16 or
// both bf16 (sqllm_fisher_accumulate), in place.
void fisher_accumulate(torch::Tensor x, torch::Tensor dy, torch::Tensor fisher, int64_t seq_len) {
    TORCH_CHECK(x.defined() && x.is_cuda() && x.is_contiguous(), "fisher_accumulate: x must be a contiguous CUDA tensor");
    TORCH_CHECK(dy.defined() && dy.is_cuda() && dy.is_contiguous(), "fisher_accumulate: dy must be a contiguous CUDA tensor");
    TORCH_CHECK(fisher.defined() && fisher.is_cuda() && fisher.is_contiguous(), "fisher_accumulate: fisher must be a contiguous CUDA tensor");
    TORCH_CHECK(dy.device() == x.device(), "fisher_accumulate: dy is on ", dy.device(), " but x is on ", x.device());
    TORCH_CHECK(fisher.device() == x.device(), "fisher_accumulate: fisher is on ", fisher.device(), " but x is on ", x.device());
    TORCH_CHECK(x.scalar_type() == torch::kFloat16 || x.scalar_type() == torch::kBFloat16,
                "fisher_accumulate: x must be fp16 or bf16 (got ", x.scalar_type(), ")");
    TORCH_CHECK(dy.scalar_type() == x.scalar_type(), "fisher_accumulate: dy must have x's dtype ", x.scalar_type(), " (got ", dy.scalar_type(), ")");
    TORCH_CHECK(fisher.scalar_type() == torch::kFloat32, "fisher_accumulate: fisher must be fp32 (got ", fisher.scalar_type(), ")");
    TORCH_CHECK(x.dim() == 2 && dy.dim() == 2, "fisher_accumulate: x must be [rows, in] and dy [rows, out]");
    TORCH_CHECK(dy.size(0) == x.size(0), "fisher_accumulate: dy has ", dy.size(0), " rows but x has ", x.size(0));
    TORCH_CHECK(fisher.dim() == 2 && fisher.size(0) == dy.size(1) && fisher.size(1) == x.size(1), "fisher_accumulate: fisher must be [out=",
                dy.size(1), ", in=", x.size(1), "] (got ", fisher.sizes(), ")");
    TORCH_CHECK(x.size(0) >= 1 && x.size(0) <= INT32_MAX, "fisher_accumulate: x must have 1 to 2^31-1 rows (got ", x.size(0), ")");
    TORCH_CHECK(x.size(1) <= INT32_MAX && dy.size(1) <= INT32_MAX, "fisher_accumulate: in and out must be below 2^31");
    TORCH_CHECK(seq_len >= 1 && x.size(0) % seq_len == 0, "fisher_accumulate: seq_len=", seq_len, " must be >= 1 and divide the ",
                x.size(0), " rows of x");
    const at::cuda::OptionalCUDAGuard guard(device_of(x));
    const int dt = x.scalar_type() == torch::kFloat16 ? SQLLM_DT_F16 : SQLLM_DT_BF16;
    check_status(sqllm_fisher_accumulate(x.data_ptr(), dy.data_ptr(), dt, (int)x.size(0), (int)seq_len, (int)x.size(1), (int)dy.size(1),
                                         fisher.data_ptr<float>(), cur_stream()),
                 "quant_cuda.fisher_accumulate");
}

// The argument checks attn_decode, attn_decode_batch, attn_extend and attn_verify share, in the order they run, each message prefixed
// with `fn`: every tensor contiguous and 16-byte aligned, qkv's dtype, the head layout, k_cache [batch (lead = 1 only), n_kv, capacity,
// head_dim], the batch, head_dim, capacity, scale, the cache and out dtypes and v_cache's shape; then own(batch, capacity, head_dim), the
// binding's own shape checks; then the rope tables.  The device checks come last, so that a CPU caller sees the same rejections.  pos:
// null for attn_extend.  -> the sqllm args with the fields the four share.
// table: the block table of attn_decode_paged and attn_extend_batch_paged ([batch, width], lead = 1) and attn_extend_paged ([width],
// lead = 0), null for the others.  With a table the caches are page pools [n_pages, n_kv, 64, head_dim], capacity is the rope tables' rows, the batch is the
// table's rows, and the table must be int32, contiguous and 4-byte aligned with width = ceil(capacity / 64).
template <typename Args, typename Own>
Args attn_args(const char *fn, int lead, const torch::Tensor &qkv, const torch::Tensor *pos, const torch::Tensor &rope_cos,
               const torch::Tensor &rope_sin, const torch::Tensor &k_cache, const torch::Tensor &v_cache, const torch::Tensor &out,
               int64_t n_heads, int64_t n_kv, double scale, Own own, const torch::Tensor *table = nullptr) {
    const std::pair<const torch::Tensor *, const char *> all[] = {{&qkv, "qkv"}, {pos, "pos"}, {&rope_cos, "rope_cos"}, {&rope_sin, "rope_sin"},
                                                                  {&k_cache, "k_cache"}, {&v_cache, "v_cache"}, {&out, "out"}};
    for (const auto &t : all) {
        if (!t.first) continue;
        TORCH_CHECK(t.first->defined() && t.first->is_contiguous(), fn, ": ", t.second, " must be a contiguous tensor");
        TORCH_CHECK(!(reinterpret_cast<uintptr_t>(t.first->data_ptr()) & 15), fn, ": ", t.second, " must be 16-byte aligned");
    }
    const auto dt = qkv.scalar_type();
    TORCH_CHECK(dt == torch::kFloat16 || dt == torch::kBFloat16, fn, ": dtype of qkv must be torch.float16 or torch.bfloat16 (got ", dt, ")");
    TORCH_CHECK(n_kv >= 1 && n_heads >= 1 && n_heads % n_kv == 0, fn, ": n_heads=", n_heads, " must be a positive multiple of n_kv=", n_kv);
    int64_t B, cap, d;
    if (table) {
        TORCH_CHECK(table->defined() && table->is_contiguous() && table->scalar_type() == torch::kInt32, fn,
                    ": block_table must be a contiguous int32 tensor");
        TORCH_CHECK(!(reinterpret_cast<uintptr_t>(table->data_ptr()) & 3), fn, ": block_table must be 4-byte aligned");
        TORCH_CHECK(k_cache.dim() == 4 && k_cache.size(1) == n_kv && k_cache.size(2) == 64 && k_cache.size(0) >= 1 &&
                    k_cache.size(0) <= INT32_MAX, fn, ": k_pages must be [n_pages, n_kv=", n_kv, ", 64, head_dim] (got ", k_cache.sizes(), ")");
        cap = rope_cos.dim() == 2 ? rope_cos.size(0) : 0;
        const int64_t width = (cap + 63) / 64;
        TORCH_CHECK(table->dim() == 1 + lead && table->size(lead) == width, fn, ": block_table must be [", lead ? "batch, " : "",
                    "ceil(capacity=", cap, " / 64)=", width, "] (got ", table->sizes(), ")");
        B = lead ? table->size(0) : 1;
        d = k_cache.size(3);
    } else {
        TORCH_CHECK(k_cache.dim() == 3 + lead && k_cache.size(lead) == n_kv, fn, ": k_cache must be [", lead ? "batch, " : "", "n_kv=", n_kv,
                    ", capacity, head_dim] (got ", k_cache.sizes(), ")");
        B = lead ? k_cache.size(0) : 1; cap = k_cache.size(lead + 1); d = k_cache.size(lead + 2);
    }
    TORCH_CHECK(B >= 1 && B <= 65535, fn, ": batch=", B, " must be in [1, 65535]");
    TORCH_CHECK(d == 64 || d == 128, fn, ": head_dim=", d, " is not 64 or 128");
    TORCH_CHECK(cap >= 1 && cap <= INT32_MAX, fn, ": capacity=", cap, " must be >= 1");
    TORCH_CHECK(std::isfinite(scale) && scale > 0 && std::isfinite((float)scale), fn, ": scale=", scale, " must be finite and > 0");
    TORCH_CHECK(k_cache.scalar_type() == dt && v_cache.scalar_type() == dt && out.scalar_type() == dt, fn,
                ": k_cache, v_cache and out must have qkv's dtype ", dt);
    TORCH_CHECK(v_cache.sizes() == k_cache.sizes(), fn, ": v_cache must have k_cache's shape ", k_cache.sizes(), " (got ", v_cache.sizes(), ")");
    own(B, cap, d);
    for (const torch::Tensor *t : {&rope_cos, &rope_sin})
        TORCH_CHECK(t->scalar_type() == torch::kFloat32 && t->dim() == 2 && t->size(0) == cap && t->size(1) == d / 2,
                    fn, ": rope_cos / rope_sin must be fp32 [capacity=", cap, ", head_dim/2=", d / 2, "] (got ", t->sizes(), ")");
    for (const auto &t : all)
        TORCH_CHECK(!t.first || (t.first->is_cuda() && t.first->device() == qkv.device()), fn, ": ", t.second,
                    " must be a CUDA tensor, on the device of qkv");
    TORCH_CHECK(!table || (table->is_cuda() && table->device() == qkv.device()), fn, ": block_table must be a CUDA tensor, on the device of qkv");
    Args a;
    a.dtype = dt == torch::kFloat16 ? SQLLM_DT_F16 : SQLLM_DT_BF16;
    a.n_heads = (int)n_heads; a.n_kv = (int)n_kv; a.head_dim = (int)d; a.capacity = (int)cap; a.scale = (float)scale;
    a.qkv = qkv.data_ptr(); a.rope_cos = rope_cos.data_ptr<float>(); a.rope_sin = rope_sin.data_ptr<float>();
    if constexpr (std::is_same<Args, sqllm_attn_decode_paged_args>::value || std::is_same<Args, sqllm_attn_extend_paged_args>::value ||
                  std::is_same<Args, sqllm_attn_extend_batch_paged_args>::value) {
        a.k_pages = k_cache.data_ptr(); a.v_pages = v_cache.data_ptr(); a.n_pages = (int)k_cache.size(0);
        a.block_table = table->data_ptr<int32_t>(); a.table_width = (int)table->size(lead);
    } else {
        a.k_cache = k_cache.data_ptr(); a.v_cache = v_cache.data_ptr();
    }
    a.out = out.data_ptr();
    return a;
}

// The own shape checks of attn_decode_batch and attn_decode_paged (attn_args' `own`), messages prefixed with `fn`: qkv [batch,
// (n_heads + 2 n_kv) head_dim], out [batch, n_heads head_dim], pos int32 [batch].
auto batch_shapes(const char *fn, const torch::Tensor &qkv, const torch::Tensor &pos, const torch::Tensor &out, int64_t n_heads,
                  int64_t n_kv) {
    return [=, &qkv, &pos, &out](int64_t B, int64_t, int64_t d) {
        TORCH_CHECK(qkv.dim() == 2 && qkv.size(0) == B && qkv.size(1) == (n_heads + 2 * n_kv) * d, fn, ": qkv must be [batch=", B,
                    ", (n_heads + 2 n_kv) head_dim=", (n_heads + 2 * n_kv) * d, "] (got ", qkv.sizes(), ")");
        TORCH_CHECK(out.dim() == 2 && out.size(0) == B && out.size(1) == n_heads * d, fn, ": out must be [batch=", B,
                    ", n_heads head_dim=", n_heads * d, "] (got ", out.sizes(), ")");
        TORCH_CHECK(pos.scalar_type() == torch::kInt32 && pos.dim() == 1 && pos.size(0) == B, fn, ": pos must be int32 [batch=", B,
                    "] (got ", pos.scalar_type(), " ", pos.sizes(), ")");
    };
}

// The own shape checks of attn_extend and attn_extend_paged, messages prefixed with `fn`: qkv [T >= 1, (n_heads + 2 n_kv) head_dim],
// start + T <= capacity, out [T, n_heads head_dim].
auto chunk_shapes(const char *fn, const torch::Tensor &qkv, int64_t start, const torch::Tensor &out, int64_t n_heads, int64_t n_kv) {
    return [=, &qkv, &out](int64_t, int64_t cap, int64_t d) {
        TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == (n_heads + 2 * n_kv) * d, fn, ": qkv must be [T, (n_heads + 2 n_kv) head_dim=",
                    (n_heads + 2 * n_kv) * d, "] (got ", qkv.sizes(), ")");
        const int64_t T = qkv.size(0);
        TORCH_CHECK(T >= 1, fn, ": qkv has no rows (T=0)");
        TORCH_CHECK(start >= 0, fn, ": start=", start, " must be >= 0");
        TORCH_CHECK(start + T <= cap, fn, ": start=", start, " + T=", T, " must be <= capacity=", cap);
        TORCH_CHECK(out.dim() == 2 && out.size(0) == T && out.size(1) == n_heads * d, fn, ": out must be [T=", T, ", n_heads head_dim=",
                    n_heads * d, "] (got ", out.sizes(), ")");
    };
}

// The own shape checks of attn_extend_batch and attn_extend_batch_paged, messages prefixed with `fn`, the segment checks of
// sqllm_attn_extend_batch made here too so that a CPU caller sees them: 1 to 128 segments, the three lists of one length, each slot in
// [0, n_slots) and named once, T >= 1, start >= 0, start + T <= capacity, the query tiles of all segments within 65535; qkv
// [sum T, (n_heads + 2 n_kv) head_dim] and out [sum T, n_heads head_dim].
auto segment_shapes(const char *fn, const torch::Tensor &qkv, const std::vector<int64_t> &slots, const std::vector<int64_t> &starts,
                    const std::vector<int64_t> &n_tokens, const torch::Tensor &out, int64_t n_heads, int64_t n_kv) {
    return [=, &qkv, &slots, &starts, &n_tokens, &out](int64_t n_slots, int64_t cap, int64_t d) {
        const int64_t n = (int64_t)slots.size();
        TORCH_CHECK(n >= 1 && n <= SQLLM_ATTN_EXTEND_MAX_SEGMENTS, fn, ": n_segments=", n, " must be in [1, ",
                    SQLLM_ATTN_EXTEND_MAX_SEGMENTS, "]");
        TORCH_CHECK((int64_t)starts.size() == n && (int64_t)n_tokens.size() == n, fn, ": slots, starts and n_tokens must have one length (got ",
                    n, ", ", starts.size(), ", ", n_tokens.size(), ")");
        int64_t rows = 0, tiles = 0;
        for (int64_t i = 0; i < n; ++i) {
            TORCH_CHECK(slots[i] >= 0 && slots[i] < n_slots, fn, ": slots[", i, "]=", slots[i], " must be in [0, n_slots=", n_slots, ")");
            for (int64_t j = 0; j < i; ++j) TORCH_CHECK(slots[j] != slots[i], fn, ": slots[", i, "]=", slots[i], " repeats slots[", j, "]");
            TORCH_CHECK(n_tokens[i] >= 1, fn, ": n_tokens[", i, "]=", n_tokens[i], " must be >= 1");
            TORCH_CHECK(starts[i] >= 0, fn, ": starts[", i, "]=", starts[i], " must be >= 0");
            TORCH_CHECK(starts[i] + n_tokens[i] <= cap, fn, ": starts[", i, "]=", starts[i], " + n_tokens[", i, "]=", n_tokens[i],
                        " must be <= capacity=", cap);
            rows += n_tokens[i];
            tiles += (n_tokens[i] * (n_heads / n_kv) + 63) / 64;
        }
        TORCH_CHECK(tiles <= 65535, fn, ": the segments need ", tiles, " query tiles of 64 per KV head, more than 65535");
        TORCH_CHECK(qkv.dim() == 2 && qkv.size(0) == rows && qkv.size(1) == (n_heads + 2 * n_kv) * d, fn, ": qkv must be [sum n_tokens=",
                    rows, ", (n_heads + 2 n_kv) head_dim=", (n_heads + 2 * n_kv) * d, "] (got ", qkv.sizes(), ")");
        TORCH_CHECK(out.dim() == 2 && out.size(0) == rows && out.size(1) == n_heads * d, fn, ": out must be [sum n_tokens=", rows,
                    ", n_heads head_dim=", n_heads * d, "] (got ", out.sizes(), ")");
    };
}

// the segment lists of an attn_extend_batch call as int32, checked by segment_shapes
struct Segments {
    std::vector<int32_t> slots, starts, n_tokens;
    Segments(const std::vector<int64_t> &s, const std::vector<int64_t> &st, const std::vector<int64_t> &t)
        : slots(s.begin(), s.end()), starts(st.begin(), st.end()), n_tokens(t.begin(), t.end()) {}
    template <typename Args>
    void into(Args &a) const {
        a.n_segments = (int)slots.size(); a.slots = slots.data(); a.starts = starts.data(); a.n_tokens = n_tokens.data();
    }
};

// One layer's decode attention (sqllm_attn_decode): rotary, the append of k / v at slot *pos of the caches, attention over slots
// 0..*pos into out, on the current stream.
void attn_decode(torch::Tensor qkv, torch::Tensor pos, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_cache,
                 torch::Tensor v_cache, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_decode_args>("attn_decode", 0, qkv, &pos, rope_cos, rope_sin, k_cache, v_cache, out, n_heads, n_kv, scale,
                                               [&](int64_t, int64_t, int64_t d) {
        TORCH_CHECK(qkv.numel() == (n_heads + 2 * n_kv) * d, "attn_decode: qkv has ", qkv.numel(), " elements, want (n_heads + 2 n_kv) head_dim = ",
                    (n_heads + 2 * n_kv) * d);
        TORCH_CHECK(out.numel() == n_heads * d, "attn_decode: out has ", out.numel(), " elements, want n_heads head_dim = ", n_heads * d);
        TORCH_CHECK(pos.scalar_type() == torch::kInt32 && pos.numel() == 1, "attn_decode: pos must be one int32 element");
    });
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.pos = pos.data_ptr<int32_t>();
    check_status(sqllm_attn_decode(&a, cur_stream()), "quant_cuda.attn_decode");
}

// Decode attention of B sequences (sqllm_attn_decode_batch): for each row b what attn_decode does, at position pos[b] in cache block b;
// a row whose pos[b] is outside the cache writes nothing.
void attn_decode_batch(torch::Tensor qkv, torch::Tensor pos, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_cache,
                       torch::Tensor v_cache, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_decode_batch_args>("attn_decode_batch", 1, qkv, &pos, rope_cos, rope_sin, k_cache, v_cache, out, n_heads,
                                                     n_kv, scale, batch_shapes("attn_decode_batch", qkv, pos, out, n_heads, n_kv));
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.batch = (int)k_cache.size(0);
    a.pos = pos.data_ptr<int32_t>();
    check_status(sqllm_attn_decode_batch(&a, cur_stream()), "quant_cuda.attn_decode_batch");
}

// Attention of a chunk of T new tokens at positions start .. start+T-1 (sqllm_attn_extend): the append of the chunk's rotated k and v
// at slots start .. start+T-1 of the caches, causal attention of every token over the cache up to its own position into out, on the
// current stream.
void attn_extend(torch::Tensor qkv, int64_t start, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_cache,
                 torch::Tensor v_cache, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_extend_args>("attn_extend", 0, qkv, nullptr, rope_cos, rope_sin, k_cache, v_cache, out, n_heads, n_kv, scale,
                                               chunk_shapes("attn_extend", qkv, start, out, n_heads, n_kv));
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.start = (int)start; a.n_tokens = (int)qkv.size(0);
    check_status(sqllm_attn_extend(&a, cur_stream()), "quant_cuda.attn_extend");
}

// Decode attention of T <= 16 new tokens at positions *pos .. *pos+T-1 (sqllm_attn_verify): the append of their rotated k and v at those
// slots, and per token attention over slots 0 .. its own position into out, on the current stream.
void attn_verify(torch::Tensor qkv, torch::Tensor pos, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_cache,
                 torch::Tensor v_cache, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_verify_args>("attn_verify", 0, qkv, &pos, rope_cos, rope_sin, k_cache, v_cache, out, n_heads, n_kv, scale,
                                               [&](int64_t, int64_t, int64_t d) {
        TORCH_CHECK(qkv.dim() == 2 && qkv.size(1) == (n_heads + 2 * n_kv) * d, "attn_verify: qkv must be [T, (n_heads + 2 n_kv) head_dim=",
                    (n_heads + 2 * n_kv) * d, "] (got ", qkv.sizes(), ")");
        const int64_t T = qkv.size(0);
        TORCH_CHECK(T >= 1 && T <= 16, "attn_verify: qkv has ", T, " rows, want T in [1, 16]");
        TORCH_CHECK(out.dim() == 2 && out.size(0) == T && out.size(1) == n_heads * d, "attn_verify: out must be [T=", T, ", n_heads head_dim=",
                    n_heads * d, "] (got ", out.sizes(), ")");
        TORCH_CHECK(pos.scalar_type() == torch::kInt32 && pos.numel() == 1, "attn_verify: pos must be one int32 element");
    });
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.n_tokens = (int)qkv.size(0);
    a.pos = pos.data_ptr<int32_t>();
    check_status(sqllm_attn_verify(&a, cur_stream()), "quant_cuda.attn_verify");
}

// Decode attention of B sequences in one page pool (sqllm_attn_decode_paged): for each row b what attn_decode_batch does, at position
// pos[b], through row b of block_table; a row whose pos[b] is outside the cache or whose table names a page outside the pool writes
// nothing.
void attn_decode_paged(torch::Tensor qkv, torch::Tensor pos, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_pages,
                       torch::Tensor v_pages, torch::Tensor block_table, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_decode_paged_args>("attn_decode_paged", 1, qkv, &pos, rope_cos, rope_sin, k_pages, v_pages, out, n_heads,
                                                     n_kv, scale, batch_shapes("attn_decode_paged", qkv, pos, out, n_heads, n_kv),
                                                     &block_table);
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.batch = (int)block_table.size(0);
    a.pos = pos.data_ptr<int32_t>();
    check_status(sqllm_attn_decode_paged(&a, cur_stream()), "quant_cuda.attn_decode_paged");
}

// The chunk attention of attn_extend for one sequence in a page pool (sqllm_attn_extend_paged), through its block table row.
void attn_extend_paged(torch::Tensor qkv, int64_t start, torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_pages,
                       torch::Tensor v_pages, torch::Tensor block_table_row, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_extend_paged_args>("attn_extend_paged", 0, qkv, nullptr, rope_cos, rope_sin, k_pages, v_pages, out, n_heads,
                                                     n_kv, scale, chunk_shapes("attn_extend_paged", qkv, start, out, n_heads, n_kv),
                                                     &block_table_row);
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    a.start = (int)start; a.n_tokens = (int)qkv.size(0);
    check_status(sqllm_attn_extend_paged(&a, cur_stream()), "quant_cuda.attn_extend_paged");
}

// The chunk attention of attn_extend for several sequences in one call (sqllm_attn_extend_batch): segment i is n_tokens[i] tokens of
// slot slots[i] at starts[i] .. , rows row0_i .. of qkv and out in the lists' order, on caches [n_slots, n_kv, capacity, head_dim].
void attn_extend_batch(torch::Tensor qkv, std::vector<int64_t> slots, std::vector<int64_t> starts, std::vector<int64_t> n_tokens,
                       torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_cache, torch::Tensor v_cache, torch::Tensor out,
                       int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_extend_batch_args>("attn_extend_batch", 1, qkv, nullptr, rope_cos, rope_sin, k_cache, v_cache, out,
                                                     n_heads, n_kv, scale,
                                                     segment_shapes("attn_extend_batch", qkv, slots, starts, n_tokens, out, n_heads, n_kv));
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    const Segments seg(slots, starts, n_tokens);
    seg.into(a);
    a.n_slots = (int)k_cache.size(0);
    check_status(sqllm_attn_extend_batch(&a, cur_stream()), "quant_cuda.attn_extend_batch");
}

// attn_extend_batch in a page pool (sqllm_attn_extend_batch_paged): segment i through row slots[i] of block_table [n_slots, width].
void attn_extend_batch_paged(torch::Tensor qkv, std::vector<int64_t> slots, std::vector<int64_t> starts, std::vector<int64_t> n_tokens,
                             torch::Tensor rope_cos, torch::Tensor rope_sin, torch::Tensor k_pages, torch::Tensor v_pages,
                             torch::Tensor block_table, torch::Tensor out, int64_t n_heads, int64_t n_kv, double scale) {
    auto a = attn_args<sqllm_attn_extend_batch_paged_args>(
        "attn_extend_batch_paged", 1, qkv, nullptr, rope_cos, rope_sin, k_pages, v_pages, out, n_heads, n_kv, scale,
        segment_shapes("attn_extend_batch_paged", qkv, slots, starts, n_tokens, out, n_heads, n_kv), &block_table);
    const at::cuda::OptionalCUDAGuard guard(device_of(qkv));
    const Segments seg(slots, starts, n_tokens);
    seg.into(a);
    a.n_slots = (int)block_table.size(0);
    check_status(sqllm_attn_extend_batch_paged(&a, cur_stream()), "quant_cuda.attn_extend_batch_paged");
}

// One token per row of logits (sqllm_sample): greedy, or temperature / top-k / top-p filtering and a Gumbel-max draw keyed by seed[b]
// and counted by pos[b], into out[b]; a row whose pos[b] < 0 writes nothing.  Current stream, no allocation: graph-capturable.  The
// device-free checks run first, as in the attention bindings.
void sample(torch::Tensor logits, torch::Tensor pos, torch::Tensor temperature, torch::Tensor top_k, torch::Tensor top_p, torch::Tensor seed,
            torch::Tensor out) {
    const std::pair<const torch::Tensor *, const char *> all[] = {{&logits, "logits"}, {&pos, "pos"}, {&temperature, "temperature"},
                                                                  {&top_k, "top_k"}, {&top_p, "top_p"}, {&seed, "seed"}, {&out, "out"}};
    for (const auto &t : all) TORCH_CHECK(t.first->defined(), "sample: ", t.second, " is undefined");
    const auto dt = logits.scalar_type();
    TORCH_CHECK(dt == torch::kFloat32 || dt == torch::kFloat16 || dt == torch::kBFloat16,
                "sample: dtype of logits must be torch.float32, torch.float16 or torch.bfloat16 (got ", dt, ")");
    TORCH_CHECK(logits.dim() == 2 && logits.size(0) >= 1 && logits.size(1) >= 1, "sample: logits must be [rows, vocab] (got ", logits.sizes(), ")");
    const int64_t R = logits.size(0), V = logits.size(1);
    TORCH_CHECK(R <= 65535, "sample: rows=", R, " must be in [1, 65535]");
    TORCH_CHECK(V <= 262144, "sample: vocab=", V, " must be in [1, 262144]");
    TORCH_CHECK(logits.stride(1) == 1 || V == 1, "sample: logits must have unit last stride (got strides ", logits.strides(), ")");
    const int64_t row_stride = R == 1 ? V : logits.stride(0);
    TORCH_CHECK(row_stride >= V, "sample: logits' row stride ", logits.stride(0), " must be >= vocab=", V);
    const std::tuple<const torch::Tensor *, const char *, c10::ScalarType> vecs[] = {
        {&pos, "pos", torch::kInt32}, {&temperature, "temperature", torch::kFloat32}, {&top_k, "top_k", torch::kInt32},
        {&top_p, "top_p", torch::kFloat32}, {&seed, "seed", torch::kInt64}, {&out, "out", torch::kInt64}};
    for (const auto &v : vecs) {
        const torch::Tensor &t = *std::get<0>(v);
        TORCH_CHECK(t.scalar_type() == std::get<2>(v) && t.dim() == 1 && t.size(0) == R && t.is_contiguous(), "sample: ", std::get<1>(v),
                    " must be a contiguous ", std::get<2>(v), " vector of rows=", R, " elements (got ", t.scalar_type(), " ", t.sizes(), ")");
    }
    for (const auto &t : all)
        TORCH_CHECK(t.first->is_cuda() && t.first->device() == logits.device(), "sample: ", t.second, " must be a CUDA tensor, on the device of logits");
    const at::cuda::OptionalCUDAGuard guard(device_of(logits));
    sqllm_sample_args a;
    a.dtype = dt == torch::kFloat32 ? SQLLM_DT_F32 : dt == torch::kFloat16 ? SQLLM_DT_F16 : SQLLM_DT_BF16;
    a.rows = (int)R; a.vocab = (int)V; a.row_stride = row_stride;
    a.logits = logits.data_ptr(); a.pos = pos.data_ptr<int32_t>(); a.temperature = temperature.data_ptr<float>(); a.top_k = top_k.data_ptr<int32_t>();
    a.top_p = top_p.data_ptr<float>(); a.seed = reinterpret_cast<const uint64_t *>(seed.data_ptr<int64_t>()); a.out = out.data_ptr<int64_t>();
    check_status(sqllm_sample(&a, cur_stream()), "quant_cuda.sample");
}

torch::Tensor unpack_indices(torch::Tensor qweight, int bits) {
    const at::cuda::OptionalCUDAGuard guard(device_of(qweight));
    need(qweight, "qweight", torch::kInt32, qweight);
    TORCH_CHECK(bits == 3 || bits == 4, "bits must be 3 or 4");
    TORCH_CHECK(qweight.dim() == 2 && qweight.size(0) % bits == 0, "qweight must be [in/32*bits, out]");
    const int K = (int)(qweight.size(0) / bits * 32), N = (int)qweight.size(1);
    torch::Tensor idx = torch::empty({K, N}, torch::TensorOptions().dtype(torch::kUInt8).device(qweight.device()));
    check_status(sqllm_unpack_indices(bits, qweight.data_ptr<int32_t>(), K, N, idx.data_ptr<uint8_t>(), cur_stream()), "unpack_indices");
    return idx;
}

std::tuple<torch::Tensor, torch::Tensor> kmeans1d(torch::Tensor w, torch::Tensor s, int k) {
    const at::cuda::OptionalCUDAGuard guard(device_of(w));
    need(w, "w", torch::kFloat32, w);
    need(s, "sample_weight", torch::kFloat32, w);
    TORCH_CHECK(w.dim() == 2 && s.sizes() == w.sizes(), "w and sample_weight must both be [rows, n]");
    const int R = (int)w.size(0), n = (int)w.size(1);
    size_t bytes = 0;
    check_status(sqllm_kmeans1d_workspace_bytes(R, n, k, &bytes), "quant_cuda.kmeans1d");
    auto opt = torch::TensorOptions().device(w.device());
    torch::Tensor ws = torch::empty({(int64_t)bytes}, opt.dtype(torch::kUInt8));
    torch::Tensor cent = torch::empty({R, k}, opt.dtype(torch::kFloat32));
    torch::Tensor labels = torch::empty({R, n}, opt.dtype(torch::kUInt8));
    check_status(sqllm_kmeans1d(w.data_ptr<float>(), s.data_ptr<float>(), R, n, k, cent.data_ptr<float>(), labels.data_ptr<uint8_t>(),
                                ws.data_ptr(), bytes, cur_stream()),
                 "quant_cuda.kmeans1d");
    return {cent, labels};
}

torch::Tensor pack_indices(torch::Tensor labels, int bits) {
    const at::cuda::OptionalCUDAGuard guard(device_of(labels));
    need(labels, "labels", torch::kUInt8, labels);
    TORCH_CHECK(bits == 3 || bits == 4, "bits must be 3 or 4");
    TORCH_CHECK(labels.dim() == 2 && labels.size(1) % 32 == 0, "labels must be [out, in] with in a multiple of 32");
    const int N = (int)labels.size(0), K = (int)labels.size(1);
    torch::Tensor q = torch::empty({K / 32 * bits, N}, torch::TensorOptions().dtype(torch::kInt32).device(labels.device()));
    check_status(sqllm_pack_indices(bits, labels.data_ptr<uint8_t>(), K, N, q.data_ptr<int32_t>(), cur_stream()), "quant_cuda.pack_indices");
    return q;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "H100-native drop-in for SqueezeLLM's quant_cuda extension";
    // the reference's 12 symbols (squeezellm/quant_cuda.cpp:258-269), same names and positional order
    m.def("vecquant3matmul_nuq_perchannel", &dense<3, false>, "3-bit per-channel LUT matvec (accumulates into mul)");
    m.def("vecquant4matmul_nuq_perchannel", &dense<4, false>, "4-bit per-channel LUT matvec (accumulates into mul)");
    m.def("vecquant3matmul_nuq_perchannel_batched", &dense<3, true>, "3-bit per-channel LUT matmul, batched");
    m.def("vecquant4matmul_nuq_perchannel_batched", &dense<4, true>, "4-bit per-channel LUT matmul, batched");
    m.def("vecquant3matmul_spmv_nuq_perchannel", &spmv<3, false>, "3-bit LUT matvec + CSR outliers");
    m.def("vecquant4matmul_spmv_nuq_perchannel", &spmv<4, false>, "4-bit LUT matvec + CSR outliers");
    m.def("vecquant3matmul_spmv_nuq_perchannel_batched", &spmv<3, true>, "3-bit LUT matmul + CSR outliers, batched");
    m.def("vecquant4matmul_spmv_nuq_perchannel_batched", &spmv<4, true>, "4-bit LUT matmul + CSR outliers, batched");
    m.def("vecquant3matmul_spmv_hybrid_nuq_perchannel", &hybrid<3, false>, "3-bit LUT matvec + CSR + dense rows");
    m.def("vecquant4matmul_spmv_hybrid_nuq_perchannel", &hybrid<4, false>, "4-bit LUT matvec + CSR + dense rows");
    m.def("vecquant3matmul_spmv_hybrid_nuq_perchannel_batched", &hybrid<3, true>, "3-bit LUT matmul + CSR + dense rows, batched");
    m.def("vecquant4matmul_spmv_hybrid_nuq_perchannel_batched", &hybrid<4, true>, "4-bit LUT matmul + CSR + dense rows, batched");
    // additions
    m.def("lutgemv_fused", &lutgemv_fused, "fused QuantLinearLUT matvec: fp16 / bf16 / fp32 x -> y in x's dtype (bias, CSR, dense rows), one launch",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias") = py::none(),
          py::arg("rows") = py::none(), py::arg("cols") = py::none(), py::arg("vals") = py::none(),
          py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none());
    m.def("lutgemm_fused", &lutgemm_fused, "fused QuantLinearLUT matmul on the tensor cores: fp16 or bf16 x [M, in] -> y [M, out] in x's dtype (bias, CSR, dense rows), one launch",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias") = py::none(),
          py::arg("rows") = py::none(), py::arg("cols") = py::none(), py::arg("vals") = py::none(),
          py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none());
    m.def("lutgemm_fused_f32", &lutgemm_fused_f32, "lutgemm_fused for fp32 x [M, in] -> fp32 y [M, out] (x split into three bf16 parts; bias, CSR, dense rows), one launch",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias") = py::none(),
          py::arg("rows") = py::none(), py::arg("cols") = py::none(), py::arg("vals") = py::none(),
          py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none());
    m.def("lutgemv_rows", &lutgemv_rows, "fused QuantLinearLUT matmul for a few rows on the CUDA cores: fp16 x [M, in] -> fp16 y [M, out] (bias, CSR, dense rows), one launch",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias") = py::none(),
          py::arg("rows") = py::none(), py::arg("cols") = py::none(), py::arg("vals") = py::none(),
          py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none());
    m.def("lutgemv_rows_bf16", &lutgemv_rows_bf16, "lutgemv_rows for bf16 x [M, in] -> bf16 y [M, out] (bias, CSR, dense rows), one launch",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias") = py::none(),
          py::arg("rows") = py::none(), py::arg("cols") = py::none(), py::arg("vals") = py::none(),
          py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none());
    m.def("lutgemm_t", &lutgemm_t, "input gradient of QuantLinearLUT: dy [M, out] -> dx [M, in] = dy . W^T (CSR, dense rows), in dy's dtype, one launch",
          py::arg("dy"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("rows") = py::none(),
          py::arg("cols") = py::none(), py::arg("vals") = py::none(), py::arg("full_rows") = py::none(),
          py::arg("full_row_indices") = py::none(), py::arg("path") = "auto");
    m.def("lut_grad", &lut_grad, "gradients of QuantLinearLUT's codebook, CSR values and dense rows from x [M, in] and dy [M, out]: "
          "(dlut, dvals, dfull_rows) fp32, None where not requested, one launch",
          py::arg("x"), py::arg("dy"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("rows") = py::none(),
          py::arg("cols") = py::none(), py::arg("vals") = py::none(), py::arg("full_rows") = py::none(),
          py::arg("full_row_indices") = py::none(), py::arg("want_lut") = true, py::arg("want_vals") = false,
          py::arg("want_full_rows") = false, py::arg("path") = "auto");
    m.def("lutgemv_fused_exchange", &lutgemv_fused_exchange,
          "fused matvec of a column shard that stores its result into every rank's symmetric arena (NVLink peer memory) and waits for the peers'",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias"), py::arg("rows"), py::arg("cols"),
          py::arg("vals"), py::arg("full_rows"), py::arg("full_row_indices"), py::arg("peer_base"), py::arg("out_offset"),
          py::arg("flag_offset"), py::arg("state_offset"), py::arg("error_offset"), py::arg("world"), py::arg("rank"), py::arg("members"),
          py::arg("out_features_full"));
    m.def("lutgemv_fused_exchange_bf16", &lutgemv_fused_exchange_bf16,
          "lutgemv_fused_exchange for bf16 x: bf16 vectors in every rank's arena",
          py::arg("x"), py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("bias"), py::arg("rows"), py::arg("cols"),
          py::arg("vals"), py::arg("full_rows"), py::arg("full_row_indices"), py::arg("peer_base"), py::arg("out_offset"),
          py::arg("flag_offset"), py::arg("state_offset"), py::arg("error_offset"), py::arg("world"), py::arg("rank"), py::arg("members"),
          py::arg("out_features_full"));
    m.def("sequence_create", &sequence_create, "one persistent launch for a list of dependent fused matvecs (see squeezellm_b200.runtime.DecodeSequence)",
          py::arg("items"), py::arg("exports"), py::arg("lut_mode") = "exact", py::arg("world") = 1, py::arg("rank") = 0,
          py::arg("arena") = py::none(), py::arg("peer_base") = 0, py::arg("dtype") = torch::kFloat16, py::kw_only(), py::arg("ops") = py::none());
    m.def("sequence_arena_bytes", [](py::list lens) {
              size_t off = 0;
              for (auto l : lens) off += ((size_t)l.cast<int64_t>() * 4 + 127) / 128 * 128;
              return (int64_t)off;
          }, "arena bytes for items with these full output lengths");
    m.def("sequence_run", [](int64_t h) { check_status(sqllm_sequence_run(reinterpret_cast<sqllm_sequence *>(h), cur_stream()), "quant_cuda.sequence_run"); },
          "run the sequence on the current stream (capturable)");
    m.def("sequence_error", [](int64_t h) {
              const int rc = sqllm_sequence_error(reinterpret_cast<sqllm_sequence *>(h), cur_stream());
              TORCH_CHECK(rc >= 0, "sequence_error: ", sqllm_last_error());
              return rc == 1;
          }, "True if a bounded in-kernel wait of the sequence ever timed out (synchronises the current stream)");
    m.def("sequence_reset_error", [](int64_t h) { check_status(sqllm_sequence_reset_error(reinterpret_cast<sqllm_sequence *>(h), cur_stream()), "quant_cuda.sequence_reset_error"); },
          "clear the sequence's error word on the current stream");
    m.def("sequence_destroy", [](int64_t h) { sqllm_sequence_destroy(reinterpret_cast<sqllm_sequence *>(h)); });
    m.def("kmeans1d", &kmeans1d, "exact weighted 1-D k-means per row: w, sample_weight fp32 [rows, n], k -> (centroids fp32 [rows, k], "
          "labels uint8 [rows, n]); deterministic", py::arg("w"), py::arg("sample_weight"), py::arg("k"));
    m.def("pack_indices", &pack_indices, "labels uint8 [out, in] -> qweight int32 [in/32*bits, out] in the reference's packed layout",
          py::arg("labels"), py::arg("bits"));
    m.def("dequantize", &dequantize, "dense weight of QuantLinearLUT: W [ncols, in] in dtype (codebook + CSR + dense rows) for output channels "
          "[col0, col0 + ncols); ncols = -1: to the last channel; one launch",
          py::arg("qweight"), py::arg("lookup_table"), py::arg("bits"), py::arg("rows") = py::none(), py::arg("cols") = py::none(),
          py::arg("vals") = py::none(), py::arg("full_rows") = py::none(), py::arg("full_row_indices") = py::none(),
          py::arg("dtype") = torch::kFloat16, py::arg("col0") = 0, py::arg("ncols") = -1);
    m.def("fisher_accumulate", &fisher_accumulate, "Fisher information of a linear layer, in place: fisher fp32 [out, in] += sum over "
          "the samples of seq_len rows of (dy_s^T x_s)^2, x [rows, in] and dy [rows, out] both fp16 or both bf16; one launch",
          py::arg("x"), py::arg("dy"), py::arg("fisher"), py::arg("seq_len"));
    m.def("attn_decode", &attn_decode, "one layer's batch-1 decode attention: rotary on q and k, k / v appended at slot pos of the caches, "
          "softmax(scale q K^T[0..pos]) V[0..pos] per head (GQA) into out, one launch on the current stream",
          py::arg("qkv"), py::arg("pos"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_cache"), py::arg("v_cache"), py::arg("out"),
          py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_decode_splits", [](int n_heads, int n_kv) {
              const int sm = sqllm_device_sm_count();
              TORCH_CHECK(sm > 0, "attn_decode_splits: ", sqllm_last_error());
              return sqllm_attn_decode_splits(n_heads, n_kv, sm);
          }, "CTAs per cluster of attn_decode on the current device (independent of pos)");
    m.def("attn_decode_batch", &attn_decode_batch, "decode attention of B sequences in one launch: per row b, attn_decode at position "
          "pos[b] in cache block b (qkv [B, (n_heads+2n_kv)*d], pos int32 [B], caches [B, n_kv, capacity, d], out [B, n_heads*d]); a row "
          "whose pos is outside the cache writes nothing; current stream",
          py::arg("qkv"), py::arg("pos"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_cache"), py::arg("v_cache"), py::arg("out"),
          py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_decode_batch_splits", [](int n_heads, int n_kv, int batch) {
              const int sm = sqllm_device_sm_count();
              TORCH_CHECK(sm > 0, "attn_decode_batch_splits: ", sqllm_last_error());
              return sqllm_attn_decode_batch_splits(n_heads, n_kv, batch, sm);
          }, "CTAs per cluster of attn_decode_batch on the current device (independent of the positions)");
    m.def("unpack_indices", &unpack_indices,"GPU unpack of the packed indices -> uint8 [in, out] (test hook)");
    m.def("attn_extend", &attn_extend, "attention of a chunk of T new tokens at positions start .. start+T-1: rotary, the append of k / v at "
          "slots start .. start+T-1, causal attention over the cache (qkv [T, ...], start, rope_cos, rope_sin, k_cache, v_cache, out [T, ...], "
          "n_heads, n_kv, scale)", py::arg("qkv"), py::arg("start"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_cache"),
          py::arg("v_cache"), py::arg("out"), py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_extend_splits", [](int n_heads, int n_kv, int n_tokens, int start) {
              const int sm = sqllm_device_sm_count();
              TORCH_CHECK(sm > 0, "attn_extend_splits: ", sqllm_last_error());
              return sqllm_attn_extend_splits(n_heads, n_kv, n_tokens, start, sm);
          }, "CTAs per cluster of attn_extend on the current device");
    m.def("attn_decode_paged", &attn_decode_paged, "attn_decode_batch on KV page pools [n_pages, n_kv, 64, head_dim]: row b at position "
          "pos[b] through row b of block_table [batch, ceil(capacity / 64)]; a row with pos outside the cache or a table entry outside the "
          "pool writes nothing", py::arg("qkv"), py::arg("pos"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_pages"),
          py::arg("v_pages"), py::arg("block_table"), py::arg("out"), py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_extend_paged", &attn_extend_paged, "attn_extend for one sequence on KV page pools [n_pages, n_kv, 64, head_dim] through "
          "its block table row [ceil(capacity / 64)]; an entry outside the pool among the chunk's blocks writes nothing", py::arg("qkv"),
          py::arg("start"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_pages"), py::arg("v_pages"), py::arg("block_table_row"),
          py::arg("out"), py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_extend_batch", &attn_extend_batch, "attn_extend for several sequences in one call: segment i is n_tokens[i] tokens of "
          "slot slots[i] at positions starts[i] .. (int lists), rows of qkv [sum T, ...] and out [sum T, ...] in the lists' order, on caches "
          "[n_slots, n_kv, capacity, head_dim]; each segment bitwise what attn_extend computes for its slot alone", py::arg("qkv"),
          py::arg("slots"), py::arg("starts"), py::arg("n_tokens"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_cache"),
          py::arg("v_cache"), py::arg("out"), py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_extend_batch_paged", &attn_extend_batch_paged, "attn_extend_batch on KV page pools [n_pages, n_kv, 64, head_dim]: segment i "
          "through row slots[i] of block_table [n_slots, ceil(capacity / 64)]; a segment with a table entry outside the pool among its "
          "blocks writes nothing", py::arg("qkv"), py::arg("slots"), py::arg("starts"), py::arg("n_tokens"), py::arg("rope_cos"),
          py::arg("rope_sin"), py::arg("k_pages"), py::arg("v_pages"), py::arg("block_table"), py::arg("out"), py::arg("n_heads"),
          py::arg("n_kv"), py::arg("scale"));
    m.def("attn_verify", &attn_verify, "decode attention of T <= 16 new tokens at device positions pos .. pos+T-1: rotary, the append of k / "
          "v at those slots, per token softmax(scale q K^T[0..p_t]) V[0..p_t] (qkv [T, ...], pos int32 [1], rope_cos, rope_sin, k_cache, "
          "v_cache, out [T, ...], n_heads, n_kv, scale); pos < 0 or pos + T > capacity writes nothing; current stream",
          py::arg("qkv"), py::arg("pos"), py::arg("rope_cos"), py::arg("rope_sin"), py::arg("k_cache"), py::arg("v_cache"), py::arg("out"),
          py::arg("n_heads"), py::arg("n_kv"), py::arg("scale"));
    m.def("attn_verify_splits", [](int n_heads, int n_kv, int n_tokens, int head_dim, at::ScalarType dtype) {
              TORCH_CHECK(dtype == torch::kFloat16 || dtype == torch::kBFloat16, "attn_verify_splits: dtype must be torch.float16 or "
                          "torch.bfloat16");
              const int S = sqllm_attn_verify_launch_splits(dtype == torch::kFloat16 ? SQLLM_DT_F16 : SQLLM_DT_BF16, n_heads, n_kv,
                                                            head_dim, n_tokens);
              TORCH_CHECK(S > 0, "attn_verify_splits: ", sqllm_last_error());
              return S;
          }, "CTAs per cluster an attn_verify launch uses on the current device (independent of pos)", py::arg("n_heads"), py::arg("n_kv"),
          py::arg("n_tokens"), py::arg("head_dim") = 128, py::arg("dtype") = torch::kFloat16);
    m.def("sample", &sample, "one token per row of logits [rows, vocab] (fp32, fp16 or bf16; unit last stride) into out int64 [rows]: greedy "
          "when temperature[b] <= 0, else temperature, top_k[b] (0: off) and top_p[b] (1: off) filtering and a Gumbel-max draw from "
          "Philox4x32-10 keyed by seed[b] (int64) at counter (i / 4, pos[b]); a row whose pos[b] (int32) < 0 writes nothing; current stream",
          py::arg("logits"), py::arg("pos"), py::arg("temperature"), py::arg("top_k"), py::arg("top_p"), py::arg("seed"), py::arg("out"));
    m.def("abi_version", []() { return sqllm_abi_version(); });
    m.def("set_deterministic", [](bool on) { sqllm_set_deterministic(on ? 1 : 0); },
          "fused path: True = bit-reproducible fixed-order reduction, False (default) = red.add accumulation");
    m.def("set_lut_mode", [](const std::string &mode) {
              TORCH_CHECK(mode == "exact" || mode == "fp16", "lut mode must be 'exact' or 'fp16' (got '", mode, "')");
              sqllm_set_lut_mode(mode == "fp16" ? SQLLM_LUT_FP16_PAIR : SQLLM_LUT_EXACT);
          },
          "fused path: 'exact' (default) = fp32 codebook as stored; 'fp16' = centroids rounded to fp16, pair tables + fp16 x fp16 -> fp32 FMAs "
          "(only taken for fp16 x)");
    m.def("get_lut_mode", []() { return std::string(sqllm_get_lut_mode() == SQLLM_LUT_FP16_PAIR ? "fp16" : "exact"); });
    m.def("workspace_error", []() {
              // error word of the current stream's fused-path workspace on the current device (synchronises the stream)
              int dev = 0;
              C10_CUDA_CHECK(cudaGetDevice(&dev));
              torch::Tensor ws;
              {
                  std::lock_guard<std::mutex> lock(g_ws_mutex);
                  auto it = g_ws.find(std::make_pair(dev, cur_stream()));
                  if (it == g_ws.end()) return false;
                  ws = it->second;
              }
              const int rc = sqllm_workspace_error(ws.data_ptr(), cur_stream());
              TORCH_CHECK(rc >= 0, "workspace_error: ", sqllm_last_error());
              return rc == 1;
          },
          "True if a bounded in-kernel wait of the fused path ever timed out on this stream's workspace (results are then incomplete)");
    m.def("sm_count", []() { return sqllm_device_sm_count(); });
    m.def("fused_limits", []() {
              py::dict d;
              d["max_topx"] = SQLLM_FUSED_MAX_TOPX;
              d["max_out_features"] = SQLLM_FUSED_MAX_OUT;
              d["rows_max_in_features"] = SQLLM_ROWS_MAX_IN;
              return d;
          },
          "largest layer the fused, exchange and sequence entry points accept: {'max_topx', 'max_out_features'} (the 12 symbols have no such "
          "limit), and the largest in_features of lutgemv_rows: 'rows_max_in_features'");
}
