"""QuantLinearLUT / make_quant_lut - host-side mirror of the reference's module interface
(squeezellm/quant.py:28-435) on top of the H100-native `quant_cuda` extension.

Same class name, constructor signature, buffer names (= checkpoint keys: qweight, lookup_table, bias,
rows, cols, vals, full_rows, full_row_indices, startrows), `pack2`, `forward` and `make_quant_lut`
as the reference, so `llama.py`-style loaders work unchanged.  Differences, all behind the same API:

  * `forward` (batch-1 branch, reference quant.py:212-312) uses ONE fused launch
    (`quant_cuda.lutgemv_fused`: fp16 / bf16 / fp32 x in, y out in x's dtype, bias + CSR + dense rows fused;
    `quant_cuda.set_deterministic(True)` selects the bit-reproducible summation) instead of
    zeros + x.float() + 1-3 launches + y.to(dtype).  Layers wider or with more dense rows than the fused launch
    takes (`FUSED_LIMITS`, from the extension) run the reference's 12 symbols instead.  Set
    `QuantLinearLUT.use_fused = False` to go through the reference's 12 symbols exactly as quant.py does.
  * `forward` with fp16 x of at least `TC_MIN_ROWS` rows, or bf16 x of at least `BF16_TC_MIN_ROWS` rows (prefill, evaluation,
    bf16 training; reference quant.py:314-379) uses ONE tensor-core launch (`quant_cuda.lutgemm_fused`, outliers and dense rows
    folded into the weight tiles, output in x's dtype, bit-reproducible) instead of zeros + x.float() + 1-3 batched launches +
    out.to(dtype).  fp32 x of at least `FP32_TC_MIN_ROWS` rows runs the same kernel with x split exactly into three bf16 parts
    (`quant_cuda.lutgemm_fused_f32`, fp32 output).
  * `forward` with fp16 x of 2 to `ROWS_MAX` rows (and fewer than `TC_MIN_ROWS`; several sequences decoding at once, speculative-
    decoding verification, short prompts) uses ONE CUDA-core launch (`quant_cuda.lutgemv_rows`: a multi-row LUT-GEMV whose
    thread-block clusters split K, outliers and dense rows folded per K-slab) instead of the same sequence; bf16 x of 2 to
    `BF16_ROWS_MAX` rows the same kernel with bf16 in and out (`quant_cuda.lutgemv_rows_bf16`).  fp32 x of fewer than
    `FP32_TC_MIN_ROWS` rows and `use_fused = False` keep the reference's batched symbols.
  * `loss.backward()` works through the layer when x requires grad (the reference has no backward: its outputs carry no
    graph).  x gets dx = dy . W^T from ONE launch (`quant_cuda.lutgemm_t`: a transposed LUT-GEMM, on the tensor cores for fp16 /
    bf16 gradients of at least `BWD_TC_MIN_ROWS` rows, else on the CUDA cores; outliers and dense rows included); the buffers are constants and get no gradient.  The forward of such a call takes the same route
    and gives the same bits as without grad; every other call goes exactly as before.  `use_fused` does not affect the
    backward.  The sharded, exchange and sequence paths (sharding.py, runtime.py) give no gradient.
  * `train_codebook()` makes the codebook (and optionally the CSR values, dense rows and bias) nn.Parameters on the same storage:
    their gradients come from ONE more launch (`quant_cuda.lut_grad`: G = x^T . dy bucketed by the packed indices); the indices
    stay fixed and the checkpoint format does not change.
  * `dequantize(dtype)` gives the dense [out, in] weight the layer stands for (codebook + CSR outliers + dense rows, one launch:
    `quant_cuda.dequantize`) and `to_linear(dtype)` an nn.Linear holding it; the reference has neither.
  * `balanced=True` raises NotImplementedError up front: the reference dispatches it to
    `vecquant{3,4}matmul_spmv_balanced_nuq_perchannel`, which its extension never defines
    (quant.py:238,282 vs quant_cuda.cpp:257-270), i.e. an AttributeError at the first forward.
  * the device is the buffers' device, not the hard-coded "cuda" (quant.py:218,317).
  * `pack2` is vectorised (numpy) instead of a Python row loop; output is bit-identical
    (tests/test_oracle_golden.py checks it against buffers produced by the reference's pack2).

There is NO CPU fallback: importing this module requires the compiled extension, and forward() requires
CUDA tensors (the extension raises otherwise).
"""
import glob
import importlib.util
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

_PKG = os.path.dirname(os.path.abspath(__file__))


def _load_extension():
    """Load the in-tree extension as top-level module `quant_cuda` (the name the reference's quant.py:5 imports) WITHOUT touching
    sys.path: putting the package directory there would make build / quant / runtime / ... importable as top-level modules and
    shadow a user's own modules of those names."""
    if "quant_cuda" in sys.modules and hasattr(sys.modules["quant_cuda"], "lutgemv_fused"):
        return sys.modules["quant_cuda"]
    cands = sorted(glob.glob(os.path.join(_PKG, "quant_cuda*.so")))
    if not cands:
        raise ImportError(
            "squeezellm_b200: the compiled CUDA extension `quant_cuda` is missing; build it with "
            "`python -m squeezellm_b200.build` (needs nvcc, sm_90a). No CPU fallback exists.")
    spec = importlib.util.spec_from_file_location("quant_cuda", cands[0])
    mod = importlib.util.module_from_spec(spec)
    try:
        spec.loader.exec_module(mod)
    except ImportError as e:  # fail loudly: no silent eager fallback
        raise ImportError(f"squeezellm_b200: cannot load {cands[0]}: {e}. Rebuild with `python -m squeezellm_b200.build`. "
                          "No CPU fallback exists.") from e
    sys.modules["quant_cuda"] = mod
    return mod


quant_cuda = _load_extension()
# largest layer the fused launch takes (include/sqllm_b200.h: SQLLM_FUSED_MAX_TOPX / SQLLM_FUSED_MAX_OUT); larger layers run the 12 symbols
FUSED_LIMITS = quant_cuda.fused_limits()


def round_to_nearest_pole_sim(w, poles):
    """Round the numbers in w to the nearest value in poles (reference quant.py:8-24)."""
    poles_t = torch.as_tensor(np.asarray(poles), dtype=w.dtype)
    idx = (w.unsqueeze(0) - poles_t.reshape(-1, *([1] * w.dim()))).abs().argmin(dim=0)
    return poles_t[idx]


def pack_indices(idx_kn, bits):
    """uint8/int idx [K, N] -> packed int32 [K/32*bits, N] in the reference layout (quant.py:171-208)."""
    v = np.ascontiguousarray(idx_kn).astype(np.uint32)
    K, N = v.shape
    assert K % 32 == 0, "infeatures must be a multiple of 32"
    if bits == 4:
        v = v.reshape(K // 8, 8, N)
        sh = (4 * np.arange(8, dtype=np.uint32))[None, :, None]
        return np.bitwise_or.reduce(v << sh, axis=1).astype(np.uint32).view(np.int32)
    if bits != 3:
        raise NotImplementedError("Only 3 and 4 bits is supported.")
    v = v.reshape(K // 32, 32, N)
    s = (3 * np.arange(10, dtype=np.uint32))[None, :, None]
    w0 = np.bitwise_or.reduce(v[:, 0:10] << s, axis=1) | (v[:, 10] << 30)
    w1 = ((v[:, 10] >> 2) & 1) | np.bitwise_or.reduce(v[:, 11:21] << (s + 1), axis=1) | (v[:, 21] << 31)
    w2 = ((v[:, 21] >> 1) & 3) | np.bitwise_or.reduce(v[:, 22:32] << (s + 2), axis=1)
    q = np.empty((K // 32 * 3, N), dtype=np.uint32)
    q[0::3], q[1::3], q[2::3] = w0, w1, w2
    return q.view(np.int32)


def _aligned(x):
    """x as one contiguous block that starts on a 16-byte boundary: the kernels read x with 16-byte loads.  A contiguous view
    whose storage offset is not a multiple of 8 fp16 / 4 fp32 elements (a slice of a larger buffer) is copied to fresh storage."""
    x = x.contiguous()
    return x.clone() if x.data_ptr() % 16 else x


class QuantLinearLUT(nn.Module):
    """Drop-in layer replacement (reference quant.py:28)."""

    use_fused = True  # class-wide switch: fused single-launch forward vs the reference's 12-symbol sequence
    # fp16 inputs of at least this many rows run the tensor-core LUT-GEMM (quant_cuda.lutgemm_fused); fewer rows, fp32 inputs
    # and use_fused = False run the batched symbols (bf16 inputs: BF16_TC_MIN_ROWS).  64: where a whole 7B decoder layer gets faster on an H100 (DESIGN.md
    # section 3.6: 32 rows 1.08 vs 0.78 ms, 64 rows 1.09 vs 1.48 ms).
    TC_MIN_ROWS = 64
    # bf16 inputs of at least this many rows run the same tensor-core LUT-GEMM with three bf16 weight parts; fewer rows run the
    # multi-row GEMV (BF16_ROWS_MAX).  80: the smallest measured row count above TC_MIN_ROWS at which a whole 7B decoder layer is faster on an
    # H100 (DESIGN.md section 3.6: 80 rows 1.48 vs 1.90 ms; the tensor cores already win at 64 rows, 1.46 vs 1.56 ms).
    BF16_TC_MIN_ROWS = 80
    # fp32 inputs of at least this many rows run the same tensor-core LUT-GEMM with x split into three bf16 parts as well
    # (quant_cuda.lutgemm_fused_f32, six part products per k-step); fewer rows and use_fused = False run the batched symbols.
    # 128: the smallest measured row count from which a whole 7B decoder layer is faster on an H100 (DESIGN.md section 3.6: 96 rows
    # 2.35 vs 2.20 ms, 128 rows 2.35 vs 2.91 ms); the kernel costs about the same up to 128 rows, the batched symbols grow per row.
    FP32_TC_MIN_ROWS = 128
    # fp16 inputs of 2 to ROWS_MAX rows (below TC_MIN_ROWS) run the multi-row GEMV (quant_cuda.lutgemv_rows).  63: it is faster than
    # the batched symbols on a whole 7B decoder layer at every measured row count up to 63 on an H100 (DESIGN.md section 3.9).
    ROWS_MAX = 63
    # bf16 inputs of 2 to BF16_ROWS_MAX rows (below BF16_TC_MIN_ROWS) run the same multi-row GEMV (quant_cuda.lutgemv_rows_bf16).
    # 79: it is faster than the batched symbols on a whole 7B decoder layer at every measured row count up to 79 on an H100
    # (DESIGN.md section 3.12).
    BF16_ROWS_MAX = 79
    # fp16 / bf16 gradients of at least this many rows run the input gradient on the tensor cores (quant_cuda.lutgemm_t path
    # "tc"); fewer rows and fp32 gradients on the CUDA cores.  96: where the two cross on a whole 7B decoder layer on an H100
    # (DESIGN.md section 3.10: 64 rows 5.96 vs 5.12 ms, 512 rows 8.05 vs 40.8 ms; the CUDA-core time grows 80 us per row).
    BWD_TC_MIN_ROWS = 96
    # codebook precision of the fused path is process-wide: quant_cuda.set_lut_mode("exact" | "fp16")  (include/sqllm_b200.h)

    def __init__(self, bits, infeatures, outfeatures, bias, include_sparse=False, numvals=0, topX=0,
                 balanced=False, num_nonzero_per_thread=10):
        super().__init__()
        if bits not in [3, 4]:
            raise NotImplementedError("Only 3 and 4 bits is supported.")
        if balanced:
            raise NotImplementedError(
                "balanced SpMV is not available: the reference dispatches to quant_cuda.*_spmv_balanced_*, "
                "which its extension never defines (quant_cuda.cpp:257-270)")
        self.infeatures = infeatures
        self.outfeatures = outfeatures
        self.bits = bits
        self.register_buffer("qweight", torch.zeros((infeatures // 32 * self.bits, outfeatures), dtype=torch.int32))
        if bias:
            self.include_bias = True
            self.register_buffer("bias", torch.zeros((outfeatures)))
        else:
            self.include_bias = False
            self.bias = None
        self.register_buffer("lookup_table", torch.zeros((outfeatures, 2**self.bits), dtype=torch.float32))
        self.include_sparse = include_sparse
        self.numvals = numvals
        self.topX = topX
        if numvals > 0:
            self.register_buffer("rows", torch.zeros(outfeatures + 1, dtype=torch.int32))
            self.register_buffer("cols", torch.zeros(numvals, dtype=torch.int32))
            self.register_buffer("vals", torch.zeros(numvals, dtype=torch.float32))
        if topX > 0:
            self.register_buffer("full_rows", torch.zeros((infeatures, topX), dtype=torch.float32))
            self.register_buffer("full_row_indices", torch.zeros(topX, dtype=torch.int32))
        self.balanced = balanced
        self._sibling_group = None  # (SiblingGroup, index) once fusion.fuse_siblings has stacked this layer with its siblings

    BUFFERS = ("qweight", "bias", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices")

    @classmethod
    def from_buffers(cls, bits, buffers):
        """The layer that holds `buffers` (checkpoint names -> tensors: qweight, lookup_table and optionally bias, rows / cols /
        vals, full_rows / full_row_indices; None and other keys are skipped) as its own buffers: no copy and no cast, so a layer
        can hold views of a larger storage (a sibling group's members) and keep a bias in the dtype it was given.  in_features
        and out_features come from qweight, numvals from vals, topX from full_rows; the CSR arrays make the layer sparse."""
        b = {k: buffers[k] for k in cls.BUFFERS if buffers.get(k) is not None}
        if "qweight" not in b or "lookup_table" not in b:
            raise ValueError("QuantLinearLUT.from_buffers: qweight and lookup_table are required")
        for group in (("rows", "cols", "vals"), ("full_rows", "full_row_indices")):
            if 0 < sum(k in b for k in group) < len(group):
                raise ValueError(f"QuantLinearLUT.from_buffers: {' / '.join(group)} come together; got only "
                                 f"{', '.join(k for k in group if k in b)}")
        with torch.device("meta"):  # the constructor's zero buffers are all replaced below
            m = cls(bits, b["qweight"].shape[0] // bits * 32, b["qweight"].shape[1], "bias" in b, include_sparse="rows" in b,
                    numvals=int(b["vals"].numel()) if "vals" in b else 0,
                    topX=int(b["full_rows"].shape[1]) if "full_rows" in b else 0)
        for name, t in b.items():
            m.register_buffer(name, t)
        return m

    # ------------------------------------------------------------------------------------------
    def pack2(self, linear, lookup_table, include_sparse, num_nonzero_per_thread=-1):
        """Fill the buffers from per-channel (centroids, indices) and an outlier matrix
        (reference quant.py:97-208).  lookup_table = (lut, outliers); lut[c][0] = (centroids, indices)."""
        if self._trained:  # it replaces the tensors, which would leave the trained parameters (and an optimizer's references) behind
            raise RuntimeError(f"QuantLinearLUT.pack2: the layer's {', '.join(self._trained)} are trained parameters "
                               "(train_codebook); pack2 fills the buffers of a layer before training, not after")
        if self.include_bias:
            self.bias = linear.bias.clone()
        lut, outliers = lookup_table
        num_channels = len(lut)
        K = linear.weight.shape[1]
        idx = np.empty((num_channels, K), dtype=np.uint8)
        cent = np.empty((num_channels, 2**self.bits), dtype=np.float32)
        for channel in range(num_channels):
            centroid, indices = lut[channel][0]  # last 0 is for group 0
            idx[channel] = np.asarray(indices)
            cent[channel] = np.asarray(centroid, dtype=np.float32)
        self.lookup_table = torch.from_numpy(cent)
        if include_sparse:
            outliers = outliers.to_dense().clone() if outliers.layout != torch.strided else outliers.clone()
            # the dense index at an outlier position encodes the centroid nearest to zero, so the sparse
            # value stored is (outlier - that centroid)  (reference quant.py:117-123)
            zero_map = torch.from_numpy(cent[np.arange(num_channels), np.abs(cent).argmin(axis=1)])
            nz = outliers != 0
            outliers = torch.where(nz, outliers - zero_map[:, None].to(outliers.dtype), outliers)
            csr = outliers.to_sparse(layout=torch.sparse_csr)
            self.register_buffer("rows", csr.crow_indices().to(torch.int32))
            self.register_buffer("cols", csr.col_indices().to(torch.int32))
            self.register_buffer("vals", csr.values().to(torch.float32))
            self.numvals = int(self.vals.shape[0])
        self.qweight = torch.from_numpy(pack_indices(idx.T, self.bits))

    # ------------------------------------------------------------------------------------------
    def _sparse_args(self):
        if not (self.include_sparse and hasattr(self, "rows")):
            return None, None, None, None, None
        fr = fri = None
        if self.topX > 0:
            fr, fri = self.full_rows, self.full_row_indices
        return self.rows, self.cols, self.vals, fr, fri

    def _fused_fits(self, full_rows):
        """The fused launch keeps its cross-CTA sums in a fixed-size workspace: more output channels or dense rows than it holds
        (a stacked q/k/v group adds up its members' dense rows) go through the 12 symbols, which have no such limit."""
        topx = int(full_rows.shape[1]) if full_rows is not None else 0
        return self.outfeatures <= FUSED_LIMITS["max_out_features"] and topx <= FUSED_LIMITS["max_topx"]

    def _rows_fits(self):
        """The layers quant_cuda.lutgemv_rows takes: out_features a multiple of 4, in_features up to the slab its CTAs stage."""
        return self.outfeatures % 4 == 0 and self.infeatures <= FUSED_LIMITS["rows_max_in_features"]

    def forward(self, x):
        # a sibling member asks its group, whose stacked layer comes back here: the gradient flows through the stacked layer's
        # node and autograd's slice backward adds the members' shares
        params = tuple(getattr(self, n) for n in self._trained)
        wants_dx = x.requires_grad and (bool(self._trained) or self._sibling_group is None)
        if torch.is_grad_enabled() and (wants_dx or any(p.requires_grad for p in params)):
            return _QuantLinearLUTFunction.apply(x, self, self._trained, *params)
        return self._forward_impl(x)

    TRAINABLE = ("lookup_table", "vals", "full_rows", "bias")
    _trained = ()  # names of the tensors train_codebook made parameters, in TRAINABLE order

    def train_codebook(self, lookup_table=True, vals=False, full_rows=False, bias=False):
        """Make the selected tensors trainable: the per-channel codebook `lookup_table` [out, 2^bits], the CSR outlier values
        `vals`, the dense rows `full_rows` [in, topX] and the `bias`.  Each becomes an nn.Parameter under the same name and on the
        same storage, so state_dict keys (the checkpoint format) do not change; the packed indices stay fixed.  Returns the list of
        the selected parameters (e.g. for an optimizer).  The backward then computes their gradients in one extra launch
        (quant_cuda.lut_grad) besides the input gradient.  Calling it again adds to the set; nothing is made untrainable."""
        if self._sibling_group is not None:
            raise RuntimeError("QuantLinearLUT.train_codebook: this layer is a member of a sibling group (fusion.fuse_siblings); "
                               "codebook training needs the layers unfused: call train_codebook before fuse_siblings")
        want = [n for n, on in zip(self.TRAINABLE, (lookup_table, vals, full_rows, bias)) if on]
        rows, cols, vals_t, fr, fri = self._sparse_args()
        have = {"lookup_table": self.lookup_table, "vals": vals_t, "full_rows": fr, "bias": self.bias}
        for n in want:
            if have[n] is None:
                what = {"vals": "CSR outliers (include_sparse with rows / cols / vals)", "full_rows": "dense rows (topX > 0)",
                        "bias": "bias"}.get(n, n)
                raise ValueError(f"QuantLinearLUT.train_codebook: the layer has no {what}, so `{n}` cannot be trained")
            if n != "bias" and have[n].dtype != torch.float32:  # checked for every tensor before any is converted
                raise ValueError(f"QuantLinearLUT.train_codebook: `{n}` must be fp32 (got {have[n].dtype})")
        for n in want:
            t = getattr(self, n)
            if not isinstance(t, nn.Parameter):
                del self._buffers[n]
                self.register_parameter(n, nn.Parameter(t))  # same storage, same state_dict key
        self._trained = tuple(n for n in self.TRAINABLE if n in want or n in self._trained)
        return [getattr(self, n) for n in want]

    def _grad_buffers(self):
        """The tensors the input gradient reads (the layer's weights as the backward sees them)."""
        return (self.qweight, self.lookup_table) + tuple(t for t in self._sparse_args() if t is not None)

    def _codebook_grad(self, x, dy, names):
        """(dlut, dvals, dfull_rows) for x [M, in] and dy [M, out] (quant_cuda.lut_grad, one launch), None where not in names."""
        rows, cols, vals, fr, fri = self._sparse_args()
        return quant_cuda.lut_grad(_aligned(x), _aligned(dy), self.qweight, self.lookup_table, self.bits, rows, cols, vals, fr, fri,
                                   want_lut="lookup_table" in names, want_vals="vals" in names,
                                   want_full_rows="full_rows" in names, path="auto")

    def _input_grad(self, dy):
        """dx [M, in] = dy [M, out] . W^T in dy's dtype (quant_cuda.lutgemm_t): the backward of every forward route.  fp16 / bf16
        gradients of at least BWD_TC_MIN_ROWS rows run on the tensor cores, everything else on the CUDA cores."""
        rows, cols, vals, fr, fri = self._sparse_args()
        path = "tc" if dy.dtype in (torch.float16, torch.bfloat16) and dy.shape[0] >= QuantLinearLUT.BWD_TC_MIN_ROWS else "cuda"
        return quant_cuda.lutgemm_t(_aligned(dy), self.qweight, self.lookup_table, self.bits, rows, cols, vals, fr, fri, path=path)

    def dequantize(self, dtype=torch.float16):
        """The dense weight this layer stands for, [out, in] (nn.Linear.weight's layout) in `dtype` (fp16, bf16 or fp32) on the
        layer's device, without gradient: codebook + CSR outliers + dense rows summed in fp32 and rounded once
        (quant_cuda.dequantize, one launch; include/sqllm_b200.h: sqllm_dequantize gives the exact order).  A sibling member
        (fusion.fuse_siblings) dequantizes its rows of the stacked layer; a layer whose codebook is being trained
        (train_codebook) uses the parameters' current values.  The bias is not part of it (see to_linear)."""
        col0, layer = 0, self
        if self._sibling_group is not None:
            group, index = self._sibling_group
            layer, col0 = group.member_columns(index)
        rows, cols, vals, fr, fri = (t.detach() if t is not None else None for t in layer._sparse_args())
        return quant_cuda.dequantize(layer.qweight, layer.lookup_table.detach(), layer.bits, rows, cols, vals, fr, fri,
                                     dtype=dtype, col0=col0, ncols=self.outfeatures)

    def to_linear(self, dtype=torch.float16):
        """An nn.Linear on the layer's device with weight = dequantize(dtype) and the bias cast to `dtype`."""
        weight = self.dequantize(dtype)
        linear = nn.Linear(self.infeatures, self.outfeatures, bias=self.bias is not None, device="meta")
        linear.weight = nn.Parameter(weight)
        if self.bias is not None:
            linear.bias = nn.Parameter(self.bias.detach().to(dtype=dtype, copy=True))
        return linear

    def _forward_impl(self, x):
        if self._sibling_group is not None:
            group, index = self._sibling_group
            return group.member_forward(index, x)
        out_shape = x.shape[:-1] + (self.outfeatures,)
        batched = x.shape[-1] != x.numel()
        if batched:
            x = x.reshape(-1, x.shape[-1])
        rows, cols, vals, fr, fri = self._sparse_args()
        launch = self._fused_launch(x, batched, fr) if QuantLinearLUT.use_fused else None
        if launch is None:
            out = self._reference_forward(x, batched)
        else:  # one row: the bias inside the launch's sum; batches: added below, in the same dtype and rounding as the reference's
            out = launch(_aligned(x), self.qweight, self.lookup_table, self.bits, None if batched else self.bias,
                         rows, cols, vals, fr, fri)
        out = out.reshape(out_shape)
        return out + self.bias if batched and self.bias is not None else out

    def _fused_launch(self, x, batched, full_rows):
        """The fused binding that runs x (one row, or [M, K]), or None where the reference's symbols run it."""
        if not batched:
            fits = x.dtype in (torch.float16, torch.float32, torch.bfloat16) and self._fused_fits(full_rows)
            return quant_cuda.lutgemv_fused if fits else None
        M, cls = x.shape[0], QuantLinearLUT
        tc_min = {torch.float16: cls.TC_MIN_ROWS, torch.bfloat16: cls.BF16_TC_MIN_ROWS, torch.float32: cls.FP32_TC_MIN_ROWS}.get(x.dtype)
        if tc_min is not None and M >= tc_min:
            return quant_cuda.lutgemm_fused_f32 if x.dtype == torch.float32 else quant_cuda.lutgemm_fused
        rows_max = {torch.float16: cls.ROWS_MAX, torch.bfloat16: cls.BF16_ROWS_MAX}.get(x.dtype)
        if rows_max is not None and 2 <= M <= rows_max and self._rows_fits():
            return quant_cuda.lutgemv_rows if x.dtype == torch.float16 else quant_cuda.lutgemv_rows_bf16
        return None

    def _reference_forward(self, x, batched):
        """The reference's sequence (quant.py:213-379): x in fp32, one of the 12 symbols into an fp32 output that one row starts
        from the bias and a batch from zero, then the output in x's dtype."""
        if batched or self.bias is None:
            shape = (x.shape[0], self.outfeatures) if batched else (self.outfeatures,)
            y = torch.zeros(shape, device=self.qweight.device, dtype=torch.float32)
        else:
            y = self.bias.clone()
        self._dispatch(_aligned(x.float()), y, batched)
        return y.to(x.dtype)

    def _dispatch(self, x, y, batched):
        """Pick 1 of the 12 quant_cuda symbols by (bits, batched, dense|spmv|hybrid) - reference quant.py:222-309,320-379."""
        b = self.bits
        sfx = "_batched" if batched else ""
        if self.include_sparse and self.topX > 0:
            fn = getattr(quant_cuda, f"vecquant{b}matmul_spmv_hybrid_nuq_perchannel{sfx}")
            fn(self.rows, self.cols, self.vals, x, self.full_rows, self.full_row_indices, y, self.outfeatures,
               self.qweight, self.lookup_table)
        elif self.include_sparse:
            fn = getattr(quant_cuda, f"vecquant{b}matmul_spmv_nuq_perchannel{sfx}")
            fn(self.rows, self.cols, self.vals, x, y, self.outfeatures, self.qweight, self.lookup_table)
        else:
            fn = getattr(quant_cuda, f"vecquant{b}matmul_nuq_perchannel{sfx}")
            fn(x, self.qweight, y, self.lookup_table)


class _QuantLinearLUTFunction(torch.autograd.Function):
    """y = QuantLinearLUT._forward_impl(x) with dx = dy . W^T.  `names` are the layer's trained tensors
    (QuantLinearLUT.train_codebook) and `params` their values: the codebook / CSR-value / dense-row gradients come from
    G = x^T . dy in one quant_cuda.lut_grad launch, dbias = sum of dy over the rows.  Without trained tensors the buffers are
    constants and only x gets a gradient.  x is saved only when one of the first three is wanted."""

    @staticmethod
    def forward(ctx, x, layer, names, *params):
        ctx.layer, ctx.names = layer, names
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        # the buffers are read again at backward time: remember their versions, so that an in-place change in between (a weight
        # reload) raises instead of silently giving the gradient of the new weights
        ctx.versions = [(t, t._version) for t in layer._grad_buffers() + ((layer.bias,) if "bias" in names else ())]
        ctx.grid_names = tuple(n for i, n in enumerate(names) if n != "bias" and ctx.needs_input_grad[3 + i])
        if ctx.grid_names:
            ctx.save_for_backward(x)
        return layer._forward_impl(x)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        layer, names = ctx.layer, ctx.names
        now = layer._grad_buffers() + ((layer.bias,) if "bias" in names else ())
        if len(now) != len(ctx.versions) or any(t is not u or t._version != v for (t, v), u in zip(ctx.versions, now)):
            raise RuntimeError("QuantLinearLUT: the layer's buffers were modified or replaced between forward and backward; "
                               "the gradients would use the new weights")
        dy = dy.reshape(-1, layer.outfeatures)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = (layer._input_grad(dy).to(ctx.x_dtype) if dy.shape[0] else
                  torch.zeros(ctx.x_shape, dtype=ctx.x_dtype, device=dy.device)).reshape(ctx.x_shape)
        grads = dict.fromkeys(names)
        if ctx.grid_names:
            (x,) = ctx.saved_tensors
            if dy.shape[0]:
                dlut, dvals, dfull = layer._codebook_grad(x.reshape(-1, layer.infeatures), dy, ctx.grid_names)
                grads.update(lookup_table=dlut, vals=dvals, full_rows=dfull)
            else:
                grads.update({n: torch.zeros_like(getattr(layer, n)) for n in ctx.grid_names})
        if "bias" in names and ctx.needs_input_grad[3 + names.index("bias")]:
            grads["bias"] = dy.sum(0, dtype=torch.float32).to(layer.bias.dtype)
        return (dx, None, None) + tuple(grads[n] if ctx.needs_input_grad[3 + i] else None for i, n in enumerate(names))


def make_quant_lut(module, names, bits, name="", include_sparse=False, numvals=None, topX=0, balanced=False,
                   num_nonzero_per_thread=10):
    """Recursively replace the nn.Linear attributes listed in `names` by QuantLinearLUT
    (reference quant.py:386-435; same signature)."""
    if isinstance(module, QuantLinearLUT):
        return
    for attr in dir(module):
        tmp = getattr(module, attr)
        name1 = name + "." + attr if name != "" else attr
        if name1 in names:
            num = numvals[name1] if numvals is not None else 0
            delattr(module, attr)
            setattr(module, attr, QuantLinearLUT(bits, tmp.in_features, tmp.out_features, tmp.bias is not None,
                                                 include_sparse=include_sparse, numvals=num, topX=topX, balanced=balanced,
                                                 num_nonzero_per_thread=num_nonzero_per_thread))
    for name1, child in module.named_children():
        make_quant_lut(child, names, bits, name + "." + name1 if name != "" else name1, include_sparse=include_sparse,
                       numvals=numvals, topX=topX, balanced=balanced, num_nonzero_per_thread=num_nonzero_per_thread)
