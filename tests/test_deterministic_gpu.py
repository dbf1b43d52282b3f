"""The deterministic fused mode (sqllm_set_deterministic(1)) runs the multi-row LUT-GEMV (lutgemv_rows.cuh) at one row.  Pinned here:
a deterministic one-row call has the same bits as that row inside a multi-row call (fp16 and bf16 x, both widths, CSR outliers and
dense rows); fp32 x, which only this mode sends to the multi-row kernel, is within the per-element bound of tests/util.py and
reproducible; in_features above SQLLM_ROWS_MAX_IN is taken; and sqllm_workspace_bytes does not depend on the mode."""
import numpy as np
import pytest
import torch

from test_decode_bf16_gpu import Mode, _torch_layer, check, fused_dt, lib, rows_dt  # noqa: F401 (lib: the module's ctypes fixture)
from util import make_activations, orc

pytestmark = pytest.mark.gpu

SHAPES = [(4096, 4096), (512, 132)]  # a 7B layer, and a narrow one with a ragged last strip


def _layer(bits, K, N, seed=0):
    L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=seed + K + N + bits, nonzero_full_rows=True, bias=True)
    return L, _torch_layer(L, 0)


def _bindings(T, x):
    from squeezellm_b200.quant import quant_cuda as qc
    lay = (T["qweight"], T["lookup_table"], T["bits"], T["bias"], T["rows"], T["cols"], T["vals"], T["full_rows"], T["full_row_indices"])
    rows = qc.lutgemv_rows_bf16 if x.dtype == torch.bfloat16 else qc.lutgemv_rows
    return qc.lutgemv_fused, rows, lay


@pytest.mark.parametrize("K,N", SHAPES, ids=[f"{k}x{n}" for k, n in SHAPES])
@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("M", [2, 5])
def test_one_row_has_the_bits_of_its_row_in_a_multirow_call(lib, K, N, bits, dtype, M):
    L, T = _layer(bits, K, N)
    x = torch.from_numpy(make_activations(K, M, seed=bits)).cuda().to(dtype)
    fused, rows, lay = _bindings(T, x)
    many = rows(x, *lay)
    many32 = rows_dt(lib, L, T, x, torch.float32, T["bias"])
    with Mode(lib, True):
        for i in range(M):
            one = fused(x[i].contiguous(), *lay)
            torch.cuda.synchronize()
            assert one.dtype == dtype and torch.equal(one, many[i]), f"row {i}, y in x's dtype"
            one32 = fused_dt(lib, L, T, x[i].contiguous(), torch.float32, T["bias"])
            assert torch.equal(one32, many32[i]), f"row {i}, fp32 y"


@pytest.mark.parametrize("K,N", SHAPES, ids=[f"{k}x{n}" for k, n in SHAPES])
@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("y_dtype", [torch.float32, torch.float16], ids=["y32", "y16"])
def test_fp32_x_within_bound_and_reproducible(lib, K, N, bits, y_dtype):
    L, T = _layer(bits, K, N, seed=1)
    x = (np.random.default_rng(K + bits).standard_normal(K) * 0.7).astype(np.float32)  # not fp16-exact
    xt = torch.from_numpy(x).cuda()
    with Mode(lib, True):
        y0 = fused_dt(lib, L, T, xt, y_dtype, T["bias"])
        y1 = fused_dt(lib, L, T, xt, y_dtype, T["bias"])
    assert torch.equal(y0, y1)
    check(y0, L, x[None, :], L["bias"], str(y_dtype).split(".")[1])


@pytest.mark.parametrize("bits", [3, 4])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
def test_in_features_above_the_rows_limit(lib, bits, dtype):
    K, N = 65536, 128
    assert K > 49152  # SQLLM_ROWS_MAX_IN: the public multi-row entry point refuses this layer
    L, T = _layer(bits, K, N, seed=2)
    xt = torch.from_numpy(make_activations(K, 1, seed=5)[0]).cuda().to(dtype)
    with Mode(lib, True):
        y = fused_dt(lib, L, T, xt, torch.float32, T["bias"])
    check(y, L, xt.float().cpu().numpy()[None, :], L["bias"])


def test_workspace_size_does_not_depend_on_the_mode(lib):
    L, T = _layer(4, 4096, 4096, seed=3)
    sizes = []
    for det in (0, 1):
        with Mode(lib, det):
            sizes.append(lib.sqllm_workspace_bytes(4, 4096, 4096, 10))
    assert sizes[0] == sizes[1] > 0
    xt = torch.from_numpy(make_activations(4096, 1, seed=6)[0]).cuda().half()
    with Mode(lib, True):
        y = fused_dt(lib, L, T, xt, torch.float32, T["bias"])  # a workspace of exactly sqllm_workspace_bytes
    check(y, L, xt.float().cpu().numpy()[None, :], L["bias"])
