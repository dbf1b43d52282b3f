#!/usr/bin/env python3
"""Generate golden outputs of the REFERENCE's own CUDA kernels on an H100 (oracle/_ref/quant_cuda_ref*.so, built by
oracle/build_ref.py from a reference checkout with the 8-site dtype patch):

    python tests/golden/make_golden_gpu.py [--out DIR]      # default DIR: tests/golden

refkernel_<case>.npz: the inputs (reference buffer format), the initial `mul`, and `mul_out` after calling the reference
symbol that squeezellm/quant.py would pick.  They pin the CPU oracle's arithmetic
(tests/test_oracle_golden.py::test_oracle_matches_reference_kernel_outputs).  Kept small so the fixtures stay a few hundred KB.

reference_outputs.npz: for every case of tests/test_gpu_parity.py that compares with the reference kernels, the reference's
output at the positions tests/util.py:sample_idx keeps, and max |output| over the whole output (key + "__absmax").  The inputs
are not stored: the tests rebuild them from the same seeds (matvec_inputs / batched_inputs).
Shapes respect the reference's unchecked preconditions (in % 128 == 0, out % 128 == 0).
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import build_ref  # noqa: E402
import oracle as orc  # noqa: E402
import test_gpu_parity as t  # noqa: E402
from util import sample_idx, to_torch  # noqa: E402

CASES = [  # name, bits, K, N, sparsity, topX, nonzero_full_rows, batch
    ("w4_dense", 4, 256, 128, 0.0, 0, False, 1),
    ("w3_dense", 3, 256, 128, 0.0, 0, False, 1),
    ("w4_spmv", 4, 256, 256, 0.01, 0, False, 1),
    ("w3_spmv", 3, 384, 128, 0.01, 0, False, 1),
    ("w4_hybrid", 4, 256, 128, 0.01, 10, True, 1),
    ("w3_hybrid", 3, 256, 128, 0.01, 10, True, 1),
    ("w4_dense_batched", 4, 128, 128, 0.0, 0, False, 3),
    ("w3_hybrid_batched", 3, 128, 128, 0.02, 4, True, 3),
]


def call(ref, L, xv, mul, batched):
    """The reference symbol squeezellm/quant.py would pick, chosen exactly as the parity tests choose it."""
    t._module_call(ref, to_torch(L), xv, mul, batched)
    torch.cuda.synchronize()


def oracle_cases(ref, out):
    for name, bits, K, N, sp, topx, nz, batch in CASES:
        L = orc.make_layer(bits, K, N, sparsity=sp, topX=topx, seed=100 + CASES.index((name, bits, K, N, sp, topx, nz, batch)), nonzero_full_rows=nz)
        x = orc.make_vec(K, batch=batch, seed=17)
        init = (np.random.default_rng(5).standard_normal((batch, N)) * 0.5).astype(np.float32)
        xv = torch.from_numpy(x).cuda() if batch > 1 else torch.from_numpy(x).cuda().reshape(-1)
        mul = torch.from_numpy(init.copy()).cuda() if batch > 1 else torch.from_numpy(init.copy()).cuda().reshape(-1)
        call(ref, L, xv, mul, batch > 1)
        d = dict(bits=bits, K=K, N=N, vec=x, mul_init=init, mul_out=mul.cpu().numpy().reshape(batch, N))
        for k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices"):
            if L[k] is not None:
                d[k] = L[k]
        np.savez_compressed(os.path.join(out, f"refkernel_{name}.npz"), **d)
        e = np.abs(d["mul_out"] - orc.forward_f64(L, x, mul_init=init)).max()
        print(f"{name}: max |ref_kernel - oracle_f64| = {e:.3e}")


def parity_cases(ref, out):
    g = {}

    def keep(key, y):
        y = y.cpu().numpy().reshape(-1)
        g[key] = y[sample_idx(y.size)].astype(np.float32)
        g[key + "__absmax"] = np.float64(np.abs(y).max())

    for shape, sid in zip(t.SHAPES, t.IDS):
        if t.ref_comparable(shape):
            L, x = t.matvec_inputs(shape)
            y = torch.zeros(shape[2], device="cuda")
            call(ref, L, torch.from_numpy(x).cuda(), y, False)
            keep("mv__" + sid, y)
    for shape in t.BATCHED_SHAPES:
        if t.ref_comparable(shape):
            for batch in t.BATCHES:
                L, x = t.batched_inputs(shape, batch)
                y = torch.zeros((batch, shape[2]), device="cuda")
                call(ref, L, torch.from_numpy(x).cuda(), y, True)
                keep(f"b{batch}__{t.batched_id(shape)}", y)
    np.savez_compressed(os.path.join(out, "reference_outputs.npz"), **g)
    print(f"reference_outputs.npz: {len(g) // 2} outputs")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    ref = build_ref.load()
    print(torch.cuda.get_device_name(0))
    oracle_cases(ref, args.out)
    parity_cases(ref, args.out)


if __name__ == "__main__":
    main()
