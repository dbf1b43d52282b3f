#!/usr/bin/env python3
"""Generate tests/golden/reference_quant_py.json: what the REFERENCE's squeezellm/quant.py asks of the `quant_cuda` extension.

Run with a reference checkout (after `python -m squeezellm_b200.build`):
    python tests/golden/make_golden_quant_py.py <reference checkout>

The reference module is imported unmodified; its `import quant_cuda` resolves to OUR extension.  Recorded: every
`quant_cuda.<name>` it calls, and the buffers (name, shape, dtype) of its QuantLinearLUT(4, 128, 128, bias=False,
include_sparse=True, numvals=5, topX=10).  tests/test_abi.py checks our extension and module against both.
"""
import importlib.util
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import squeezellm_b200.quant  # noqa: F401  (registers the in-tree extension as module `quant_cuda`)
    path = os.path.join(sys.argv[1], "squeezellm", "quant.py")
    spec = importlib.util.spec_from_file_location("reference_quant", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    called = sorted(set(re.findall(r"quant_cuda\.(\w+)", open(path).read())))
    m = mod.QuantLinearLUT(4, 128, 128, False, include_sparse=True, numvals=5, topX=10)
    buffers = {k: [list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in m.state_dict().items()}
    out = os.path.join(ROOT, "tests", "golden", "reference_quant_py.json")
    with open(out, "w") as f:
        json.dump({"called_symbols": called, "quantlinearlut_w4_128x128_sparse5_topx10": buffers}, f, indent=1)
        f.write("\n")
    print(out)


if __name__ == "__main__":
    main()
