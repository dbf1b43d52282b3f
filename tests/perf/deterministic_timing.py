#!/usr/bin/env python3
"""Cost of the deterministic fused mode (sqllm_set_deterministic(1)) against the default one, per one-row GEMV, on the four launch
shapes of one LLaMA-7B decoder layer (q/k/v 4096x12288, o 4096x4096, gate/up 4096x22016, down 11008x4096), w4-s45 and w3-s45
(0.45 % CSR outliers, 10 dense rows), fp16 x -> fp16 y and fp32 x -> fp32 y, through sqllm_lutgemv_fused_dt.

Every library named with --lib (default: this tree's) is loaded side by side through ctypes, so that two builds can be compared in
one process: the (library, mode) arms are alternated inside every repetition.  An arm is one CUDA graph of CALLS launches, warmed
up, then timed with CUDA events over REPLAYS replays; the median of REPS repetitions is kept.

Output, one JSON line each: the card and its power limit (nvidia-smi, read-only query); per (bits, x dtype, shape) the us per call of
every arm and each arm's max relative error against the first library's default mode on the timed input; per (bits, x dtype) the
sum over the four launches of every arm and its ratio to the same library's default mode.

    python tests/perf/deterministic_timing.py [--lib A.so --lib B.so ...] [--quick]
"""
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from prefill_tc_timing import rel, synth  # noqa: E402
from util import Args  # noqa: E402

SHAPES = [("qkv", 4096, 12288), ("o", 4096, 4096), ("gate_up", 4096, 22016), ("down", 11008, 4096)]
CALLS, REPLAYS, REPS = 20, 10, 7
F32, F16 = 0, 1


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    lib.sqllm_last_error.restype = ctypes.c_char_p
    lib.sqllm_workspace_bytes.restype = ctypes.c_size_t
    lib.sqllm_lutgemv_fused_dt.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return lib


class Arm:
    """One library in one mode on one layer: its own zeroed workspace and output, and a graph of CALLS launches."""

    def __init__(self, lib, det, L, x):
        self.lib, self.det = lib, det
        a = Args(bits=L["bits"], in_features=L["K"], out_features=L["N"], batch=1, qweight=L["qweight"].data_ptr(),
                 lookup_table=L["lut"].data_ptr(), rows=L["rows"].data_ptr(), cols=L["cols"].data_ptr(), vals=L["vals"].data_ptr(),
                 full_rows=L["full_rows"].data_ptr(), full_row_indices=L["fri"].data_ptr(), topX=L["full_rows"].shape[1])
        self.a, self.x = a, x
        self.xdt = F32 if x.dtype == torch.float32 else F16
        self.y = torch.empty(L["N"], dtype=x.dtype, device="cuda")
        lib.sqllm_set_deterministic(det)
        self.nbytes = lib.sqllm_workspace_bytes(a.bits, a.in_features, a.out_features, a.topX)
        assert self.nbytes > 0, lib.sqllm_last_error()
        self.ws = torch.zeros(self.nbytes, dtype=torch.uint8, device="cuda")
        for _ in range(3):  # warm-up: module load, shared-memory set-up and the one-time probe stay out of the capture
            self.call()
        torch.cuda.synchronize()
        self.g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g):
            for _ in range(CALLS):
                self.call()
        self.g.replay()
        torch.cuda.synchronize()

    def call(self):
        rc = self.lib.sqllm_lutgemv_fused_dt(ctypes.byref(self.a), self.x.data_ptr(), self.xdt, self.y.data_ptr(), self.xdt, None,
                                             self.ws.data_ptr(), self.nbytes, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, self.lib.sqllm_last_error()

    def us_per_call(self):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(REPLAYS):
            self.g.replay()
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) * 1e3 / (REPLAYS * CALLS)


def main():
    quick = "--quick" in sys.argv
    paths = [sys.argv[i + 1] for i, v in enumerate(sys.argv) if v == "--lib"] or [os.path.join(ROOT, "squeezellm_b200", "libsqllm_b200.so")]
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"kind": "card", "nvidia_smi": q.stdout.strip().splitlines()[:1], "libs": paths}), flush=True)
    libs = [load(p) for p in paths]
    names = [f"lib{i}" for i in range(len(libs))]
    reps = 2 if quick else REPS
    for bits in (4, 3):
        for xdt in (torch.float16, torch.float32):
            layer = {}
            for shape, K, N in (SHAPES[:1] if quick else SHAPES):
                L = synth(bits, K, N, 0.0045, 10)
                x = (torch.randn(K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(K)) * 0.5).to(xdt)
                arms = {(n, det): Arm(lib, det, L, x) for n, lib in zip(names, libs) for det in (0, 1)}
                ts = {k: [] for k in arms}
                for _ in range(reps):
                    for k, arm in arms.items():
                        ts[k].append(arm.us_per_call())
                want = arms[(names[0], 0)].y
                line = {"kind": "shape", "bits": bits, "x": str(xdt).split(".")[1], "shape": shape, "K": K, "N": N}
                for (n, det), arm in arms.items():
                    key = f"{n}_{'det' if det else 'default'}"
                    line[key + "_us"] = round(statistics.median(ts[(n, det)]), 3)
                    line[key + "_spread_us"] = round(max(ts[(n, det)]) - min(ts[(n, det)]), 3)
                    line[key + "_rel_err"] = float(f"{rel(arm.y.float(), want.float()):.3e}")
                    layer[key] = layer.get(key, 0.0) + line[key + "_us"]
                print(json.dumps(line), flush=True)
                del arms
                torch.cuda.synchronize()
            out = {"kind": "layer", "bits": bits, "x": str(xdt).split(".")[1]}
            for n in names:
                out[f"{n}_default_us"] = round(layer[f"{n}_default"], 3)
                out[f"{n}_det_us"] = round(layer[f"{n}_det"], 3)
                out[f"{n}_det_over_default"] = round(layer[f"{n}_det"] / layer[f"{n}_default"], 3)
            print(json.dumps(out), flush=True)
    for lib in libs:
        lib.sqllm_set_deterministic(0)


if __name__ == "__main__":
    main()
