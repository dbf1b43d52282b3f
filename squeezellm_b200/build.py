"""In-tree build of the two native artefacts (no JIT cache, so the .so files travel with the tree):

  squeezellm_b200/libsqllm_b200.so                 CUDA kernels + C ABI   (nvcc, sm_90a only)
  squeezellm_b200/quant_cuda.<abi>.so              pybind11 adapter        (g++, links the above)

`python -m squeezellm_b200.build` or `__graft_entry__.build()`.
"""
import os
import shutil
import subprocess
import sys
import sysconfig

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
INCLUDE = os.path.join(ROOT, "include")

NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
              "-Xcompiler", "-fPIC"]  # fast-math deliberately NOT used


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")


def lib_path():
    return os.path.join(PKG, "libsqllm_b200.so")


def ext_path():
    return os.path.join(PKG, "quant_cuda" + sysconfig.get_config_var("EXT_SUFFIX"))


def build_lib(verbose=False):
    src = os.path.join(CSRC, "lutgemv_kernels.cu")
    hdr = os.path.join(INCLUDE, "sqllm_b200.h")
    out = lib_path()
    if _newer(out, [src, hdr, os.path.join(CSRC, "lutgemv_v2.cuh"), os.path.join(CSRC, "lutgemv_seq.cuh"),
                    os.path.join(CSRC, "lutgemm_batched.cuh")]):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        cmd = [nvcc] + NVCC_FLAGS + ["-ccbin", _cxx(), "-I", INCLUDE, "-shared", "-o", out, src]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return out


def build_ext(verbose=False):
    import torch
    from torch.utils import cpp_extension

    build_lib(verbose)
    src = os.path.join(CSRC, "quant_cuda_pybind.cpp")
    hdr = os.path.join(INCLUDE, "sqllm_b200.h")
    out = ext_path()
    if _newer(out, [src, hdr]):
        tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
        inc = []
        for p in cpp_extension.include_paths("cuda") + [sysconfig.get_paths()["include"], INCLUDE]:
            inc += ["-isystem" if "torch" in p or "cuda" in p else "-I", p]
        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
        cmd = [_cxx(), "-std=c++17", "-O2", "-fPIC", "-shared", "-fvisibility=hidden",
               f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=quant_cuda", "-DTORCH_API_INCLUDE_EXTENSION_H",
               *inc, src, "-o", out,
               "-L", PKG, "-lsqllm_b200", "-Wl,-rpath,$ORIGIN",
               "-L", tlib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
               f"-Wl,-rpath,{tlib}"]
        cuda_lib = "/usr/local/cuda/lib64"
        if os.path.isdir(cuda_lib):
            cmd += ["-L", cuda_lib, "-lcudart"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return out


def build_all(verbose=False):
    return build_lib(verbose), build_ext(verbose)


if __name__ == "__main__":
    print(build_all(verbose="-v" in sys.argv))
