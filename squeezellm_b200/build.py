"""In-tree build of the two native artefacts (no JIT cache, so the .so files travel with the tree):

  squeezellm_b200/libsqllm_b200.so                 CUDA kernels + C ABI   (nvcc, sm_90a only)
  squeezellm_b200/quant_cuda.<abi>.so              pybind11 adapter        (g++, links the above)

The library is one translation unit per kernel family (csrc/*.cu), compiled in parallel into squeezellm_b200/obj/ and linked
with one `nvcc -shared`.  A unit is recompiled when it or any header is newer than its object.

`python -m squeezellm_b200.build` or `__graft_entry__.build()`.
"""
import glob
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
INCLUDE = os.path.join(ROOT, "include")
OBJ = os.path.join(PKG, "obj")

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
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    hdrs = [os.path.join(INCLUDE, "sqllm_b200.h")] + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.inc"))
    os.makedirs(OBJ, exist_ok=True)
    objs, jobs = [], []
    for src in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if _newer(obj, [src] + hdrs):
            cmd = [nvcc] + NVCC_FLAGS + ["-ccbin", _cxx(), "-I", INCLUDE, "-c", "-o", obj, src]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd))
            jobs.append((subprocess.Popen(cmd), cmd))
    rcs = [(p.wait(), cmd) for p, cmd in jobs]  # every compile ends before a failure is raised
    for rc, cmd in rcs:
        if rc:
            raise subprocess.CalledProcessError(rc, cmd)
    out = lib_path()
    if _newer(out, objs):
        cmd = [nvcc] + NVCC_FLAGS + ["-ccbin", _cxx(), "-shared", "-o", out] + objs
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return out


def build_ext(verbose=False):
    import torch
    from torch.utils import cpp_extension

    src = os.path.join(CSRC, "quant_cuda_pybind.cpp")
    hdr = os.path.join(INCLUDE, "sqllm_b200.h")
    out = ext_path()
    if not _newer(out, [src, hdr]):
        build_lib(verbose)
        return out
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    inc = []
    for p in cpp_extension.include_paths("cuda") + [sysconfig.get_paths()["include"], INCLUDE]:
        inc += ["-isystem" if "torch" in p or "cuda" in p else "-I", p]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    tmp = tempfile.mkdtemp(prefix="sqllm_ext_")
    obj = os.path.join(tmp, "quant_cuda_pybind.o")
    compile_cmd = [_cxx(), "-std=c++17", "-O2", "-fPIC", "-fvisibility=hidden",
                   f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=quant_cuda", "-DTORCH_API_INCLUDE_EXTENSION_H",
                   *inc, "-c", src, "-o", obj]
    link_cmd = [_cxx(), "-shared", obj, "-o", out,
                "-L", PKG, "-lsqllm_b200", "-Wl,-rpath,$ORIGIN",
                "-L", tlib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
                f"-Wl,-rpath,{tlib}"]
    cuda_lib = "/usr/local/cuda/lib64"
    if os.path.isdir(cuda_lib):
        link_cmd += ["-L", cuda_lib, "-lcudart"]
    if verbose:
        print(" ".join(compile_cmd))
    try:
        # the adapter compiles against the header alone: its compile runs while nvcc builds the library, only the link waits
        proc = subprocess.Popen(compile_cmd)
        try:
            build_lib(verbose)
        finally:
            rc = proc.wait()
        if rc:
            raise subprocess.CalledProcessError(rc, compile_cmd)
        if verbose:
            print(" ".join(link_cmd))
        subprocess.check_call(link_cmd)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return out


def build_all(verbose=False):
    ext = build_ext(verbose)  # builds the library too, overlapped with the adapter's compile
    return lib_path(), ext


if __name__ == "__main__":
    print(build_all(verbose="-v" in sys.argv))
