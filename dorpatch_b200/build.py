"""Build libdorpatch.so in-tree with nvcc for sm_90a (H100).

    python -m dorpatch_b200.build [--force]

The library links the CUDA runtime, cuDNN and cublasLt dynamically by SONAME; at run time
they resolve to the copies PyTorch has already loaded (same process) or, in a torch-free
process, through the RPATH entries below.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdorpatch.so")
SOURCES = ["kernels_net.cu", "kernels_patch.cu", "kernels_stem.cu", "kernels_gemm.cu", "kernels_wgrad.cu", "engine.cu"]
HEADERS = ["common.cuh", "kernels.h", os.path.join("..", "..", "include", "dorpatch.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _site_nvidia():
    import importlib.util
    spec = importlib.util.find_spec("nvidia")
    if spec is None or not spec.submodule_search_locations:
        return None
    return list(spec.submodule_search_locations)[0]


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    srcs = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return _newest(srcs) > os.path.getmtime(LIB_PATH)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nv = _site_nvidia()
    inc, libdirs = [], []
    if nv:
        for sub in ("cudnn", "cublas", "cuda_runtime"):
            i, l = os.path.join(nv, sub, "include"), os.path.join(nv, sub, "lib")
            if os.path.isdir(i):
                inc += ["-I", i]
            if os.path.isdir(l):
                libdirs.append(l)
    sys_inc = "/usr/include/x86_64-linux-gnu"
    if os.path.exists(os.path.join(sys_inc, "cudnn.h")):
        inc += ["-I", sys_inc]
    libdirs += ["/usr/lib/x86_64-linux-gnu", "/usr/local/cuda/lib64"]
    common = ["nvcc", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wno-deprecated-declarations",
              "-Wno-deprecated-declarations", "-cudart", "shared"] + ARCH + inc
    if verbose:
        common += ["-Xptxas", "-v"]
    objs = []
    for s in SOURCES:
        o = os.path.join(LIB_DIR, s.replace(".cu", ".o"))
        cmd = common + ["-c", os.path.join(CSRC, s), "-o", o]
        subprocess.run(cmd, check=True)
        objs.append(o)
    link = ["nvcc", "-shared", "-cudart", "shared"] + ARCH + objs + ["-o", LIB_PATH]
    for d in libdirs:
        link += ["-L", d, "-Xlinker", "-rpath," + d]
    link += ["-l:libcudnn.so.9", "-l:libcublasLt.so.12"]
    subprocess.run(link, check=True)
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
