"""In-tree native build of the wukong_b200 libraries (explicit nvcc / g++; no JIT cache).

  libwukong_b200.so   CUDA kernels for sm_90a (H100) + the C-ABI declared in include/wukong_b200.h
  libwukong_host.so   host-side C++ (reference-surface mirror, store builder, data generators),
                      linked against libwukong_b200.so

Both are written next to this file, where capi.py and host.py load them from.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(ROOT, "include")
LIB_CUDA = os.path.join(HERE, "libwukong_b200.so")
LIB_HOST = os.path.join(HERE, "libwukong_host.so")

CUDA_SOURCES = ["kernels/engine.cu", "kernels/store_build.cu", "kernels/table_ops.cu"]
HOST_SOURCES = ["datagen/lubm_gen.cpp", "datagen/rmat_gen.cpp", "store/host_builder.cpp", "host/host_capi.cpp"]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-fopenmp", "-shared",
              "-cudart", "static"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", "-shared", "-Wall", "-Wno-sign-compare", "-pthread"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    for s in sources:
        if os.path.getmtime(s) > t:
            return True
    return False


def _deps(subdirs):
    out = []
    for d in subdirs:
        for base, _, files in os.walk(d):
            for f in files:
                if f.endswith((".cu", ".cuh", ".cpp", ".hpp", ".h")):
                    out.append(os.path.join(base, f))
    return out


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: the CUDA library cannot be built")


def build_cuda(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in CUDA_SOURCES]
    deps = _deps([os.path.join(CSRC, "kernels"), INCLUDE])
    if not force and not _newer(LIB_CUDA, deps + [__file__]):
        return LIB_CUDA
    cmd = [_nvcc()] + NVCC_FLAGS + ["-I", INCLUDE, "-I", os.path.join(CSRC, "kernels")]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += srcs + ["-o", LIB_CUDA]
    print("[build]", " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB_CUDA


def build_host(force=False):
    srcs = [os.path.join(CSRC, s) for s in HOST_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = _deps([os.path.join(CSRC, "datagen"), os.path.join(CSRC, "store"), os.path.join(CSRC, "host"), INCLUDE])
    if not force and not _newer(LIB_HOST, deps + [__file__]):
        return LIB_HOST
    # the system g++: a $CXX wrapper that links libstdc++ statically breaks iostreams in a dlopen()ed library
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
    cmd = [cxx] + CXX_FLAGS + ["-I", INCLUDE, "-I", CSRC] + srcs + ["-o", LIB_HOST]
    # the host library calls the GPU engine through the C-ABI only
    cmd += ["-L", HERE, "-l:libwukong_b200.so", "-Wl,-rpath,$ORIGIN"]
    print("[build]", " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return LIB_HOST


def build_all(force=False, verbose=False):
    build_cuda(force=force, verbose=verbose)
    build_host(force=force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
