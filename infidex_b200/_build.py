"""Build the native libraries of infidex_b200 in-tree (sm_90a, H100, only)."""
import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
GPU_LIB = os.path.join(PKG, "libinfidex_gpu.so")
HOST_LIB = os.path.join(PKG, "libinfidex_host.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC"]
GXX_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-pthread"]


def _stale(lib, srcs):
    return not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs)


def _sources():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(PKG, "..", "include", f) for f in ("infidex_gpu.h", "infidex_host.h")]


def build_host(force=False):
    if force or _stale(HOST_LIB, _sources()):
        subprocess.check_call(["g++"] + GXX_FLAGS + ["-o", HOST_LIB, os.path.join(CSRC, "ifx_host_build.cpp"), os.path.join(CSRC, "ifx_synth.cpp")])
    return HOST_LIB


def build_gpu(force=False, verbose=False):
    if force or _stale(GPU_LIB, _sources()):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", GPU_LIB, os.path.join(CSRC, "ifx_api.cu")]
        subprocess.check_call(cmd)
    return GPU_LIB


def build_all(force=False):
    return build_host(force), build_gpu(force)
