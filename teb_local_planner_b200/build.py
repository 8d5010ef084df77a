"""Builds the in-tree CUDA shared library (sm_90a, H100) with nvcc. No JIT cache: the .so travels with the repo."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libteb_b200.so")
SOURCES = [os.path.join(CSRC, "teb_cabi.cu")]
DEPS = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))) + [
    os.path.join(os.path.dirname(HERE), "include", "teb_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-Xlinker", "-rpath=/usr/local/cuda/lib64"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = [NVCC] + FLAGS + ["-o", LIB] + SOURCES + ["-lcudart", "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libteb_b200.so")
    with open(os.path.join(HERE, "ptxas_info.txt"), "w") as f:
        f.write(res.stderr)
    return LIB


HOST_DIR = os.path.join(HERE, "host")
HOST_LIB = os.path.join(HERE, "libteb_local_planner_b200.so")
HOST_TEST = os.path.join(HOST_DIR, "test", "test_dropin")
HOST_TEST_LARGE = os.path.join(HOST_DIR, "test", "test_dropin_large")  # the drop-in classes on a 3000-obstacle scene
HOST_PIN = os.path.join(HOST_DIR, "test", "libteb_host_pin.so")   # test infrastructure: band operations for tests/test_host_pin.py
HOST_SRCS = [os.path.join(HOST_DIR, "src", f) for f in ("timed_elastic_band.cpp", "optimal_planner.cpp",
                                                         "homotopy_class_planner.cpp", "graph_search.cpp")]


def build_host(force=False, verbose=False):
    """Drop-in C++ classes (TebOptimalPlanner, HomotopyClassPlanner, TimedElasticBand ...) over the C-ABI + their test."""
    inc = ["-I", os.path.join(os.path.dirname(HERE), "include"), "-I", os.path.join(HOST_DIR, "include")]
    hdrs = [os.path.join(dp, f) for dp, _, fs in os.walk(os.path.join(HOST_DIR, "include")) for f in fs]
    deps = HOST_SRCS + hdrs + [os.path.join(HOST_DIR, "test", "test_dropin.cpp"), os.path.join(HOST_DIR, "test", "pin_api.cpp"),
                                  os.path.join(HOST_DIR, "test", "test_dropin_large.cpp"), LIB]
    outs = (HOST_LIB, HOST_TEST, HOST_PIN, HOST_TEST_LARGE)
    if (not force and all(os.path.exists(o) for o in outs)
            and all(os.path.getmtime(d) <= min(os.path.getmtime(o) for o in outs) for d in deps)):
        return HOST_LIB
    gxx = os.environ.get("CXX", "g++")
    # -ffp-contract=off: no fused multiply-adds, like the generic x86-64 builds of the reference - the drop-in layer's
    # arithmetic is pinned bit for bit against the reference's code (tests/test_host_pin.py)
    common = [gxx, "-std=c++17", "-O2", "-fPIC", "-Wall", "-Wextra", "-march=x86-64-v3", "-ffp-contract=off"] + inc
    link = ["-L", HERE, "-lteb_b200", "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + HERE]
    cmds = [common + ["-shared", "-o", HOST_LIB] + HOST_SRCS + link,
            common + ["-I", "/usr/local/cuda/include", "-o", HOST_TEST, os.path.join(HOST_DIR, "test", "test_dropin.cpp"), "-L", HERE,
                      "-lteb_local_planner_b200", "-lteb_b200", "-L", "/usr/local/cuda/lib64", "-lcudart",
                      "-Wl,-rpath," + HERE, "-Wl,-rpath,/usr/local/cuda/lib64"],
            common + ["-o", HOST_TEST_LARGE, os.path.join(HOST_DIR, "test", "test_dropin_large.cpp"), "-L", HERE,
                      "-lteb_local_planner_b200", "-lteb_b200", "-Wl,-rpath," + HERE],
            common + ["-shared", "-o", HOST_PIN, os.path.join(HOST_DIR, "test", "pin_api.cpp"), "-L", HERE,
                      "-lteb_local_planner_b200", "-lteb_b200", "-Wl,-rpath," + HERE]]
    for cmd in cmds:
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host drop-in layer")
    return HOST_LIB


if __name__ == "__main__":
    build(force=True, verbose=True)
    build_host(force=True, verbose=True)
    print(LIB, HOST_LIB)
