"""Builds and binds tests/probe/depth_probe.cu: depth_deficit, depth_bounds, bankers_rounding and vote_thresholds of
polypolish_b200/csrc/polish_dev.cuh evaluated per element, on the CPU (g++ against tests/emu/cuda_emu.h) or on the GPU (nvcc for
sm_90a with the product's flags).  TEST INFRASTRUCTURE ONLY; never used by the product."""
import ctypes as C
import os
import subprocess

import numpy as np

from polypolish_b200 import build as product

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "probe", "depth_probe.cu")
LIBS = {"cpu": os.path.join(ROOT, "build", "libdepth_probe_cpu.so"), "gpu": os.path.join(ROOT, "build", "libdepth_probe_gpu.so")}
DEPS = [SRC, os.path.join(ROOT, "tests", "emu", "cuda_emu.h"), os.path.join(ROOT, "polypolish_b200", "csrc", "polish_dev.cuh"),
        os.path.join(ROOT, "polypolish_b200", "csrc", "nib_utils.h"), os.path.join(ROOT, "include", "pp_abi.h"), product.__file__]

IN_DTYPE = np.dtype([("k", "<u4"), ("cover", "<u4"), ("deficit", "<u8"), ("x", "<f8"), ("fv", "<f8"), ("fi", "<f8"),
                     ("min_depth", "<u4"), ("pad", "<u4")])
OUT_DTYPE = np.dtype([("dd", "<u8"), ("lo", "<f8"), ("hi", "<f8"), ("fx", "<f8"), ("br", "<u4"), ("vt", "<u4"), ("it", "<u4"), ("low", "<u4")])


def build(backend):
    lib = LIBS[backend]
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in DEPS):
        tmp = "%s.%d.tmp" % (lib, os.getpid())           # several test workers may build at once: compile aside, rename atomically
        if backend == "cpu":
            cmd = ["g++", "-std=c++20", "-O2", "-shared", "-fPIC", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                   "-Wno-unused-variable", "-ffp-contract=off", "-DPROBE_CPU", "-I", os.path.join(ROOT, "tests", "emu"), "-x", "c++", SRC,
                   "-o", tmp]
        else:                                            # the product's flags: -fmad=false, -ffp-contract=off, sm_90a
            cmd = [product.NVCC] + product.ARCH + product.COMMON + ["-shared", "-x", "cu", SRC, "-o", tmp]
        subprocess.check_call(cmd)
        os.replace(tmp, lib)
    return lib


_libs = {}


def lib(backend):
    if backend not in _libs:
        h = C.CDLL(build(backend))
        h.depth_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong]
        h.depth_probe.restype = C.c_int
        _libs[backend] = h
    return _libs[backend]


def run(backend, **cols):
    """Evaluate the helpers on the elements given as equal-length columns of IN_DTYPE (missing columns are 0); returns the
    OUT_DTYPE array."""
    n = max(len(v) for v in cols.values())
    a = np.zeros(n, IN_DTYPE)
    for k, v in cols.items():
        a[k] = v
    out = np.zeros(n, OUT_DTYPE)
    rc = lib(backend).depth_probe(a.ctypes.data, out.ctypes.data, n)
    assert rc == 0, "depth_probe (%s): CUDA error %d" % (backend, rc)
    return out
