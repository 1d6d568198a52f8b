"""Builds and binds tests/emu/emu_depth.cpp: the emulated polish kernels (tests/emu_lib.py) in depth mode (and status mode), with the
runs kernels; and depth_tenths with the host's depth text.  TEST INFRASTRUCTURE ONLY (logic checks without a GPU); never used by the
product."""
import ctypes as C
import os
import subprocess

import numpy as np

from polypolish_b200 import api
from tests import emu_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "emu_depth.cpp")
LIB = os.path.join(ROOT, "build", "libemu_depth.so")
DEPS = emu_lib.DEPS + [SRC, os.path.join(ROOT, "polypolish_b200", "csrc", "debug_rows.h")]


def build():
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        tmp = "%s.%d.tmp" % (LIB, os.getpid())           # several test workers may build at once: compile aside, rename atomically
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-g", "-shared", "-fPIC", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                               "-Wno-unused-variable", "-Wno-strict-aliasing", "-ffp-contract=off", "-I", os.path.join(ROOT, "tests", "emu"), SRC,
                               "-o", tmp])
        os.replace(tmp, LIB)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.emu_polish_depth.argtypes = [C.POINTER(api.Contigs), C.POINTER(api.Alignments), C.POINTER(api.PolishParams),
                                          C.POINTER(api.PolishResult), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_ulonglong), C.POINTER(C.c_char_p),
                                          C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        _lib.emu_depth_tenths.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        _lib.emu_depth_tenths.restype = C.c_uint64
        _lib.emu_depth_text.argtypes = [C.c_void_p, C.c_uint64]
        _lib.emu_depth_text.restype = C.c_void_p
        _lib.emu_free.argtypes = [C.c_void_p]
    return _lib


def _take(p):
    text = C.string_at(p.value) if p.value else b""
    lib().emu_free(p.value)
    return text


def polish(fasta, packed, grid_tiles=2, with_changes=False, with_status=False, **opts):
    """Like emu_lib.polish, plus the depth runs (the bytes `polish --depth-bedgraph` writes) under "bedgraph", and with with_status
    the status runs of the same call (the bytes of `polish --status-bed`) under "bed"."""
    prm = api._params(**opts)
    n = fasta.view.n_contigs
    G = int(fasta.off[-1])
    cap = G + G // 4 + (1 << 20)
    keep = dict(off=np.zeros(n + 1, np.uint64), bases=np.zeros(cap, np.uint8), changed=np.zeros(n, np.uint64), zero=np.zeros(n, np.uint64),
                tdepth=np.zeros(n, np.float64))
    res = api.PolishResult()
    res.out_off, res.out_bases, res.out_cap = keep["off"].ctypes.data, keep["bases"].ctypes.data, cap
    res.changed, res.zero_depth, res.total_depth = keep["changed"].ctypes.data, keep["zero"].ctypes.data, keep["tdepth"].ctypes.data
    err = C.c_ulonglong()
    names = (C.c_char_p * max(1, n))(*[x.encode() for x in fasta.names])
    bedgraph, bed = C.c_void_p(), C.c_void_p()
    rc = lib().emu_polish_depth(C.byref(fasta.view), C.byref(packed.view), C.byref(prm), C.byref(res), grid_tiles, int(with_changes),
                                int(with_status), C.byref(err), names, C.byref(bedgraph), C.byref(bed))
    bedgraph, bed = _take(bedgraph), _take(bed)
    if rc == api.PP_ERR_INPUT:
        return dict(error=emu_lib.ERR_TEXT.get(err.value & 0xFF, "?"), error_aln=err.value >> 8)
    assert rc == 0, rc
    off = keep["off"]
    return dict(sequences=[keep["bases"][int(off[i]):int(off[i + 1])].tobytes() for i in range(n)], changed=keep["changed"].tolist(),
                zero=keep["zero"].tolist(), tdepth=keep["tdepth"].tolist(), bedgraph=bedgraph, bed=bed)


def depth_tenths(x):
    """depth_tenths of every double in x (numpy array), and the index of the first whose depth text is not snprintf("%.1f") (len(x):
    none)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    t = np.zeros(max(1, len(x)), np.uint64)
    bad = lib().emu_depth_tenths(x.ctypes.data, len(x), t.ctypes.data)
    return t[:len(x)], int(bad)


def depth_text(tenths):
    """The host's depth text (pp::depth_text) of every key, one per line."""
    t = np.ascontiguousarray(tenths, dtype=np.uint64)
    return _take(C.c_void_p(lib().emu_depth_text(t.ctypes.data, len(t))))
