"""Builds and binds tests/emu/emu_polish.cpp: the polish kernels (polypolish_b200/csrc/polish_dev.cuh) compiled for the CPU
against a small CUDA-emulation shim, with the per-position reports on request.  TEST INFRASTRUCTURE ONLY (logic checks without a
GPU); never used by the product."""
import ctypes as C
import os
import subprocess

import numpy as np

from polypolish_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "emu_polish.cpp")
LIB = os.path.join(ROOT, "build", "libemu_polish.so")
DEPS = [SRC, os.path.join(ROOT, "tests", "emu", "cuda_emu.h"), os.path.join(ROOT, "polypolish_b200", "csrc", "polish_dev.cuh"),
        os.path.join(ROOT, "polypolish_b200", "csrc", "nib_utils.h"), os.path.join(ROOT, "include", "pp_abi.h"),
        os.path.join(ROOT, "polypolish_b200", "csrc", "debug_rows.h")]
# the report texts emu_polish returns, in the order of its `reports` bits
REPORTS = ("changes", "debug_tsv", "bed", "bedgraph")


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
        _lib.emu_polish_reports.argtypes = [C.POINTER(api.Contigs), C.POINTER(api.Alignments), C.POINTER(api.PolishParams),
                                            C.POINTER(api.PolishResult), C.c_int, C.c_uint, C.POINTER(C.c_char_p), C.POINTER(C.c_ulonglong),
                                            C.POINTER(C.c_void_p)]
        _lib.emu_last_layout.argtypes = [C.POINTER(C.c_uint32)] * 3 + [C.c_void_p] * 3
        _lib.emu_depth_tenths.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        _lib.emu_depth_tenths.restype = C.c_uint64
        _lib.emu_depth_text.argtypes = [C.c_void_p, C.c_uint64]
        _lib.emu_depth_text.restype = C.c_void_p
        _lib.emu_free.argtypes = [C.c_void_p]
    return _lib


ERR_TEXT = {1: "query name in SAM but not in assembly", 2: "CIGAR string does not match read sequence", 3: "unexpected character",
            4: "alignment extends past the end of its reference sequence", 5: "no alignments for read contain sequence"}


def _take(p):
    text = C.string_at(p) if p else b""
    lib().emu_free(p)
    return text


def polish(fasta, packed, grid_tiles=2, changes=False, debug=False, status=False, depth=False, **opts):
    """The emulated kernels on a loaded assembly + packed alignments: dict like Context.polish_packed, or ('err', code, aln).  The
    reports asked for are recorded in the same call, the bytes `polish` writes for them under "changes" (--changes), "debug_tsv"
    (--debug), "bed" (--status-bed) and "bedgraph" (--depth-bedgraph)."""
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
    asked = (changes, debug, status, depth)
    names = (C.c_char_p * max(1, n))(*([x.encode() for x in fasta.names] if any(asked) else []))
    texts = (C.c_void_p * len(REPORTS))()
    rc = lib().emu_polish_reports(C.byref(fasta.view), C.byref(packed.view), C.byref(prm), C.byref(res), grid_tiles,
                                  sum(1 << i for i, on in enumerate(asked) if on), names, C.byref(err), texts)
    reports = {key: _take(texts[i]) for i, key in enumerate(REPORTS) if asked[i]}
    if rc == api.PP_ERR_INPUT:
        return dict(error=ERR_TEXT.get(err.value & 0xFF, "?"), error_aln=err.value >> 8)
    assert rc == 0, rc
    off = keep["off"]
    return dict(sequences=[keep["bases"][int(off[i]):int(off[i + 1])].tobytes() for i in range(n)], changed=keep["changed"].tolist(),
                zero_depth=keep["zero"].tolist(), total_depth=keep["tdepth"].tolist(), n_aln_used=res.n_aln_used,
                global_k=bool(lib().emu_last_global_k()), max_ext=lib().emu_last_max_ext(), n_long=lib().emu_last_n_long(), **reports)


def last_layout():
    """How the last polish laid the alignments out for k_tile: bin_start (n_bins + 2 entries; the long list is
    [bin_start[n_bins], bin_start[n_bins + 1])), sval (the alignment index in each slot) and tile_order (the order the tiles are
    dealt in: heaviest first)."""
    nb, ns, nt = C.c_uint32(), C.c_uint32(), C.c_uint32()
    lib().emu_last_layout(C.byref(nb), C.byref(ns), C.byref(nt), None, None, None)
    out = dict(bin_start=np.zeros(nb.value + 2, np.uint32), sval=np.zeros(ns.value, np.uint32), tile_order=np.zeros(nt.value, np.uint32))
    lib().emu_last_layout(C.byref(nb), C.byref(ns), C.byref(nt), out["bin_start"].ctypes.data, out["sval"].ctypes.data, out["tile_order"].ctypes.data)
    return out


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
    return _take(lib().emu_depth_text(t.ctypes.data, len(t)))


def fasta_bytes(fasta, seqs):
    return b"".join(b">" + fasta.names[i].encode() + ((b" " + fasta.descriptions[i].encode()) if fasta.descriptions[i] else b"") +
                    b" polypolish\n" + seqs[i] + b"\n" for i in range(len(seqs)))
