"""The emulator readouts tests/test_emu_ring.py needs, on the libraries tests/emu_lib.py and tests/emu_changes_lib.py build: how the
last emulated run laid the alignments out for k_tile, and one run that records both the change report and the whole --debug TSV.
TEST INFRASTRUCTURE ONLY (logic checks without a GPU); never used by the product."""
import ctypes as C

import numpy as np

from polypolish_b200 import api
from tests import emu_changes_lib, emu_lib


def last_layout():
    """How the last emu_lib.polish laid the alignments out for k_tile: bin_start (n_bins + 2 entries; the long list is
    [bin_start[n_bins], bin_start[n_bins + 1])), sval (the alignment index in each slot) and tile_order (the order the tiles are
    dealt in: heaviest first)."""
    L = emu_lib.lib()
    L.emu_last_layout.argtypes = [C.POINTER(C.c_uint32)] * 3 + [C.c_void_p] * 3
    nb, ns, nt = C.c_uint32(), C.c_uint32(), C.c_uint32()
    L.emu_last_layout(C.byref(nb), C.byref(ns), C.byref(nt), None, None, None)
    out = dict(bin_start=np.zeros(nb.value + 2, np.uint32), sval=np.zeros(ns.value, np.uint32), tile_order=np.zeros(nt.value, np.uint32))
    L.emu_last_layout(C.byref(nb), C.byref(ns), C.byref(nt), out["bin_start"].ctypes.data, out["sval"].ctypes.data, out["tile_order"].ctypes.data)
    return out


def polish_report(fasta, packed, grid_tiles=2, **opts):
    """Like emu_changes_lib.polish, with the statistics of emu_lib.polish and the bytes `polish --debug` writes under "debug_tsv"."""
    L = emu_changes_lib.lib()
    L.emu_polish_report.argtypes = [C.POINTER(api.Contigs), C.POINTER(api.Alignments), C.POINTER(api.PolishParams), C.POINTER(api.PolishResult),
                                    C.c_int, C.POINTER(C.c_ulonglong), C.POINTER(C.c_char_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
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
    tsv, dtsv = C.c_void_p(), C.c_void_p()
    rc = L.emu_polish_report(C.byref(fasta.view), C.byref(packed.view), C.byref(prm), C.byref(res), grid_tiles, C.byref(err), names,
                             C.byref(tsv), C.byref(dtsv))
    texts = []
    for p in (tsv, dtsv):
        texts.append(C.string_at(p.value) if p.value else b"")
        if p.value:
            L.emu_free(p.value)
    if rc == api.PP_ERR_INPUT:
        return dict(error=emu_lib.ERR_TEXT.get(err.value & 0xFF, "?"), error_aln=err.value >> 8)
    assert rc == 0, rc
    off = keep["off"]
    return dict(sequences=[keep["bases"][int(off[i]):int(off[i + 1])].tobytes() for i in range(n)], changed=keep["changed"].tolist(),
                zero_depth=keep["zero"].tolist(), total_depth=keep["tdepth"].tolist(), n_aln_used=res.n_aln_used, changes=texts[0],
                debug_tsv=texts[1])
