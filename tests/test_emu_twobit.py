"""The 2-bit staged reads of k_tile on the CPU emulator (tests/emu): the case of tests/twobitgen.py against the oracle - FASTA,
statistics, the whole --debug TSV and the --changes report, byte for byte - each run in a child process under the strict model of
the chunk ring; the escape reads are walked in the chunk loop (none goes to the queue).  And the expansion of 2-bit staged bases into
the 4-bit codes the general walk compares (nib_utils.h read32_2bit) against the 4-bit pool's load_read32.  CPU only."""
import ctypes as C
import os
import random
import subprocess

import pytest

from tests import twobitgen as tg
from tests.test_emu_changes import changed_rows
from tests.test_emu_staged import run_child, tile_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def case(tmp_path_factory, oracle):
    d = tmp_path_factory.mktemp("twobit")
    c = tg.twobit(41)
    fa, sams = c.write(d)
    return d, c, oracle.polish(fa, sams, debug=True)


@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("mode", ["plain", "report"])
def test_emu_twobit(case, mode, grid):
    d, c, exp = case
    r = run_child(d, mode, grid)
    assert "error" not in r, r
    assert r["seq_bits"] == 4
    assert r["fasta"] == exp["fasta"]
    assert r["changed"] == exp["changed"] and r["zero_depth"] == exp["zero_depth"] and r["n_aln_used"] == exp["used_total"]
    for got, want in zip(r["total_depth"], exp["total_depth"]):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want))
    if mode == "plain":
        assert r["n_long"] == 0 and r["n_queued"] == 0
        tiles = tile_slots(c, r["layout"], r["max_ext"])
        esc = lambda k: k.startswith("esc")
        assert sum(ks.count(k) for ks in tiles for k in set(ks) if esc(k)) >= c.facts["n_esc"] > 0
        lane31 = sum(1 for ks in tiles for o in range(31, len(ks), 32) if esc(ks[o]))
        dense = max(sum(map(esc, ks[o:o + 32])) for ks in tiles for o in range(0, len(ks), 32))
        assert lane31 >= 2 and dense >= 4, (lane31, dense)
        assert any(k == "len192" for ks in tiles for k in ks[31::32])
    else:
        assert r["debug_tsv"] == exp["debug_tsv"]
        assert r["changes"] == changed_rows(exp["debug_tsv"])
    assert sum(exp["changed"]) > 0


HARNESS = r"""
#include "nib_utils.h"
extern "C" void nib16_to_2bit(unsigned long long x, uint32_t* code, uint32_t* bad) { *code = pp_nib16_to_2bit(x, *bad); }
extern "C" void r32_2bit(const uint32_t* w, uint32_t ri, unsigned long long* r) { read32_2bit(w, ri, r[0], r[1]); }
extern "C" void r32_4bit(const unsigned long long* w, uint32_t ri, unsigned long long* r) { load_read32(w, 224, false, ri, r[0], r[1]); }
"""


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    d = tmp_path_factory.mktemp("twobit_harness")
    src, out = d / "h.cpp", d / "h.so"
    src.write_text(HARNESS)
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "polypolish_b200", "csrc"), "-o", str(out), str(src)])
    return C.CDLL(str(out))


def test_read32_2bit_every_offset(H):
    """32 bases at every offset of a 192-base read (and the two words past it) from the 2-bit words equal the 4-bit pool's."""
    rng = random.Random(5)
    r2, r4 = (C.c_uint64 * 2)(), (C.c_uint64 * 2)()
    for _ in range(40):
        codes = [rng.randrange(4) for _ in range(224)]
        w2 = (C.c_uint32 * 16)(*[sum(c << (2 * j) for j, c in enumerate(codes[16 * i:16 * i + 16])) for i in range(14)])
        w4 = (C.c_uint64 * 18)(*[sum((1 << c) << (4 * j) for j, c in enumerate(codes[16 * i:16 * i + 16])) for i in range(14)])
        for ri in range(192):
            H.r32_2bit(w2, ri, r2)
            H.r32_4bit(w4, ri, r4)
            assert (r2[0], r2[1]) == (r4[0], r4[1]), ri


def test_nib16_to_2bit(H):
    """Codes of A/C/G/T nibbles, and the escape mask: 01 at every nibble that is not exactly one of the four."""
    rng = random.Random(6)
    code, bad = C.c_uint32(), C.c_uint32()
    for _ in range(3000):
        nib = [rng.choice([1, 2, 4, 8]) if rng.random() < 0.8 else rng.randrange(16) for _ in range(16)]
        H.nib16_to_2bit(C.c_uint64(sum(n << (4 * j) for j, n in enumerate(nib))), C.byref(code), C.byref(bad))
        onehot = [n in (1, 2, 4, 8) for n in nib]
        assert bad.value == sum(0 if o else 1 << (2 * j) for j, o in enumerate(onehot))
        for j, n in enumerate(nib):
            if onehot[j]:
                assert (code.value >> (2 * j)) & 3 == n.bit_length() - 1
