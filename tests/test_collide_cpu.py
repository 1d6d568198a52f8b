"""Strings with one 64-bit key (tests/collidegen.py) through the device path's logic on the CPU.

The pairs are checked against the product's own code: tok::fnv1a of the contig table and the quick parse's QNAME / RNAME keys
(tests/tok_harness.cpp), make_sig over the 4-bit pool, the 2-bit staged copy and the 8-bit pool (polish_dev.cuh under
tests/emu/cuda_emu.h).  Then the tokeniser's contig lookup against the host packer with both colliding contig names in the assembly
(both FASTA orders) and with one of them missing, and the other-allele chain of k_tile on the emulator against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import collidegen as cg
from tests import emu_lib
from tests.test_emu_changes import changed_rows
from tests.test_emu_staged import run_child
from tests.test_tok_cpu import H, PP_OK, assert_same, ftok_cpu, host_pack, tok_cpu  # noqa: F401  (H is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PP_CONTIG_UNKNOWN = 0xFFFFFFFF


def regen(key):
    return "the pair no longer collides: regenerate it with `gcc -O3 -pthread -o fnv_collide tests/manual/fnv_collide.c && ./%s`" % cg.REGEN[key]


def fnv(H, s):
    H.fnv1a_cpu.restype = C.c_uint64
    b = s.encode()
    return H.fnv1a_cpu(C.c_char_p(b), C.c_uint64(len(b)))


def quick_keys(H, qnames, rnames):
    """(QNAME key, RNAME key) of one quick-parsed record per pair."""
    text = "".join(cg.sam(q, 0, r, 0, "4M", "ACGT") + "\n" for q, r in zip(qnames, rnames)).encode()
    out = ftok_cpu(H, text, ref_hash=True)
    assert list(out[0]) == [1] * len(qnames)
    return [(int(a), int(b)) for a, b in zip(out[7], out[8])]


def test_name_pairs_collide_in_the_product_hashes(H):
    sets = {"name": [cg.NAME_A, cg.NAME_B], "joux": cg.JOUX}
    for key, names in sets.items():
        assert len(set(names)) == len(names)
        for suffix in ("", "/1", "_x"):
            ks = {fnv(H, n + suffix) for n in names}
            assert len(ks) == 1, regen(key)
            assert ks == {cg.fnv1a(names[0] + suffix)}
            qk = quick_keys(H, [n + suffix for n in names], [n + suffix for n in names])
            assert len({q for q, _ in qk}) == 1 and len({r for _, r in qk}) == 1, regen(key)
            assert qk[0][0] == qk[0][1] == fnv(H, names[0] + suffix)
    assert cg.CLAW_Q != cg.CLAW_R
    (q, _), (_, r) = quick_keys(H, [cg.CLAW_Q, "x"], ["c1", cg.CLAW_R])
    assert q == r ^ cg.REF_DOMAIN, regen("claw")


SIG_HARNESS = r"""
#include "cuda_emu.h"
#include "../../polypolish_b200/csrc/polish_dev.cuh"
// make_sig over alignment 0 of a one-alignment pool (reverse complement on the fly when rc) and over a 2-bit staged copy.
extern "C" unsigned long long sig_pool(int bits, const uint8_t* pool, uint32_t len, int rc, uint32_t start, uint32_t n) {
    for (int i = 0; i < 256; ++i) c_comp[i] = 'N';
    c_comp['A'] = 'T'; c_comp['T'] = 'A'; c_comp['C'] = 'G'; c_comp['G'] = 'C';
    DevData d{};
    const uint32_t off = 0;
    const uint16_t l = (uint16_t)len;
    const uint8_t fl = rc ? PP_FLAG_RC : 0;
    d.seq_pool = pool; d.seq_off = &off; d.seq_len = &l; d.flags = &fl;
    return bits == 4 ? make_sig<4>(PoolBases<4>(d, 0ull), start, n) : make_sig<8>(PoolBases<8>(d, 0ull), start, n);
}
extern "C" unsigned long long sig_staged(const uint32_t* w, uint32_t start, uint32_t n) { return make_sig<4>(StagedBases{w}, start, n); }
"""


@pytest.fixture(scope="module")
def S(tmp_path_factory):
    d = tmp_path_factory.mktemp("sig_harness")
    src, out = d / "sig.cpp", d / "sig.so"
    src.write_text(SIG_HARNESS)
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-shared", "-fPIC", "-pthread", "-w", "-I", os.path.join(ROOT, "tests", "emu"), "-o", str(out),
                           str(src)])
    lib = C.CDLL(str(out))
    lib.sig_pool.restype = lib.sig_staged.restype = C.c_ulonglong
    return lib


NIB = {"A": 1, "C": 2, "G": 4, "T": 8}


def pool4(s):
    b = bytearray((len(s) + 31) // 32 * 16 + 16)
    for i, c in enumerate(s):
        b[i >> 1] |= NIB[c] << (4 * (i & 1))
    return bytes(b)


def staged2(s):
    w = [0] * ((len(s) + 15) // 16 + 2)
    for i, c in enumerate(s):
        w[i >> 4] |= "ACGT".index(c) << (2 * (i & 15))
    return (C.c_uint32 * len(w))(*w)


def product_sigs(S, allele, bits, flank=("GATTACA", "CCTG")):
    """make_sig of the allele inside a read (flank before and after), forward and reverse-complemented in the pool, and staged."""
    read = flank[0] + allele + flank[1]
    start, n = len(flank[0]), len(allele)
    if bits == 4:
        fw = S.sig_pool(4, pool4(read), len(read), 0, start, n)
        rv = S.sig_pool(4, pool4(cg.rc(read)), len(read), 1, start, n)
        st = S.sig_staged(staged2(read), start, n)
        return {fw, rv, st}
    pad = lambda s: s.encode() + bytes(64 - len(s) % 32)
    return {S.sig_pool(8, pad(read), len(read), 0, start, n), S.sig_pool(8, pad(cg.rc(read)), len(read), 1, start, n)}


@pytest.mark.parametrize("key,pair,bits", [("sig4", cg.SIG4, 4), ("sig8", cg.SIG8, 8), ("sig8_len", cg.SIG8_LEN, 8)])
def test_allele_pairs_collide_in_make_sig(S, key, pair, bits):
    a, b = pair
    assert a != b and a[0] == b[0] == "A"
    assert (len(a) != len(b)) == (key == "sig8_len")
    sa, sb = product_sigs(S, a, bits), product_sigs(S, b, bits)
    assert len(sa) == 1 and sa == {cg.sig(a, bits)}
    assert sa == sb, regen(key)
    assert next(iter(sa)) & (15 if bits == 4 else 255) == 0      # a hashed signature: equality falls back to allele_equal


# ---- the tokeniser's contig lookup ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["ab", "ba"])
def test_tok_colliding_contig_names(H, tmp_path, order):
    """Both names in the table: each read's contig is the one its RNAME spells, in both FASTA orders (whichever name comes first,
    the other one's reads meet its slot first and must go on)."""
    case = cg.contig_case(order)
    text = case.sam_texts[0].encode()
    f, p = host_pack(tmp_path, case.fasta_text, [text])
    host = p.arrays()
    rc, dev, _ = tok_cpu(H, f.names, [text])
    assert rc == PP_OK
    assert_same(dev, host)
    idx = {n: i for i, n in enumerate(f.names)}
    rnames = [ln.split("\t")[2] for ln in case.sam_texts[0].splitlines()]
    assert list(dev["contig"]) == [idx[r] for r in rnames]
    assert len(set(rnames)) == 2


def test_tok_colliding_contig_missing(H, tmp_path):
    """The assembly holds NAME_A only: the reads naming NAME_B are on no contig (not on NAME_A, whose key they share)."""
    case = cg.contig_case("ab", only="a")
    text = case.sam_texts[0].encode()
    f, p = host_pack(tmp_path, case.fasta_text, [text])
    rc, dev, _ = tok_cpu(H, f.names, [text])
    assert rc == PP_OK
    assert_same(dev, p.arrays())
    want = [0 if ln.split("\t")[2] == cg.NAME_A else PP_CONTIG_UNKNOWN for ln in case.sam_texts[0].splitlines()]
    assert list(dev["contig"]) == want and PP_CONTIG_UNKNOWN in want


# ---- the other-allele chain on the emulator ---------------------------------------------------------------------------------
# (counts, reads with a secondary): statuses at P separate -> merged  too_close -> changed, multiple -> changed, changed -> changed
VOTES = {"too_close": ((7, 5), (0,)), "multiple": ((6, 6), (0, 1)), "changed": ((13, 2), (0, 1))}
ALLELES = [("sig4", v, 4) for v in VOTES] + [("sig8", "too_close", 8), ("sig8_len", "too_close", 8), ("sig8_len", "changed", 8)]
PAIR = {"sig4": cg.SIG4, "sig8": cg.SIG8, "sig8_len": cg.SIG8_LEN}


def allele_case(key, vote, bits, twin=False):
    counts, multi = VOTES[vote]
    return cg.allele_case(counts, PAIR[key], bits, twin=twin, multi=multi)


def check_sharp(oracle, tmp_path, key, vote, bits):
    """The oracle's answers for the case and its twin (the two alleles one string): the status at P as designed, and they differ."""
    out = {}
    for twin in (False, True):
        d = tmp_path / ("twin" if twin else "case")
        d.mkdir()
        fa, sams = allele_case(key, vote, bits, twin).write(d)
        out[twin] = oracle.polish(fa, sams, debug=True)
    st = cg.row(out[False]["debug_tsv"], cg.P)[7].decode(), cg.row(out[True]["debug_tsv"], cg.P)[7].decode()
    assert st == (vote, "changed"), st
    assert cg.row(out[False]["debug_tsv"], cg.P) != cg.row(out[True]["debug_tsv"], cg.P)
    return out[False]


@pytest.mark.parametrize("key,vote,bits", ALLELES)
def test_emu_colliding_alleles(oracle, tmp_path, key, vote, bits):
    exp = check_sharp(oracle, tmp_path, key, vote, bits)
    d = tmp_path / "emu"
    d.mkdir()
    allele_case(key, vote, bits).write(d)
    r = run_child(d, "report", 2)
    assert "error" not in r, r
    assert r["seq_bits"] == bits
    assert r["fasta"] == exp["fasta"]
    assert r["debug_tsv"] == exp["debug_tsv"]
    assert r["changes"] == changed_rows(exp["debug_tsv"])
