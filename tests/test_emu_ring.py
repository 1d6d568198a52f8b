"""k_tile's chunk ring on the CPU emulator (tests/emu), under its strict model of bulk copies and mbarriers: the cases of
tests/ringgen.py against the oracle - FASTA, statistics, the whole --debug TSV and the --changes report, byte for byte - with 1 and 3
CTAs.  Each run is a child process, because a protocol error ends the emulator with a "ring model:" line; the test fails with it.
Before it trusts a pass, each case checks from the emulator's layout readouts (bin_start, the alignment in each slot, the tile order)
that it reached its shapes.  The model's own checks are driven one error at a time by tests/emu/ring_selftest.cpp.  CPU only."""
import os
import pickle
import subprocess
import sys

import pytest

import polypolish_b200 as pp
from tests import emu_lib, ringgen as rg
from tests.test_emu_changes import changed_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"A": lambda: rg.chunk_shapes(11), "B": lambda: rg.chunk_shapes(12, eight_bit=True), "C": lambda: rg.queue_overflow(13)}


def child(case_dir, mode, grid):
    """In the child process: one emulated run of the case in case_dir, its result pickled next to it."""
    fa, sams = os.path.join(case_dir, "asm.fasta"), [os.path.join(case_dir, "reads_1.sam")]
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    if mode == "plain":
        r = emu_lib.polish(f, p, grid_tiles=grid)
        r["layout"] = {k: v.tolist() for k, v in emu_lib.last_layout().items()}
    else:
        r = emu_lib.polish(f, p, grid_tiles=grid, changes=True, debug=True)
    r["seq_bits"] = p.view.seq_bits
    if "sequences" in r:                                    # (else an input error: the parent reports it)
        r["fasta"] = emu_lib.fasta_bytes(f, r.pop("sequences"))
    with open(os.path.join(case_dir, "%s%d.pkl" % (mode, grid)), "wb") as out:
        pickle.dump(r, out)


def run_child(case_dir, mode, grid):
    env = dict(os.environ, PYTHONPATH=ROOT)
    code = "from tests.test_emu_ring import child; child(%r, %r, %d)" % (str(case_dir), mode, grid)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        lines = [x for x in r.stderr.splitlines() if x.startswith("ring model:")]
        pytest.fail(lines[0] if lines else "emulator exited with %d:\n%s" % (r.returncode, r.stderr[-3000:]))
    with open(os.path.join(case_dir, "%s%d.pkl" % (mode, grid)), "rb") as f:
        return pickle.load(f)


def shapes(case, lay, max_ext):
    """What the layout of the last run gives k_tile's chunk loop: per tile (contig order) its slot count and each warp's chunks, and
    the shapes reached."""
    kinds = case.facts["kinds"]
    bs, sval, order = lay["bin_start"], lay["sval"], lay["tile_order"]
    n_bins = len(bs) - 2
    lb = (max_ext + rg.BIN - 1) // rg.BIN
    ranges = [(bs[max(0, 8 * t - lb)], bs[min(8 * t + 8, n_bins)]) for t in range(len(order))]
    n = [hi - lo for lo, hi in ranges]
    chunks = [rg.warp_chunks(x) for x in n]
    s = dict(lb=lb, n=n, ranges=ranges, kinds_in_tiles=set(), lane31_192=0, max_chunks=max(max(c) for c in chunks))
    for lo, hi in ranges:
        for o in range(hi - lo):
            k = kinds[sval[lo + o]]
            s["kinds_in_tiles"].add(k)
            if o % 32 == 31 and k == "len192":
                s["lane31_192"] += 1
    s["counts"] = {"empty": n.count(0), "partial": sum(1 <= x <= 31 for x in n), "mod0": sum(x > 0 and x % 32 == 0 for x in n),
                   "mod1": sum(x % 32 == 1 for x in n), "mod31": sum(x % 32 == 31 for x in n)}
    s["warp_chunks"] = {m: sum(c.count(m) for c in chunks) for m in range(1, 5)}
    # the parity word of every warp in the order the tiles are dealt (on the CPU, block 0 takes them all): tiles that start with
    # a stage's parity bit set, and neighbours with odd and even chunk counts
    par = [0] * rg.WARPS
    s["carry"] = {0: 0, 1: 0}
    s["odd_even"] = set()
    prev = None
    for t in order:
        for w, m in enumerate(chunks[t]):
            for st in (0, 1):
                if m > st and (par[w] >> st) & 1:
                    s["carry"][st] += 1
            if prev is not None and m and chunks[prev][w]:
                s["odd_even"].add((chunks[prev][w] % 2, m % 2))
            par[w] ^= ((m + 1) // 2 % 2) | ((m // 2 % 2) << 1)
        prev = t
    return s


def check_shapes(name, case, r):
    s = shapes(case, r["layout"], r["max_ext"])
    assert s["lb"] == 1 and r["max_ext"] <= rg.BIN
    if name in ("A", "B"):
        assert s["n"] == case.facts["schedule"]
        assert all(v > 0 for v in s["counts"].values()), s["counts"]
        assert all(s["warp_chunks"][m] > 0 for m in (1, 2, 3, 4)), s["warp_chunks"]
        assert s["carry"][0] > 0 and s["carry"][1] > 0 and {(0, 1), (1, 0)} <= s["odd_even"], (s["carry"], s["odd_even"])
        assert s["lane31_192"] >= 5
        assert {"short", "len8_15", "tail7", "tail8", "indel", "cross", "multi2", "multi3", "multi3_indel", "zp", "len192"} <= s["kinds_in_tiles"]
        assert r["seq_bits"] == (8 if name == "B" else 4) and r["n_long"] == 0
    else:
        kinds = case.facts["kinds"]
        lo, hi = s["ranges"][1]
        n_indel = sum(kinds[a] == "indel" for a in r["layout"]["sval"][lo:hi])
        assert n_indel >= 1100 > rg.QCAP and r["n_long"] == kinds.count("long_indel") == 4
    return s


@pytest.fixture(scope="module")
def cases(tmp_path_factory, oracle):
    out = {}
    for name, make in CASES.items():
        d = tmp_path_factory.mktemp("ring" + name)
        case = make()
        fa, sams = case.write(d)
        out[name] = (d, case, fa, sams, oracle.polish(fa, sams, debug=True))
    return out


@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("mode", ["plain", "report"])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_ring(cases, name, mode, grid):
    d, case, fa, sams, exp = cases[name]
    r = run_child(d, mode, grid)
    assert "error" not in r, r
    assert r["fasta"] == exp["fasta"]
    assert r["changed"] == exp["changed"] and r["zero_depth"] == exp["zero_depth"] and r["n_aln_used"] == exp["used_total"]
    for got, want in zip(r["total_depth"], exp["total_depth"]):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want))
    if mode == "plain":
        check_shapes(name, case, r)
    else:
        assert r["debug_tsv"] == exp["debug_tsv"]
        assert r["changes"] == changed_rows(exp["debug_tsv"]) and r["changes"].count(b"\n") - 1 == sum(exp["changed"])
    assert sum(exp["changed"]) > 0


# ---- the model itself -----------------------------------------------------------------------------------------------------------
SELFTEST = os.path.join(ROOT, "build", "ring_selftest")


@pytest.fixture(scope="module")
def selftest():
    src = os.path.join(ROOT, "tests", "emu", "ring_selftest.cpp")
    deps = [src] + emu_lib.DEPS[1:]
    if not os.path.exists(SELFTEST) or any(os.path.getmtime(x) > os.path.getmtime(SELFTEST) for x in deps):
        os.makedirs(os.path.dirname(SELFTEST), exist_ok=True)
        tmp = "%s.%d.tmp" % (SELFTEST, os.getpid())
        subprocess.check_call(["g++", "-std=c++20", "-O1", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                               "-Wno-unused-variable", "-ffp-contract=off", "-I", os.path.join(ROOT, "tests", "emu"), src, "-o", tmp])
        os.replace(tmp, SELFTEST)
    return SELFTEST


@pytest.mark.parametrize("err, line", [
    ("no_flip", "a parity that was not flipped"),
    ("extra_tx", "would hang: lane"),
    ("second_arrival", "second arrival (expect_tx 64) in an unfinished phase"),
    ("early_refill", "a refill of a stage the warp may still be reading"),
    ("misaligned", "not 16-byte aligned"),
    ("in_flight_exit", "the block exits with barrier"),
    ("no_prologue_issue", "would hang: lane"),
])
def test_ring_model_catches(selftest, err, line):
    r = subprocess.run([selftest, err], capture_output=True, text=True, env=dict(os.environ, EMU_RING_HANG_MS="300"), timeout=120)
    got = [x for x in r.stderr.splitlines() if x.startswith("ring model:")]
    assert r.returncode == 86 and len(got) == 1 and line in got[0], r.stderr


def test_ring_model_passes_the_protocol(selftest):
    r = subprocess.run([selftest, "none"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout == "ok\n" and not r.stderr, r.stderr
