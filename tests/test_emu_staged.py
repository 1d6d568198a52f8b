"""The staged general walk of k_tile on the CPU emulator (tests/emu): the cases of tests/stagedgen.py against the oracle - FASTA,
statistics, the whole --debug TSV and the --changes report, byte for byte - each run in a child process under the strict model of
the chunk ring (tests/test_emu_ring.py).  Each case checks from the emulator's layout readouts that it reached its shapes, and from
its count of reads the chunk loop left to the queue that only what is not staged went there: none of the generator's 150-base
reads, some of the 193-base ones, every 8-bit one.  CPU only."""
import os
import pickle
import subprocess
import sys

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import emu_lib, stagedgen as sg
from tests.test_emu_changes import changed_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {"S": lambda: sg.staged(31), "B": lambda: sg.staged(32, eight_bit=True, scale=0.3), "Q": lambda: sg.queue_long(33)}
FAST = "plain"                                            # the only kind the fast walk takes (when its tail is short)


def queued_counter():
    """The emulator's count of reads the chunk loop handed to the queue (polish_dev.cuh `emu_n_queued`, a global of the library)."""
    return emu_lib.C.c_ulonglong.in_dll(emu_lib.lib(), "emu_n_queued")


def child(case_dir, mode, grid):
    """In the child process: one emulated run of the case in case_dir (or of the generator's data when case_dir names no case),
    its result pickled next to it."""
    if os.path.exists(os.path.join(case_dir, "asm.fasta")):
        f = pp.load_fasta(os.path.join(case_dir, "asm.fasta"))
        p = pp.pack_sams(f, [os.path.join(case_dir, "reads_1.sam")])
    else:
        syn = api.Synth(seed=2, n_contigs=1, contig_len=200_000, depth=100)
        f = syn.fasta()
        p = syn.pack(f)
    if mode == "plain":
        queued = queued_counter()
        queued.value = 0
        r = emu_lib.polish(f, p, grid_tiles=grid)
        r["n_queued"] = queued.value
        r["layout"] = {k: v.tolist() for k, v in emu_lib.last_layout().items()}
    else:
        r = emu_lib.polish(f, p, grid_tiles=grid, changes=True, debug=True)
    r["seq_bits"] = p.view.seq_bits
    if "sequences" in r:
        r["fasta"] = emu_lib.fasta_bytes(f, r.pop("sequences"))
    with open(os.path.join(case_dir, "%s%d.pkl" % (mode, grid)), "wb") as out:
        pickle.dump(r, out)


def run_child(case_dir, mode, grid):
    env = dict(os.environ, PYTHONPATH=ROOT)
    code = "from tests.test_emu_staged import child; child(%r, %r, %d)" % (str(case_dir), mode, grid)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        lines = [x for x in r.stderr.splitlines() if x.startswith("ring model:")]
        pytest.fail(lines[0] if lines else "emulator exited with %d:\n%s" % (r.returncode, r.stderr[-3000:]))
    with open(os.path.join(case_dir, "%s%d.pkl" % (mode, grid)), "rb") as f:
        return pickle.load(f)


def tile_slots(case, lay, max_ext):
    """Per tile (contig order): the kinds of its slots [lo, hi) in slot order."""
    kinds = case.facts["kinds"]
    bs, sval = lay["bin_start"], lay["sval"]
    n_bins = len(bs) - 2
    lb = (max_ext + sg.BIN - 1) // sg.BIN
    return [[kinds[a] for a in sval[bs[max(0, 8 * t - lb)]:bs[min(8 * t + 8, n_bins)]]] for t in range(case.facts["n_tiles"])]


def check_shapes(name, case, r):
    assert r["n_long"] == 0
    tiles = tile_slots(case, r["layout"], r["max_ext"])
    n_len193 = sum(ks.count("len193") for ks in tiles)
    if name == "S":
        assert r["seq_bits"] == 4
        seen = set().union(*map(set, tiles))
        want = {"boundary", "order", "xeq", "ins_len", "ins_locus", "del_border", "lookback", "tail_plain", "tail_di", "tail_di2",
                "tail_d2i", "tail_I", "tail_D", "multi2", "multi3", "len192", "len193"}
        assert want <= seen, want - seen
        cig = case.facts["cigars"]
        assert any("DI" in "".join(c for c in x if c.isalpha()) for x in cig) and any("ID" in "".join(c for c in x if c.isalpha()) for x in cig)
        assert any("X" in x and "=" in x for x in cig)
        # staged reads that are not plain: several in one chunk, in lane 31, and many in one warp's chunks of one tile
        staged = lambda k: k not in (FAST, "len193")
        lane31 = sum(1 for ks in tiles for o in range(31, len(ks), 32) if staged(ks[o]))
        dense = max(sum(map(staged, ks[o:o + 32])) for ks in tiles for o in range(0, len(ks), 32))
        per_warp = max(sum(sum(map(staged, ks[o:o + 32])) for o in range(32 * w, len(ks), 32 * 16)) for ks in tiles for w in range(16))
        assert lane31 >= 3 and dense >= 8 and per_warp >= 20, (lane31, dense, per_warp)
        # the reads of the look-back start in the bin before tile 4
        starts = [s for s, k in zip(case.facts["starts"], case.facts["kinds"]) if k == "lookback"]
        assert all(4 * sg.TILE - sg.BIN <= s < 4 * sg.TILE for s in starts) and tiles[4].count("lookback") == len(starts)
        # the 193-base reads, and nothing else, went to the queue
        assert r["n_queued"] == n_len193 > 0
    elif name == "B":
        assert r["seq_bits"] == 8
        assert r["n_queued"] == sum(len(ks) for ks in tiles) > 0        # (every read: the 8-bit pool has no staged copies)
    else:
        assert r["seq_bits"] == 4
        assert tiles[1].count("long2") == case.facts["n_long"] > sg.QCAP
        assert r["n_queued"] == sum(ks.count("long2") for ks in tiles)


@pytest.fixture(scope="module")
def cases(tmp_path_factory, oracle):
    out = {}
    for name, make in CASES.items():
        d = tmp_path_factory.mktemp("staged" + name)
        case = make()
        fa, sams = case.write(d)
        out[name] = (d, case, oracle.polish(fa, sams, debug=True))
    return out


@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("mode", ["plain", "report"])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_staged(cases, name, mode, grid):
    d, case, exp = cases[name]
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


def test_emu_synth_queue_empty(tmp_path):
    """The generator's data (150-base reads, 200 kbp x 100x): the chunk loop walks every read itself, the queue stays empty."""
    r = run_child(tmp_path, "plain", 3)
    assert "error" not in r, r
    assert r["seq_bits"] == 4 and r["n_long"] == 0 and r["n_aln_used"] > 100_000
    assert r["n_queued"] == 0
