"""The one-indel fast walk of k_tile on the CPU emulator (tests/emu): the cases of tests/indelgen.py against the oracle - FASTA,
statistics, the whole --debug TSV and the --changes report, byte for byte - each run in a child process under the strict model of
the chunk ring (tests/test_emu_ring.py).  Before it trusts a pass, each case checks from the emulator's layout readouts that it
reached its shapes.  CPU only."""
import pytest

from tests import indelgen as ig
from tests.test_emu_changes import changed_rows
from tests.test_emu_ring import run_child

CASES = {"E": lambda: ig.edges(21), "Q": lambda: ig.queue_general(22)}


def tile_slots(case, lay, max_ext):
    """Per tile (contig order): the kinds of its slots [lo, hi) in slot order."""
    kinds = case.facts["kinds"]
    bs, sval = lay["bin_start"], lay["sval"]
    n_bins = len(bs) - 2
    lb = (max_ext + ig.BIN - 1) // ig.BIN
    return [[kinds[a] for a in sval[bs[max(0, 8 * t - lb)]:bs[min(8 * t + 8, n_bins)]]] for t in range(case.facts["n_tiles"])]


def check_shapes(name, case, r):
    assert r["n_long"] == 0 and r["seq_bits"] == 4
    tiles = tile_slots(case, r["layout"], r["max_ext"])
    if name == "E":
        seen = set().union(*map(set, tiles))
        want = {"boundary", "ins_len", "ins_locus", "del_border", "a_before", "b_past", "multi2", "multi3", "len192"}
        want |= {"tail_c%d_r%d" % (c, t) for c in range(1, 9) for t in (c - 1, c, c + 1) if t >= 1}
        assert want <= seen, want - seen
        one = lambda k: k != "plain"                                             # every other kind is a one-indel read
        lane31 = sum(1 for ks in tiles for o in range(31, len(ks), 32) if ks[o] == "len192")
        dense = max(sum(map(one, ks[o:o + 32])) for ks in tiles for o in range(0, len(ks), 32))
        assert lane31 >= 3 and dense >= 8, (lane31, dense)
        # the look-back: the reads whose segment A ends before tile 4 are among tile 4's slots, and start in the bin before it
        a_before = [s for s, k in zip(case.facts["starts"], case.facts["kinds"]) if k == "a_before"]
        assert all(4 * ig.TILE - ig.BIN <= s < 4 * ig.TILE for s in a_before) and tiles[4].count("a_before") == len(a_before)
    else:
        assert tiles[1].count("indel2") == case.facts["n_two"] > ig.QCAP


@pytest.fixture(scope="module")
def cases(tmp_path_factory, oracle):
    out = {}
    for name, make in CASES.items():
        d = tmp_path_factory.mktemp("indel" + name)
        case = make()
        fa, sams = case.write(d)
        out[name] = (d, case, oracle.polish(fa, sams, debug=True))
    return out


@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("mode", ["plain", "report"])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_indel(cases, name, mode, grid):
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
