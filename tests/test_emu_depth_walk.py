"""The ordered depth walk's merge on the CPU emulator (tests/emu) against the oracle: probe positions on a vote boundary whose
covering reads are spread over the runs the walk merges - bins b-1 and b (depth_walk_two), b-2, b-1 and b, and the long list
(depth_walk_steps) - with k > 32 in the step merge and the printed depth of --changes through each walker.  The cases come from
tests/walkgen.py; each first asserts what it reaches: the runs it fills, how many bins a tile looks back, the long list, and that a
merge emptying one run first would land on the other side of the boundary."""
import math

import pytest

import polypolish_b200 as pp
from tests import walkgen as wg
from tests.test_emu_changes import check_changes
from tests.test_emu_polish import check


def check_facts(case, spec, on):
    f = case.facts
    if on:
        assert f["sum"] == spec["target"]
        if len(spec["labels"]) > 1:                              # a run-first merge flips the outcome
            assert all((c - spec["target"]) * spec["side"] > 0 for c in f["concat"]), f["concat"]
    else:
        assert f["sum"] == math.nextafter(spec["target"], spec["side"] * math.inf)
    assert all(f["run_counts"][lab] >= spec["per_run"] for lab in spec["labels"]), f["run_counts"]
    lay = spec["layout"]
    if lay == "contig_border":                                   # P among the first positions of `probe`, in a bin `head` ends in
        assert f["head_in_bin"] > 0 and f["head"] % wg.BIN and f["P"] // wg.BIN == f["head"] // wg.BIN and f["probe_local"] < 16
    else:
        assert f["decoys"] > 0
    if lay.startswith("border"):                                 # the first / last position of a tile; reads cross the border
        assert f["P"] % wg.TILE in (0, wg.TILE - 1) and f["sub"] in (0, wg.TILE // wg.SUB - 1)
    assert f["lb"] == (2 if lay in ("three", "border_at", "border_before") else 1) and f["max_ext"] <= wg.LONG_E
    if spec["windowed"]:                                         # several windows per run; both mis-merges of depth_walk_two cross
        m = f["merge"]
        assert min(f["windows"]) >= 3
        assert m["ok"] == f["sum"]
        if on:
            assert all((m[x] - spec["target"]) * spec["side"] > 0 for x in ("max", "batch")), m
    assert f["sub"] == (f["P"] % wg.TILE) // wg.SUB and f["bin"] == f["P"] // wg.BIN
    if lay == "long":
        assert f["n_long"] > f["run_counts"]["long"] and any(k != 1 for k in f["long_k"])
    else:
        assert f["n_long"] == 0


def expected(spec, on):
    """P's vote and printed depth: the on / off orders of a boundary vote differently; of the print pair both change."""
    if spec["side"] < 0:
        return (1 if on else 0), spec["printed"]
    return 1, (spec["printed"] if on else b"3.3")


@pytest.mark.parametrize("name", list(wg.CASES))
def test_emu_depth_walk(oracle, tmp_path, name):
    on_case, off_case, spec = wg.case_pair(name)
    for on, case in ((True, on_case), (False, off_case)):
        check_facts(case, spec, on)
        assert case.facts["n_records"] < 5000
        d = tmp_path / ("on" if on else "off")
        d.mkdir()
        fa, sams = case.write(d)
        f = pp.load_fasta(fa)
        p = pp.pack_sams(f, sams)
        assert p.view.seq_bits == (8 if spec["eight_bit"] else 4)
        p.close()
        want, printed = expected(spec, on)
        exp = oracle.polish(fa, sams, debug=True, **case.opts)
        P, ci = case.facts["P"], (1 if case.facts["head"] else 0)
        local = str(case.facts["probe_local"]).encode()
        row = exp["debug_tsv"].split(b"\n")[1 + P].split(b"\t")
        assert row[:2] == [b"probe", local] and row[3] == printed and exp["changed"][ci] == want
        for g in (1, 3):
            r = check(oracle, fa, sams, grid_tiles=g, **case.opts)
            assert r["changed"][ci] == want
            assert r["max_ext"] == case.facts["max_ext"] and r["n_long"] == case.facts["n_long"]      # what k_bin made of it
            r = check_changes(oracle, fa, sams, grid_tiles=g, **case.opts)
            assert r["changed"][ci] == want
            rows = [x.split(b"\t") for x in r["changes"].split(b"\n")[1:] if x]
            assert [x[3] for x in rows if x[:2] == [b"probe", local]] == ([printed] if want else [])
