"""Second restatement as cross-check: oracle/pyport.py (plain Python, written from the Rust source independently of the C++
oracle) against the golden fixtures and against the C++ oracle on fuzz cases.  Two separate readings of
reference src/*.rs have to agree byte for byte on FASTA, debug TSV, statistics and filtered SAM."""
import importlib.util
import json
import os
import pathlib

import pytest

from tests import fuzzgen

ROOT = pathlib.Path(__file__).resolve().parent.parent
spec = importlib.util.spec_from_file_location("pyport", ROOT / "oracle" / "pyport.py")
pyport = importlib.util.module_from_spec(spec)
spec.loader.exec_module(pyport)

G = ROOT / "tests" / "golden"
POLISH = sorted(p.name for p in G.glob("polish_*"))


@pytest.mark.parametrize("name", POLISH)
def test_pyport_reproduces_golden(name):
    d = G / name
    opts = json.loads((d / "opts.json").read_text())
    sams = sorted(d.glob("reads_*.sam"))
    r = pyport.polish(d / "asm.fasta", sams, debug=True, **opts)
    assert r["fasta"] == (d / "expected.fasta").read_bytes()
    assert r["debug_tsv"] == (d / "expected_debug.tsv").read_bytes()
    st = json.loads((d / "expected_stats.json").read_text())
    assert (r["changed"], r["zero_depth"], r["used_total"]) == (st["changed"], st["zero_depth"], st["used_total"])


def test_pyport_reproduces_golden_filter():
    d = G / "filter_6"
    r = pyport.filter_sams(d / "in_1.sam", d / "in_2.sam")
    assert r["out1"] == (d / "expected_1.sam").read_bytes() and r["out2"] == (d / "expected_2.sam").read_bytes()
    e = json.loads((d / "expected.json").read_text())
    assert (r["low"], r["high"], r["orientation"]) == (e["low"], e["high"], e["orientation"])


@pytest.mark.parametrize("seed", [100, 101, 104, 105, 108, 113, 120, 131, 300, 301, 305])
def test_pyport_agrees_with_cpp_oracle(oracle, tmp_path, seed):
    kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)
    fa, sams = case.write(tmp_path)
    try:
        exp = ("ok", oracle.polish(fa, sams, debug=True, **case.opts))
    except Exception as e:
        exp = ("err", e.msg)
    try:
        got = ("ok", pyport.polish(fa, sams, debug=True, **case.opts))
    except pyport.RefError as e:
        got = ("err", str(e))
    assert exp[0] == got[0], (exp[1] if exp[0] == "err" else "", got[1] if got[0] == "err" else "")
    if exp[0] == "ok":
        assert got[1]["fasta"] == exp[1]["fasta"]
        assert got[1]["debug_tsv"] == exp[1]["debug_tsv"]
        assert (got[1]["changed"], got[1]["zero_depth"], got[1]["used_total"]) == (exp[1]["changed"], exp[1]["zero_depth"], exp[1]["used_total"])


def test_pyport_filter_agrees_with_cpp_oracle(oracle, tmp_path):
    from polypolish_b200 import api
    syn = api.Synth(seed=17, contig_len=20_000, depth=30)
    fa, sams = syn.write(tmp_path)
    exp = oracle.filter(sams[0], sams[1])
    got = pyport.filter_sams(sams[0], sams[1])
    assert got["out1"] == exp["out1"] and got["out2"] == exp["out2"]
    assert (got["low"], got["high"], got["orientation"]) == (exp["low"], exp["high"], exp["orientation"])
    po = pyport.polish(fa, sams)
    assert po["fasta"] == oracle.polish(fa, sams)["fasta"]


def test_pyport_reference_unit_vectors():
    """A few of the reference's own unit-test vectors (misc.rs:280-304, filter.rs:450-462, alignment.rs:386-399)."""
    assert [pyport.bankers_rounding(x) for x in (0.5, 1.5, 2.5, 3.5, 42.55, 0.49, 7.0)] == [0, 2, 2, 4, 43, 0, 7]
    assert pyport.reverse_complement("ACGTNRYX") == "NRYNACGT"
    s = [15, 20, 35, 40, 50]
    assert [pyport.get_percentile(s, p) for p in (5.0, 30.0, 40.0, 50.0, 100.0)] == [15, 20, 20, 35, 50]
    assert pyport.get_expanded_cigar("3M1I2D") == "MMMIDD" and pyport.get_expanded_cigar("*") == ""
    for bad in ("10Q", "10MM1I10M", "100M5"):
        with pytest.raises(ValueError):
            pyport.get_expanded_cigar(bad)
