"""Contig ends on the CPU emulator (tests/emu): the cases of tests/endgen.py against the oracle, each run in a child process under the
strict model of the chunk ring (tests/test_emu_staged.py).  Legal cases (E, its 8-bit twin, P) compare FASTA, statistics, the whole
--debug TSV and the --changes report byte for byte; error cases compare the error: the reference's message where it quits, and where
it panics on an overrun, ERR_OOB on the first alignment in SAM order of the read the panic names.  CPU only."""
import re

import pytest

from tests import emu_lib, endgen as eg
from tests.oracle_lib import OracleError
from tests.test_emu_changes import changed_rows
from tests.test_emu_staged import run_child, tile_slots

LEGAL = {"E": lambda: eg.edges(41), "E8": lambda: eg.edges(41, eight_bit=True), "P": lambda: eg.past_end(42)}
ERRORS = eg.error_cases(43)
PANIC = re.compile(r"panic: alignment of read (\S+) extends past the end of (\S+)$")


def check_edges(case):
    """What E was built to reach: the contig starts' residues, the tiny contigs, and a read of every kind whose last kept entry is
    its contig's last base."""
    f = case.facts
    starts = f["cstarts"]
    assert {s % 32 for s in starts} == set(range(32))
    for t in range(1, f["n_tiles"]):
        assert {eg.TILE * t - 1, eg.TILE * t, eg.TILE * t + 1} <= set(starts)
    assert {256 * 3 - 1, 256 * 3, 256 * 3 + 1, 256 * 11 - 1, 256 * 11, 256 * 11 + 1} <= set(starts)
    assert {1, 2, 7, 8, 9} <= set(f["lens"])
    assert any(sum(1 for s in starts if s // 8 == x // 8) >= 3 for x in starts)          # one k_compact thread's VT_ITEMS
    assert any(sum(1 for s in starts if s // 128 == x // 128) >= 5 for x in starts)      # one warp's vote positions
    at_end, past = set(), set()
    for kind, c, s, kept in zip(f["kinds"], f["contigs"], f["starts"], f["kept"]):
        if kept:
            assert s + kept <= f["lens"][c], (kind, c, s, kept)
            if s + kept == f["lens"][c]:
                at_end.add(kind)
    assert set(eg.KINDS) | {"insend", "delend", "tiny"} <= at_end, set(eg.KINDS) - at_end
    assert {"first", "firstins", "firstdel"} <= {k for k, s in zip(f["kinds"], f["starts"]) if s == 0}
    covered = set(f["contigs"])
    assert f["uncovered"] and not covered & set(f["uncovered"])


def check_past(case, oracle, fa, sams, exp, d):
    """P: every record past the end is good, and each probe vote is sharp: the FASTA changes when that P record is deleted (its partner
    then carries the read's SEQ)."""
    f = case.facts
    past = [i for i, k in enumerate(f["kinds"]) if k == "past"]
    assert all(f["starts"][i] >= f["lens"][f["contigs"][i]] for i in past) and len(past) >= 48
    assert any(f["contigs"][i] == f["c_last"] for i in past) and any(f["contigs"][i] == f["c_mid"] for i in past)
    assert exp["used_total"] == len(f["lines"])                  # every record is a good alignment
    text = sams[0].read_text().split("\n")
    n_sharp = 0
    for p in f["probes"]:
        if p["probe"] is None:
            continue
        drop = [i for i in past if f["lines"][i].split("\t")[0] == p["qname"]]
        assert len(drop) == 1
        s2 = d / "drop.sam"
        rows = []
        for j, x in enumerate(text):
            f9 = x.split("\t")
            if j != drop[0] and f9[0] == p["qname"] and f9[9] == "*":
                f9[9] = p["partner_seq"]
            if j != drop[0]:
                rows.append("\t".join(f9))
        s2.write_text("\n".join(rows))
        assert oracle.polish(fa, [s2])["fasta"] != exp["fasta"], p
        n_sharp += 1
    assert n_sharp == 32


@pytest.fixture(scope="module")
def legal(tmp_path_factory, oracle):
    out = {}
    for name, make in LEGAL.items():
        d = tmp_path_factory.mktemp("ends" + name)
        case = make()
        fa, sams = case.write(d)
        out[name] = (d, case, fa, sams, oracle.polish(fa, sams, debug=True))
    return out


def test_end_facts(legal, oracle, tmp_path):
    for name in ("E", "E8"):
        check_edges(legal[name][1])
    d, case, fa, sams, exp = legal["P"]
    check_past(case, oracle, fa, sams, exp, tmp_path)
    for name in LEGAL:
        assert sum(legal[name][4]["changed"]) > 0 and 0 in legal[name][4]["changed"] and any(legal[name][4]["zero_depth"])


@pytest.mark.parametrize("grid", [1, 3])
@pytest.mark.parametrize("mode", ["plain", "report"])
@pytest.mark.parametrize("name", list(LEGAL))
def test_emu_ends(legal, name, mode, grid):
    d, case, fa, sams, exp = legal[name]
    r = run_child(d, mode, grid)
    assert "error" not in r, r
    assert r["fasta"] == exp["fasta"]
    assert r["changed"] == exp["changed"] and r["zero_depth"] == exp["zero_depth"] and r["n_aln_used"] == exp["used_total"]
    for got, want in zip(r["total_depth"], exp["total_depth"]):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want))
    if mode == "plain":
        assert r["seq_bits"] == case.facts["seq_bits"]
        tiles = tile_slots(case, r["layout"], r["max_ext"])
        if case.facts["seq_bits"] == 8:
            assert r["n_queued"] == sum(len(ks) for ks in tiles) > 0
        else:
            n_q = sum(ks.count("queued") for ks in tiles)
            assert r["n_queued"] == n_q and (name == "P" or n_q > 5)
        if name != "P":
            assert r["n_long"] > 0
    else:
        assert r["debug_tsv"] == exp["debug_tsv"]
        assert r["changes"] == changed_rows(exp["debug_tsv"]) and r["changes"].count(b"\n") - 1 == sum(exp["changed"])


def library_message(case, code, aln):
    """The library's message for a device error on alignment `aln` (host_api.cpp job_error)."""
    f = case.facts["lines"][aln].split("\t")
    if code == "query name in SAM but not in assembly":
        return "query name %s in SAM but not in assembly" % f[2]
    if code == "CIGAR string does not match read sequence":
        return "CIGAR string for read %s does not match read sequence" % f[0]
    if code == "unexpected character":
        return ('unexpected character (other than M, =, X, I or D) in CIGAR string for read %s: "%s" - did you use BWA MEM to generate '
                'your alignments?' % (f[0], f[5]))
    return "%s (read %s)" % (code, f[0])


def expected_error(case, oracle, d):
    """(oracle message, kind) for an error case, after checking it raises what it was built to raise."""
    fa, sams = case.write(d)
    with pytest.raises(OracleError) as e:
        oracle.polish(fa, sams)
    msg = e.value.msg
    kind, qname = case.facts["expect"]
    m = PANIC.match(msg)
    if kind == "oob":
        assert m and m.group(1) == qname, msg
    else:
        assert not m and qname in msg, msg
    return msg, m


def first_oob(case, qname):
    """The first alignment in SAM order of read `qname` whose last kept entry lies past its contig's end."""
    f = case.facts
    for i, line in enumerate(f["lines"]):
        if line.split("\t")[0] == qname and f["kept"][i] and f["starts"][i] + f["kept"][i] > f["lens"][f["contigs"][i]]:
            return i
    raise AssertionError(qname)


@pytest.mark.parametrize("name", list(ERRORS))
def test_emu_end_errors(oracle, tmp_path, name):
    case = ERRORS[name]
    msg, m = expected_error(case, oracle, tmp_path)
    r = run_child(tmp_path, "plain", 2)
    assert "error" in r, r
    if m:
        assert r["error"] == emu_lib.ERR_TEXT[4]
        assert case.facts["lines"][r["error_aln"]].split("\t")[0] == m.group(1)
        assert r["error_aln"] == first_oob(case, m.group(1))
    else:
        assert library_message(case, r["error"], r["error_aln"]) == msg
    if name == "oob_queued8":
        assert r["seq_bits"] == 8
