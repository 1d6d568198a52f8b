"""Read selection on the CPU emulator (tests/emu) against the oracle: which records are good, k of every read group, used_total
and the errors only good records raise, for the cases of tests/selectgen.py under every option set of their grid.  The exact model
(limitgen.record_good) is pinned to the oracle first; every case asserts what it was built to reach before it trusts a pass.
Datasets of case E are loaded with --careful and polished with and without it.  CPU only."""
import pytest

import polypolish_b200 as pp
from tests import emu_lib, limitgen as lg, selectgen as sg
from tests.oracle_lib import OracleError

CASES = {"A": lambda: sg.option_grid(11), "B": lambda: sg.block_edges(12), "C": lambda: sg.global_k(13), "D": lambda: sg.errors(14)}
CASES.update({"E-" + v: (lambda v=v: sg.careful_noseq(15, v)) for v in sg.NOSEQ_VARIANTS})


def opt_sets(name):
    return sg.ERR_OPTS if name == "D" else sg.OPTS


def load_careful(name):
    """Case E is loaded with --careful (the packer keeps its groups without SEQ); the others without."""
    return name.startswith("E")


def aligned_rows(texts):
    """The fields of every aligned record (flag 4 clear), in SAM order: row i is alignment i of a packed dataset."""
    return [l.split("\t") for t in texts for l in t.split("\n") if l and not l.startswith("@") and not int(l.split("\t")[1]) & 4]


def reference_message(rows, kind, aln):
    """What the reference prints for error `kind` raised on alignment `aln` (alignment.rs, pileup.rs; the oracle's panic text)."""
    r = rows[aln]
    return {"noseq": "no alignments for read %s contain sequence" % r[0],
            "unknown_contig": "query name %s in SAM but not in assembly" % r[2],
            "seq_mismatch": "CIGAR string for read %s does not match read sequence" % r[0],
            "bad_op": 'unexpected character (other than M, =, X, I or D) in CIGAR string for read %s: "%s" - did you use BWA MEM to '
                      'generate your alignments?' % (r[0], r[5]),
            "oob": "panic: alignment of read %s extends past the end of %s" % (r[0], r[2])}[kind]


def run_oracle(oracle, fa, sams, opts):
    try:
        return oracle.polish(fa, sams, **opts)
    except OracleError as e:
        return dict(error=e.msg)


@pytest.fixture(scope="module")
def cases(tmp_path_factory, oracle):
    """name -> (case, fasta, sams, [(opts, model, oracle result)])."""
    out = {}
    for name, make in CASES.items():
        case = make()
        d = tmp_path_factory.mktemp("select" + name.replace("-", ""))
        fa, sams = case.write(d)
        runs = [(o, lg.record_good(case.sam_texts, contigs=case.contigs, detail=True, **o), run_oracle(oracle, fa, sams, o))
                for o in opt_sets(name)]
        out[name] = (case, fa, sams, runs)
    return out


def check_model(case, runs):
    """The model against the oracle: used_total where the call succeeds, and the error's kind and the record it names."""
    rows = aligned_rows(case.sam_texts)
    for opts, m, exp in runs:
        if m["error"]:
            assert exp.get("error") == reference_message(rows, *m["error"]), (opts, m["error"], exp.get("error"))
        else:
            assert "error" not in exp, (opts, exp["error"])
            assert exp["used_total"] == m["used"], opts


@pytest.mark.parametrize("name", list(CASES))
def test_model_matches_oracle(cases, name):
    case, fa, sams, runs = cases[name]
    check_model(case, runs)


def good_sets(runs):
    return [frozenset(i for i, g in enumerate(m["good"]) if g) for _, m, _ in runs]


def test_select_facts(cases, oracle, tmp_path):
    # A and C: the good set changes between every two neighbouring option sets; k takes every value 0-9; some pair of option sets
    # changes used_total and some pair the FASTA
    for name in ("A", "C"):
        case, fa, sams, runs = cases[name]
        gs = good_sets(runs)
        assert all(a != b for a, b in zip(gs, gs[1:])), name
        assert set(range(10)) <= {k for _, m, _ in runs for k in m["k"]}, name
        assert len({exp["used_total"] for _, _, exp in runs}) > 1 and len({exp["fasta"] for _, _, exp in runs}) > 1, name
        nms = {int(x[5:]) for r in aligned_rows(case.sam_texts) for x in r[11:] if x.startswith("NM:i:")}
        assert set(sg.NMS) <= nms
        # a probe flips at every max_errors of the grid: no two sets without --careful polish alike
        by_me = {o.get("max_errors", 10): exp["fasta"] for o, _, exp in runs if not o.get("careful") and o.get("max_errors") != sg.U32 - 1}
        assert len(set(by_me.values())) == len(by_me) > 5, name
    # C: global-k mode under every option set where a record of the big group is good
    case, fa, sams, runs = cases["C"]
    f = pp.load_fasta(fa)
    rid = pp.pack_sams(f, sams).arrays()["read_id"]
    gk = [lg.expect_global_k(rid, m["good"]) for _, m, _ in runs]
    assert gk == [not o.get("careful") for o, _, _ in runs]
    assert case.facts["big"]["size"] == 9000
    # B: first records -3 .. +3 from a block edge, groups of 257 and 513 records, one across a multiple of 512; k changes with the
    # options; and splitting an edge-crossing group at the edge changes the oracle's total depth or FASTA
    case, fa, sams, runs = cases["B"]
    groups = case.facts["groups"]
    offs = {((g["start"] + 128) % 256) - 128 for g in groups}
    assert set(range(-3, 4)) <= offs
    assert {257, 513} <= {g["size"] for g in groups}
    assert any(g["start"] < e < g["start"] + g["size"] for g in groups for e in range(512, case.facts["n_aln"], 512))
    gs = good_sets(runs)
    assert all(a != b for a, b in zip(gs, gs[1:]))
    base = runs[0][2]
    n_sharp = 0
    for g in groups:
        edge = (g["start"] // 256 + 1) * 256
        if edge >= g["start"] + g["size"]:
            continue
        d = tmp_path / ("split%d" % g["start"])
        d.mkdir()
        s = d / "split.sam"
        s.write_text(sg.split_group(case, g, edge)[0])
        exp = oracle.polish(fa, [s])
        assert exp["fasta"] != base["fasta"] or exp["total_depth"] != base["total_depth"], g
        n_sharp += 1
    assert n_sharp >= 7                        # offsets -3 .. -1, the big groups and the one across 512
    # D: the reference names a different error as the options change, and some calls succeed between them
    case, fa, sams, runs = cases["D"]
    assert [m["error"] and m["error"][0] for _, m, _ in runs] == case.facts["expect"]
    assert len({exp["fasta"] for _, _, exp in runs if "fasta" in exp}) > 1
    # E: the no-SEQ group's error under every set without --careful (or the earlier group's), nothing under --careful
    for v in sg.NOSEQ_VARIANTS:
        case, fa, sams, runs = cases["E-" + v]
        for o, m, _ in runs:
            want = case.facts["expect"] if (not o.get("careful") or v == "after") else None
            assert (m["error"] and m["error"][0]) == want, (v, o)
        zz = [r for r in aligned_rows(case.sam_texts) if r[0] == "zz"]
        assert len(zz) == 2 and all(r[9] == "*" for r in zz)
        assert (min(int(r[11][5:]) for r in zz) > 10) == (v == "none")           # a good record under the defaults, or none
        assert (zz[0][2] not in case.contigs) == (v == "unknown")


def emu_check(f, p, exp, model, opts):
    r = emu_lib.polish(f, p, grid_tiles=2, **opts)
    if model["error"]:
        kind, aln = model["error"]
        assert r.get("error") == emu_lib.ERR_TEXT[lg.ERR_KIND[kind]] and r["error_aln"] == aln, (opts, model["error"], r)
        return r
    assert "error" not in r, (opts, r)
    assert emu_lib.fasta_bytes(f, r["sequences"]) == exp["fasta"], opts
    assert r["changed"] == exp["changed"] and r["zero_depth"] == exp["zero_depth"] and r["n_aln_used"] == exp["used_total"], opts
    for got, want in zip(r["total_depth"], exp["total_depth"]):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), opts
    return r


@pytest.mark.parametrize("name", list(CASES))
def test_emu_select(cases, name):
    case, fa, sams, runs = cases[name]
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams, careful=load_careful(name))
    rid = p.arrays()["read_id"]
    for opts, m, exp in runs:
        r = emu_check(f, p, exp, m, opts)
        if "error" not in r:
            assert r["global_k"] == lg.expect_global_k(rid, m["good"]), opts
