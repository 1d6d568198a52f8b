"""The status runs (--status-bed) of the emulated kernels (tests/emu): k_tile's status mode under the strict model of the chunk ring,
then k_status_heads and k_status_runs, against the run-length encoding of the oracle's --debug status column, byte for byte.  CPU
only."""
import pytest

import polypolish_b200 as pp
from tests import emu_lib, endgen, fuzzgen, statusgen


def check_status(oracle, fa, sams, grid_tiles=2, with_changes=False, **opts):
    exp = oracle.polish(fa, sams, debug=True, **opts)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams, careful=opts.get("careful", False))
    r = emu_lib.polish(f, p, grid_tiles=grid_tiles, status=True, changes=with_changes, **opts)
    assert "error" not in r, r
    assert emu_lib.fasta_bytes(f, r["sequences"]) == exp["fasta"]
    assert r["bed"] == statusgen.bed_from_debug_tsv(exp["debug_tsv"])
    assert sum(int(x.split(b"\t")[2]) - int(x.split(b"\t")[1]) for x in r["bed"].splitlines()) == int(f.off[-1])
    return r, exp


def test_bed_from_debug_tsv():
    tsv = (b"name\tpos\tbase\tdepth\tinvalid\tvalid\tcounts\tstatus\tnew\n"
           b"a\t0\tA\t0.0\t0\t5\t\tlow_depth\tA\na\t1\tA\t0.0\t0\t5\t\tlow_depth\tA\na\t2\tC\t9.0\t2\t5\tC:9\tkept\tC\n"
           b"b\t0\tG\t9.0\t2\t5\tG:9\tkept\tG\nb\t1\tG\t9.0\t2\t5\tG:9\tkept\tG\n")
    assert statusgen.bed_from_debug_tsv(tsv) == b"a\t0\t2\tlow_depth\na\t2\t3\tkept\nb\t0\t2\tkept\n"


@pytest.mark.parametrize("seed", [100, 101, 104, 107, 112, 116, 121, 133, 140, 152, 164, 175])
def test_emu_status_fuzz(oracle, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0)
    fa, sams = case.write(tmp_path)
    try:
        oracle.polish(fa, sams, **case.opts)
    except Exception:
        pytest.skip("the reference rejects this input")
    check_status(oracle, fa, sams, with_changes=seed % 2 == 1, **case.opts)


@pytest.mark.parametrize("seed", [300, 303, 307])
def test_emu_status_deep_multimap(oracle, tmp_path, seed):
    """Non-dyadic k everywhere: the thresholds come from the reference's ordered sum, not the fixed-point estimate."""
    case = fuzzgen.make_case(seed, n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False))
    fa, sams = case.write(tmp_path)
    check_status(oracle, fa, sams, **case.opts)


@pytest.mark.parametrize("name", sorted(statusgen.CASES))
def test_emu_status_boundary(oracle, tmp_path, name):
    """P's depth sums exactly to a status boundary in one SAM order and to one ulp below it in the other: the oracle's statuses
    differ, the base does not, and the fixed-point bound's lower end gives the wrong one for the "on" order."""
    on, off, spec = statusgen.case_pair(name)
    assert spec["th_on"] != spec["th_off"] and on.facts["th_lo"] == off.facts["th_lo"] == spec["th_off"]
    assert on.facts["seq_bits"] == (8 if spec["eight_bit"] else 4)
    fastas = []
    for c, want in ((on, spec["st_on"]), (off, spec["st_off"])):
        d = tmp_path / ("on" if c is on else "off")
        d.mkdir()
        fa, sams = c.write(d)
        r, exp = check_status(oracle, fa, sams, grid_tiles=1, **c.opts)
        assert statusgen.status_at(exp["debug_tsv"], "probe", spec["P"]) == want
        fastas.append(exp["fasta"])
    assert fastas[0] == fastas[1]


@pytest.mark.parametrize("name,case", [("E", lambda: endgen.edges(41)), ("E8", lambda: endgen.edges(41, eight_bit=True))])
def test_emu_status_contig_ends(oracle, tmp_path, name, case):
    """Contigs of 1-9 bp, contig starts at every residue mod 32, contigs no read covers: every contig start begins a run."""
    c = case()
    fa, sams = c.write(tmp_path)
    r, _ = check_status(oracle, fa, sams, **c.opts)
    assert r["bed"].count(b"\n") >= len(c.facts["lens"])


GRID = [dict(min_depth=d, **fr) for d in (0, 1, 2, 5)
        for fr in (dict(), dict(fraction_invalid=0.001, fraction_valid=0.5), dict(fraction_invalid=0.01, fraction_valid=0.02))]


@pytest.mark.parametrize("seed", [101, 116])
@pytest.mark.parametrize("opts", GRID, ids=lambda o: "-".join("%s%s" % (k[0] + k[-1], v) for k, v in sorted(o.items())))
def test_emu_status_option_grid(oracle, tmp_path, seed, opts):
    """min_depth 0, 1, 2 and 5; fraction pairs under which the invalid threshold is 0 (an A/C/G/T count of zero is then
    intermediate: too_close)."""
    case = fuzzgen.make_case(seed)
    fa, sams = case.write(tmp_path)
    check_status(oracle, fa, sams, **dict(case.opts, **opts))
