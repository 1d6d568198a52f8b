"""The change report (--changes) of the emulated kernels (tests/emu): k_tile's change list, k_allele_strings and the shared row
formatter against the oracle's --debug TSV filtered to its `changed` rows, byte for byte.  CPU only."""
import pytest

import polypolish_b200 as pp
from tests import emu_lib, fuzzgen
from tests.test_emu_depth_boundary import HALF_BELOW, HALF_ON, MIN_DEPTH_BELOW, MIN_DEPTH_ON, _seq_sum, write_case

# k of the alignments over the probed position in two SAM orders: the reference's depth is 3.25 (printed "3.2") in the first and
# 3.2500000000000004 (printed "3.3") in the second, so the report's depth column depends on the order of the sum
PRINT_ON = [12, 6, 3, 12, 6, 10, 6, 1, 10, 3, 6, 5, 10, 6, 12]
PRINT_ABOVE = [6, 6, 3, 12, 10, 12, 6, 5, 10, 6, 10, 1, 3, 6, 12]


def changed_rows(debug_tsv):
    lines = debug_tsv.split(b"\n")
    return b"\n".join([lines[0]] + [x for x in lines[1:] if x.split(b"\t")[7:8] == [b"changed"]]) + b"\n"


def check_changes(oracle, fa, sams, grid_tiles=2, **opts):
    exp = oracle.polish(fa, sams, debug=True, **opts)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams, careful=opts.get("careful", False))
    r = emu_lib.polish(f, p, grid_tiles=grid_tiles, changes=True, **opts)
    assert "error" not in r, r
    assert emu_lib.fasta_bytes(f, r["sequences"]) == exp["fasta"]
    assert r["changes"] == changed_rows(exp["debug_tsv"])
    assert r["changes"].count(b"\n") - 1 == sum(exp["changed"])
    return r


@pytest.mark.parametrize("seed", [100, 101, 104, 107, 112, 116, 121, 133, 140, 152, 164, 175])
def test_emu_changes_fuzz(oracle, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0)
    fa, sams = case.write(tmp_path)
    try:
        oracle.polish(fa, sams, **case.opts)
    except Exception:
        pytest.skip("the reference rejects this input")
    check_changes(oracle, fa, sams, **case.opts)


@pytest.mark.parametrize("seed", [300, 303, 307])
def test_emu_changes_deep_multimap(oracle, tmp_path, seed):
    """Non-dyadic k everywhere: the printed depth is the reference's ordered sum, not the fixed-point estimate."""
    case = fuzzgen.make_case(seed, n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False))
    fa, sams = case.write(tmp_path)
    check_changes(oracle, fa, sams, **case.opts)


@pytest.mark.parametrize("ks", [MIN_DEPTH_ON, MIN_DEPTH_BELOW], ids=["on", "below"])
def test_emu_changes_depth_on_min_depth(oracle, tmp_path, ks):
    fa, sam, P = write_case(tmp_path, ks)
    r = check_changes(oracle, fa, [sam], grid_tiles=1, min_depth=5)
    assert r["changes"].count(b"\n") == (2 if ks is MIN_DEPTH_ON else 1)


@pytest.mark.parametrize("ks", [HALF_ON, HALF_BELOW], ids=["on", "below"])
def test_emu_changes_depth_on_half(oracle, tmp_path, ks):
    fa, sam, P = write_case(tmp_path, ks, x_reads=3)
    r = check_changes(oracle, fa, [sam], grid_tiles=1, min_depth=1, fraction_valid=0.9, fraction_invalid=0.5)
    assert r["changes"].count(b"\n") == (2 if ks is HALF_ON else 1)


@pytest.mark.parametrize("ks", [PRINT_ON, PRINT_ABOVE], ids=["on", "above"])
def test_emu_changes_printed_depth_follows_sam_order(oracle, tmp_path, ks):
    """A changed position whose depth is x.x5 in one SAM order and one ulp above it in the other: "3.2" or "3.3"."""
    assert _seq_sum(ks) == (3.25 if ks is PRINT_ON else 3.2500000000000004)
    fa, sam, P = write_case(tmp_path, ks)
    r = check_changes(oracle, fa, [sam], grid_tiles=1, min_depth=1)
    row = r["changes"].split(b"\n")[1].split(b"\t")
    assert row[:2] == [b"probe", str(P).encode()] and row[3] == (b"3.2" if ks is PRINT_ON else b"3.3")
