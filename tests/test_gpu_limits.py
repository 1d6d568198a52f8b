"""The polish path past its size limits on the GPU, against the oracle through every entry point a case can reach: long other alleles,
output growth (unstaged compaction chunks, the output-capacity repeats of the library and of its callers), node-pool growth, read
groups past the in-block scan limit (global-k mode) and across SAM files, and depths exactly on a vote boundary.  The cases come
from tests/limitgen.py; each asserts first that it crosses its limit."""
import os
import subprocess

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import limitgen as lg
from tests.test_emu_changes import PRINT_ABOVE, PRINT_ON
from tests.test_emu_depth_boundary import HALF_BELOW, HALF_ON, MIN_DEPTH_BELOW, MIN_DEPTH_ON, write_case
from tests.test_emu_limits import BOUNDARY_SETS, LONG, LONG8, pileup_alleles
from tests.test_gpu_changes import changed_rows

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def fasta_of(f, seqs):
    return b"".join(b">" + f.names[i].encode() + ((b" " + f.descriptions[i].encode()) if f.descriptions[i] else b"") + b" polypolish\n" +
                    seqs[i] + b"\n" for i in range(len(seqs)))


def same_stats(r, exp):
    assert r["changed"] == exp["changed"] and r["zero_depth"] == exp["zero_depth"] and r["n_aln_used"] == exp["used_total"]
    for got, want in zip(r["total_depth"], exp["total_depth"]):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want))


def check_files(ctx, oracle, tmp_path, fa, sams, exp=None, **opts):
    """ctx.polish_files with the device tokeniser and the host parser, --debug and --changes on: FASTA, debug TSV, change report."""
    exp = exp or oracle.polish(fa, sams, debug=True, **opts)
    for parser in (0, 1):
        dbg, chg = tmp_path / ("debug%d.tsv" % parser), tmp_path / ("changes%d.tsv" % parser)
        ctx.set_parser(parser)
        try:
            assert ctx.polish_files(fa, sams, debug=dbg, changes=chg, **opts) == exp["fasta"], parser
        finally:
            ctx.set_parser(0)
        assert dbg.read_bytes() == exp["debug_tsv"], parser
        assert chg.read_bytes() == changed_rows(exp["debug_tsv"]), parser
        assert chg.read_bytes().count(b"\n") - 1 == sum(exp["changed"])
    return exp


def check_packed(ctx, oracle, fa, sams, f, p, opt_sets):
    """polish_packed with the first option set, then the resident dataset with every option set: FASTA and statistics."""
    out = []
    r = ctx.polish_packed(f.view, p.view, **opt_sets[0])
    exp = oracle.polish(fa, sams, **opt_sets[0])
    assert fasta_of(f, r["sequences"]) == exp["fasta"]
    same_stats(r, exp)
    out.append(r)
    ctx.upload(f.view, p.view)
    for opts in opt_sets:
        r = ctx.polish_resident(**opts)
        exp = oracle.polish(fa, sams, **opts)
        assert fasta_of(f, r["sequences"]) == exp["fasta"], opts
        same_stats(r, exp)
        out.append(r)
    return out


# ---- A. long other alleles -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["4bit", "8bit", "huge"])
def test_long_alleles(ctx, oracle, tmp_path, kind):
    case = (lg.long_alleles(1, LONG) if kind == "4bit" else lg.long_alleles(2, LONG8, eight_bit=True) if kind == "8bit"
            else lg.long_alleles(3, [16, 300], huge=True))
    fa, sams = case.write(tmp_path)
    exp = check_files(ctx, oracle, tmp_path, fa, sams, **case.opts)
    lens = {len(a) for _, _, a, n in pileup_alleles(exp["debug_tsv"]) if n >= 5}
    assert set(case.facts["allele_lengths"]) <= lens and max(lens) > (7 if kind == "8bit" else 15)
    assert sum(exp["changed"]) >= len(case.facts["allele_lengths"])
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == case.facts["seq_bits"]
    check_packed(ctx, oracle, fa, sams, f, p, [case.opts, dict(min_depth=1, fraction_invalid=0.1), dict(careful=True), case.opts])


def test_long_alleles_cli(oracle, tmp_path):
    """The CLI binary on the long-allele case: FASTA on stdout, --debug and --changes files."""
    case = lg.long_alleles(1, LONG)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, min_depth=4)
    dbg, chg = tmp_path / "debug.tsv", tmp_path / "changes.tsv"
    r = subprocess.run([os.path.join(ROOT, "build", "polypolish"), "polish", "--min_depth", "4", "--debug", str(dbg), "--changes", str(chg),
                        str(fa)] + [str(s) for s in sams], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"] and dbg.read_bytes() == exp["debug_tsv"] and chg.read_bytes() == changed_rows(exp["debug_tsv"])


# ---- B. output growth ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def growth(tmp_path_factory, oracle):
    d = tmp_path_factory.mktemp("growth")
    case = lg.output_growth(4)
    fa, sams = case.write(d)
    exp = oracle.polish(fa, sams, debug=True)
    G = case.facts["G"]
    total = sum(len(l) for l in exp["fasta"].split(b"\n")[1::2])
    assert total == case.facts["total"] > G + G // 16 + (1 << 20)                   # past the library's and the callers' first capacity
    assert case.facts["chunk_bytes"][case.facts["boundary_chunk"]] > lg.CP_STAGE
    assert sum(1 for b in case.facts["chunk_bytes"].values() if b > lg.CP_STAGE) == len(case.facts["chunk_bytes"])
    return d, fa, sams, exp


def test_output_growth_files(ctx, oracle, growth, tmp_path):
    d, fa, sams, exp = growth
    assert string_pool_excess(exp["debug_tsv"]) > 0
    with pp.Context(0) as c:                                       # a fresh context: the first output and string-pool capacities
        check_files(c, oracle, tmp_path, fa, sams, exp=exp)


def test_output_growth_packed_and_resident(oracle, growth):
    d, fa, sams, exp = growth
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    with pp.Context(0) as c:
        rs = check_packed(c, oracle, fa, sams, f, p, [dict(), dict(min_depth=3), dict()])
        assert rs[0]["out_len"] == sum(len(l) for l in exp["fasta"].split(b"\n")[1::2])


def test_output_growth_pinned_too_small(oracle, growth):
    """A caller's pinned buffer smaller than the output: PP_ERR_ARG with the needed out_len, and nothing copied into it."""
    d, fa, sams, exp = growth
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    G = int(f.off[-1])
    need = sum(len(l) for l in exp["fasta"].split(b"\n")[1::2])
    with pp.Context(0) as c:
        res, keep = c.pinned_result(len(f.names), G + (1 << 20))
        try:
            for k in ("off", "bases", "changed", "zero"):
                keep[k][:] = 0xA5 if k == "bases" else 7
            with pytest.raises(pp.PolypolishError) as e:
                c.polish_packed(f.view, p.view, into=(res, keep))
            assert e.value.code == api.PP_ERR_ARG and res.out_len == need
            assert (keep["bases"] == 0xA5).all() and (keep["off"] == 7).all() and (keep["changed"] == 7).all() and (keep["zero"] == 7).all()
        finally:
            c.free_pinned_result(keep)
        res, keep = c.pinned_result(len(f.names), need)
        try:
            c.polish_packed(f.view, p.view, into=(res, keep))
            assert fasta_of(f, [keep["bases"][int(keep["off"][i]):int(keep["off"][i + 1])].tobytes() for i in range(len(f.names))]) == exp["fasta"]
        finally:
            c.free_pinned_result(keep)


# ---- C. node pool and allele-string pool ---------------------------------------------------------------------------------------------
def string_pool_excess(debug_tsv):
    """The largest excess, over the contigs of an oracle --debug TSV, of the allele-string bytes k_allele_strings writes for the rows
    with other alleles over the string pool's first capacity, rows * 16 + 4096 (polish_kernels.cu allele_strings; one call per
    contig here).  The emitted alleles are left out of the bytes, so this is a lower bound: > 0 means the first pool overflowed."""
    rows = {}
    for c, p, a, _ in pileup_alleles(debug_tsv):
        if len(a) > 1 or a not in "ACGT-":
            rows.setdefault((c, p), []).append(a)
    per = {}
    for (c, _), alleles in rows.items():
        b, n = per.get(c, (0, 0))
        per[c] = (b + 8 + sum(8 + len(a) for a in alleles), n + 1)
    return max(b - (n * 16 + 4096) for b, n in per.values())


def test_node_pool_growth(oracle, tmp_path):
    """More distinct (position, allele) pairs than the first node capacity: the call repeats with a grown pool, which stays grown for
    more option sets on the same dataset; then, on the same context, --debug calls whose allele strings overflow the first string pool."""
    case = lg.node_pool(8)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True)
    distinct = {(c, p, a) for c, p, a, _ in pileup_alleles(exp["debug_tsv"]) if len(a) > 1}
    assert len(distinct) > case.facts["node_cap"] == 65536
    assert string_pool_excess(exp["debug_tsv"]) > 0
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    with pp.Context(0) as c:
        check_packed(c, oracle, fa, sams, f, p, [dict(), dict(max_errors=0), dict(fraction_invalid=0.01, fraction_valid=0.02)])
        check_files(c, oracle, tmp_path, fa, sams, exp=exp)


# ---- D. read groups ------------------------------------------------------------------------------------------------------------------
GPU_GROUPS = [([2, 255, 256, 257, 511, 8191], 0, "first", False), ([8192, 8193], 1, "last", False), ([8448, 257], 255, "first", True),
              ([20_000], 0, "last", True)]


@pytest.mark.parametrize("sizes,offset,where,global_k", GPU_GROUPS, ids=["small-0-first", "8192-8193-1-last", "8448-255-first", "20000-0-last"])
def test_read_groups(ctx, oracle, tmp_path, sizes, offset, where, global_k):
    case = lg.read_groups(31 + offset, sizes, offset=offset, where=where)
    fa, sams = case.write(tmp_path)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    rid = p.arrays()["read_id"].copy()
    groups = dict(lg.group_records(rid))
    for g in case.facts["groups"]:
        assert groups[g["start"]] == g["size"] and g["start"] % 256 == offset
    assert groups[case.facts["split_cut"] - 3] == 3 and groups[case.facts["split_cut"]] == 4          # `split`: two groups
    assert lg.expect_global_k(rid, lg.record_good(case.sam_texts)) == global_k
    check_files(ctx, oracle, tmp_path, fa, sams)
    # k is recounted per call in global-k mode: launches 4 (k_classify_multi) once the mode is on, 3 otherwise
    rs = check_packed(ctx, oracle, fa, sams, f, p, [dict(), dict(max_errors=0), dict(careful=True), dict()])
    assert [r["timing"]["launches"] for r in rs] == [4 if global_k else 3] * len(rs)
    # a later dataset without big groups: global-k is off again
    small = lg.read_groups(3, [2, 5], offset=0, where="first", filler=300)
    d2 = tmp_path / "small"
    d2.mkdir()
    fa2, sams2 = small.write(d2)
    f2 = pp.load_fasta(fa2)
    p2 = pp.pack_sams(f2, sams2)
    rs = check_packed(ctx, oracle, fa2, sams2, f2, p2, [dict()])
    assert [r["timing"]["launches"] for r in rs] == [3, 3]
    # contig shards (ghost records count towards k), both loaders, and the 2-bit upload
    exp = oracle.polish(fa, sams, debug=True)
    for devices in ([0, 0], [0, 0, 0]):
        for parser in (0, 1):
            chg = tmp_path / "multi.tsv"
            assert api.polish_files_multi(fa, sams, devices=devices, parser=parser, changes=chg) == exp["fasta"], (devices, parser)
            assert chg.read_bytes() == changed_rows(exp["debug_tsv"])
    tb = api.TwoBit(p.view)
    r = ctx.polish_packed(f.view, tb.view)
    exp = oracle.polish(fa, sams)
    assert fasta_of(f, r["sequences"]) == exp["fasta"] and r["timing"]["launches"] == (4 if global_k else 3)
    same_stats(r, exp)
    tb.close()


# ---- E. depth on a vote boundary -----------------------------------------------------------------------------------------------------
def check_plain(ctx, oracle, fa, sams, **opts):
    """The case without --debug and --changes, where the vote decides from the fixed-point depth bound (depth_bounds) and walks only
    where the bound straddles a boundary: polish_files with both parsers, polish_packed and the resident dataset.  Returns the GPU's
    `changed` of the first contig."""
    exp = oracle.polish(fa, sams, **opts)
    for parser in (0, 1):
        ctx.set_parser(parser)
        try:
            assert ctx.polish_files(fa, sams, **opts) == exp["fasta"], parser
        finally:
            ctx.set_parser(0)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    rs = check_packed(ctx, oracle, fa, sams, f, p, [opts])
    return [r["changed"][0] for r in rs]


HALF_OPTS = dict(min_depth=1, fraction_valid=0.9, fraction_invalid=0.5)
# k in SAM order, the reference's depth at the probed position (exactly the boundary, or one ulp below / above it), options, reads with
# the second allele, and what the oracle does there: changed or not, and the depth --debug / --changes print
E_SETS = {"min-on": (MIN_DEPTH_ON, 5.0, dict(min_depth=5), 0, 1, b"5.0"),
          "min-below": (MIN_DEPTH_BELOW, np.nextafter(5.0, 0.0), dict(min_depth=5), 0, 0, b"5.0"),
          "half-on": (HALF_ON, 7.0, HALF_OPTS, 3, 1, b"7.0"),
          "half-below": (HALF_BELOW, np.nextafter(7.0, 0.0), HALF_OPTS, 3, 0, b"7.0"),
          "print-on": (PRINT_ON, 3.25, dict(min_depth=1), 0, 1, b"3.2"),
          "print-above": (PRINT_ABOVE, np.nextafter(3.25, np.inf), dict(min_depth=1), 0, 1, b"3.3")}


@pytest.mark.parametrize("name", list(E_SETS))
def test_depth_boundary(ctx, oracle, tmp_path, name):
    """The depth-boundary cases of the emulator tests on the GPU: with --debug / --changes (every k != 1 position walks), and without
    them (the directed-rounding bound has to see that the position straddles the boundary).  The on / below sets of a boundary vote
    differently; the print sets both change and print "3.2" or "3.3"."""
    ks, depth, opts, x, want, printed = E_SETS[name]
    assert lg.seq_sum(ks) == depth
    fa, sam, P = write_case(tmp_path, ks, x_reads=x)
    exp = check_files(ctx, oracle, tmp_path, fa, [sam], **opts)
    assert exp["changed"][0] == want and exp["debug_tsv"].split(b"\n")[1 + P].split(b"\t")[3] == printed
    assert check_plain(ctx, oracle, fa, [sam], **opts) == [want, want]


@pytest.mark.parametrize("ks,target", BOUNDARY_SETS, ids=["k34-min", "k35-half", "k32-k33-min"])
def test_depth_boundary_past_the_table(ctx, oracle, tmp_path, ks, target):
    """k > 32 (the walk divides instead of reading its 1/k table), with and without --debug / --changes."""
    opts = HALF_OPTS if target == 7.0 else dict(min_depth=5)
    on, below = lg.boundary_orders(5, ks, target)
    assert lg.seq_sum(on) == target and lg.seq_sum(below) == np.nextafter(target, 0.0)
    got, plain = [], []
    for name, ks_ in (("on", on), ("below", below)):
        d = tmp_path / name
        d.mkdir()
        fa, sam, P = lg.boundary_case(d, ks_, x_reads=3 if target == 7.0 else 0)
        got.append(check_files(ctx, oracle, d, fa, [sam], **opts)["changed"][0])
        plain.append(check_plain(ctx, oracle, fa, [sam], **opts))
    assert got == [1, 0]                                                   # the oracle's two orders really vote differently
    assert plain == [[1, 1], [0, 0]]                                       # and so do polish_packed and the resident dataset
