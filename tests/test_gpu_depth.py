"""The depth runs (`polish --depth-bedgraph`, pp_polish_set_depth / pp_polish_depth_fetch) on the GPU: the run-length encoding of the
oracle's --debug depth column, byte for byte, whichever loader, context count or entry point produced them; the FASTA and the other
reports never change."""
import os
import shutil
import subprocess
import tempfile

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import depthgen, endgen, fuzzgen, statusgen
from tests.depthgen import bedgraph_from_debug_tsv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def of_runs(f, runs):
    return depthgen.bedgraph_from_runs(f.names, [int(x) for x in f.off], runs)


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
@pytest.mark.parametrize("seed", [100, 101, 104, 105, 300, 303])
def test_depth_parity(ctx, oracle, tmp_path, seed, parser):
    """The --debug parity seeds (4-bit and 8-bit pools, insertions, IUPAC drafts, deep multi-maps), both SAM parsers."""
    kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    out = tmp_path / "depth.bedgraph"
    ctx.set_parser(parser)
    try:
        assert ctx.polish_files(fa, sams, depth_bedgraph=out, **case.opts) == exp["fasta"]
    finally:
        ctx.set_parser(0)
    assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])


@pytest.mark.parametrize("name", sorted(depthgen.CASES) + sorted(depthgen.DYADIC))
def test_depth_print_boundary(ctx, oracle, tmp_path, name):
    """depthgen: P's depth prints one tenth in one SAM order and the tenth below in the other; the FASTA does not change."""
    on, off, spec = depthgen.case_pair(name)
    for c, want in ((on, spec["on"]), (off, spec["off"])):
        d = tmp_path / ("on" if c is on else "off")
        d.mkdir()
        fa, sams = c.write(d)
        exp = oracle.polish(fa, sams, debug=True, **c.opts)
        assert depthgen.depth_at(exp["debug_tsv"], "probe", spec["P"]) == want
        out = d / "depth.bedgraph"
        assert ctx.polish_files(fa, sams, depth_bedgraph=out, **c.opts) == exp["fasta"]
        assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])


@pytest.mark.parametrize("eight", [False, True], ids=["4bit", "8bit"])
def test_depth_contig_ends(ctx, oracle, tmp_path, eight):
    """endgen's contig ends: contigs of 1-9 bp, starts at every residue mod 32, contigs no read covers."""
    c = endgen.edges(41, eight_bit=eight)
    fa, sams = c.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **c.opts)
    out = tmp_path / "depth.bedgraph"
    assert ctx.polish_files(fa, sams, depth_bedgraph=out, **c.opts) == exp["fasta"]
    assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])


def test_depth_without_sam_files(ctx, oracle, tmp_path):
    """No alignments: one 0.0 run per contig."""
    case = fuzzgen.make_case(101)
    fa, _ = case.write(tmp_path)
    exp = oracle.polish(fa, [], debug=True)
    out = tmp_path / "depth.bedgraph"
    assert ctx.polish_files(fa, [], depth_bedgraph=out) == exp["fasta"]
    f = pp.load_fasta(fa)
    want = b"".join(b"%s\t0\t%d\t0.0\n" % (n.encode(), int(f.off[i + 1] - f.off[i])) for i, n in enumerate(f.names))
    assert out.read_bytes() == want == bedgraph_from_debug_tsv(exp["debug_tsv"])


def test_depth_eight_bit_pool(ctx, oracle, tmp_path):
    """A read with a SEQ byte outside the 4-bit alphabet: the 8-bit pool and k_tile<8> in depth mode."""
    syn = api.Synth(seed=8, n_contigs=2, contig_len=20_000, depth=40, draft_error_rate=2e-3)
    fa, sams = syn.write(tmp_path)
    text = open(sams[0], "rb").read().split(b"\n")
    for i, line in enumerate(text):
        c = line.split(b"\t")
        if len(c) > 10 and not line.startswith(b"@") and len(c[9]) > 20:
            c[9] = c[9][:10] + b"." + c[9][11:]
            text[i] = b"\t".join(c)
            break
    open(sams[0], "wb").write(b"\n".join(text))
    exp = oracle.polish(fa, sams, debug=True)
    f = pp.load_fasta(fa)
    assert pp.pack_sams(f, sams).view.seq_bits == 8
    out = tmp_path / "depth.bedgraph"
    assert ctx.polish_files(fa, sams, depth_bedgraph=out) == exp["fasta"]
    assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])


def test_depth_resident(ctx, oracle, tmp_path):
    """One resident dataset through the option grid, depth on alternate calls (with the status runs or the change report on some of
    them); a failed call leaves nothing recording."""
    syn = api.Synth(seed=3, n_contigs=3, contig_len=40_000, depth=80, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    f = syn.fasta()
    p = syn.pack(f)
    ctx.upload(f.view, p.view)
    grid = [dict(min_depth=d, **fr) for d in (0, 1, 2, 5) for fr in (dict(), dict(fraction_invalid=0.001, fraction_valid=0.5))]
    grid += [dict(careful=True), dict(max_errors=2), dict(fraction_invalid=0.05, fraction_valid=0.95)]
    for i, opts in enumerate(grid):
        exp = oracle.polish(fa, sams, debug=True, **opts)
        if i % 2:
            r = ctx.polish_resident(**opts)
            assert "depth" not in r
            with pytest.raises(pp.PolypolishError):
                ctx.depth_runs()
        else:
            r = ctx.polish_resident(depth_runs=True, status=i % 4 == 0, changes=i % 8 == 2, **opts)
            assert of_runs(f, r["depth"]) == bedgraph_from_debug_tsv(exp["debug_tsv"]), opts
            assert int((r["depth"]["end"] - r["depth"]["start"]).sum()) == int(f.off[-1])
            if i % 4 == 0:
                assert int((r["status"]["end"] - r["status"]["start"]).sum()) == int(f.off[-1])
        assert [int(x) for x in r["changed"]] == exp["changed"], opts
    # a failed call, then a plain one: nothing to fetch
    with pytest.raises(pp.PolypolishError):
        ctx.polish_resident(depth_runs=True, fraction_valid=1.5)
    with pytest.raises(pp.PolypolishError):
        ctx.depth_runs()
    ctx.polish_resident()
    with pytest.raises(pp.PolypolishError):
        ctx.depth_runs()


def test_depth_change_list_retry(oracle, tmp_path):
    """A draft with about 5 % errors on a fresh context: more changed positions than the change list's first capacity, so the call
    repeats itself; the runs come from the final attempt."""
    syn = api.Synth(seed=12, contig_len=200_000, depth=40, draft_error_rate=0.05)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True)
    assert sum(exp["changed"]) > 4096
    out, chg = tmp_path / "depth.bedgraph", tmp_path / "changes.tsv"
    with pp.Context(0) as c:
        assert c.polish_files(fa, sams, changes=chg, depth_bedgraph=out) == exp["fasta"]
    assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])


def test_depth_contexts(ctx, oracle, tmp_path):
    """Every context reports the runs of its own contigs; 1, 2, 3 and 8 contexts on one device write the same bytes."""
    syn = api.Synth(seed=9, n_contigs=8, contig_len=12_000, depth=50, draft_error_rate=2e-3)
    fa, sams = syn.write(tmp_path)
    one = tmp_path / "one.bedgraph"
    exp = ctx.polish_files(fa, sams, depth_bedgraph=one)
    assert one.read_bytes() == bedgraph_from_debug_tsv(oracle.polish(fa, sams, debug=True)["debug_tsv"])
    for n in (2, 3, 8):
        for parser in (0, 1):
            out = tmp_path / ("multi%d_%d.bedgraph" % (n, parser))
            assert api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser, depth_bedgraph=out) == exp
            assert out.read_bytes() == one.read_bytes(), (n, parser)


@pytest.mark.parametrize("n_ctx", [1, 2, 3])
def test_depth_filter_polish(oracle, tmp_path, n_ctx):
    """filter + polish in one call: the runs of the oracle's `filter`, then `polish --debug` of its output."""
    syn = api.Synth(seed=5, n_contigs=3, contig_len=30_000, depth=60, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    ef = oracle.filter(sams[0], sams[1])
    f1, f2 = tmp_path / "f1.sam", tmp_path / "f2.sam"
    f1.write_bytes(ef["out1"])
    f2.write_bytes(ef["out2"])
    exp = oracle.polish(fa, [f1, f2], debug=True)
    out = tmp_path / "depth.bedgraph"
    assert api.filter_polish_files_multi(fa, sams[0], sams[1], devices=[0] * n_ctx, depth_bedgraph=out) == exp["fasta"]
    assert out.read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])
    if n_ctx == 1:
        with pp.Context(0) as c:
            out1 = tmp_path / "single.bedgraph"
            assert c.filter_polish_files(fa, sams[0], sams[1], depth_bedgraph=out1) == exp["fasta"]
            assert out1.read_bytes() == out.read_bytes()


def test_depth_cli(oracle, tmp_path):
    """--debug, --changes, --status-bed, --vcf and --depth-bedgraph together: each file equals its single-report run, the bedGraph is
    the run-length encoding of the TSV written beside it, the FASTA does not change; and the file-creation error."""
    syn = api.Synth(seed=4, n_contigs=2, contig_len=30_000, depth=40, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, min_depth=4)
    flags = dict(debug="debug.tsv", changes="changes.tsv", status_bed="status.bed", vcf="edits.vcf", depth_bedgraph="depth.bedgraph")
    all_dir, one_dir = tmp_path / "all", tmp_path / "one"
    all_dir.mkdir()
    one_dir.mkdir()
    args = [a for k, v in flags.items() for a in ("--" + k.replace("_", "-"), str(all_dir / v))]
    r = subprocess.run([EXE, "polish", "--min_depth", "4"] + args + [fa] + sams, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"] and (all_dir / "debug.tsv").read_bytes() == exp["debug_tsv"]
    assert (all_dir / "depth.bedgraph").read_bytes() == bedgraph_from_debug_tsv(exp["debug_tsv"])
    assert (all_dir / "status.bed").read_bytes() == statusgen.bed_from_debug_tsv(exp["debug_tsv"])
    for k, v in flags.items():
        r1 = subprocess.run([EXE, "polish", "-d4", "--%s=%s" % (k.replace("_", "-"), one_dir / v), fa] + sams, capture_output=True)
        assert r1.returncode == 0 and r1.stdout == exp["fasta"], k
        assert (one_dir / v).read_bytes() == (all_dir / v).read_bytes(), k
    r = subprocess.run([EXE, "polish", "--depth-bedgraph", str(tmp_path / "no" / "x.bedgraph"), fa] + sams, capture_output=True)
    assert r.returncode == 1 and r.stderr.endswith(b'Error: unable to create "%s"\n' % str(tmp_path / "no" / "x.bedgraph").encode())
    with pytest.raises(pp.PolypolishError) as e:
        pp.polish(fa, sams, depth_bedgraph=tmp_path / "no" / "y.bedgraph")
    assert e.value.msg == 'unable to create "%s"' % (tmp_path / "no" / "y.bedgraph")


def test_depth_full_size(oracle):
    """BASELINE config 2 (5 Mbp x 100x): the bedGraph is the run-length encoding of this build's own --debug TSV and covers every
    base; the FASTA is the same."""
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_dep_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        syn = api.Synth(seed=2, contig_len=5_000_000, depth=100)
        fa, sams = syn.write(d)
        dbg, bg = os.path.join(d, "debug.tsv"), os.path.join(d, "depth.bedgraph")
        r1 = subprocess.run([EXE, "polish", "--debug", dbg, fa] + sams, capture_output=True)
        r2 = subprocess.run([EXE, "polish", "--depth-bedgraph", bg, fa] + sams, capture_output=True)
        assert r1.returncode == 0 and r2.returncode == 0, (r1.stderr.decode(), r2.stderr.decode())
        assert r2.stdout == r1.stdout
        got = open(bg, "rb").read()
        assert got == bedgraph_from_debug_tsv(open(dbg, "rb").read())
        rows = [x.split(b"\t") for x in got.splitlines()]
        assert sum(int(c[2]) - int(c[1]) for c in rows) == int(pp.load_fasta(fa).off[-1])
    finally:
        shutil.rmtree(d, ignore_errors=True)
