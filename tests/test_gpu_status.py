"""The status runs (`polish --status-bed`, pp_polish_set_status / pp_polish_status_fetch) on the GPU: the run-length encoding of the
oracle's --debug status column, byte for byte, whichever loader, context count or entry point produced them; the FASTA never
changes."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import endgen, fuzzgen, statusgen
from tests.statusgen import bed_from_debug_tsv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")
WORDS = [x.decode() for x in statusgen.STATUS]


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def bed_of_runs(f, runs):
    """Context.status_runs (global positions) as the BED lines of --status-bed."""
    out = []
    for s, e, st in zip(runs["start"].tolist(), runs["end"].tolist(), runs["status"].tolist()):
        c = int(np.searchsorted(f.off, s, side="right")) - 1
        out.append("%s\t%d\t%d\t%s\n" % (f.names[c], s - int(f.off[c]), e - int(f.off[c]), WORDS[st]))
    return "".join(out).encode()


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
@pytest.mark.parametrize("seed", [100, 101, 104, 105, 300, 303])
def test_status_parity(ctx, oracle, tmp_path, seed, parser):
    """The --debug parity seeds (4-bit and 8-bit pools, insertions, IUPAC drafts, deep multi-maps), both SAM parsers."""
    kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    out = tmp_path / "status.bed"
    ctx.set_parser(parser)
    try:
        assert ctx.polish_files(fa, sams, status=out, **case.opts) == exp["fasta"]
    finally:
        ctx.set_parser(0)
    assert out.read_bytes() == bed_from_debug_tsv(exp["debug_tsv"])


@pytest.mark.parametrize("name", sorted(statusgen.CASES))
def test_status_boundary(ctx, oracle, tmp_path, name):
    """statusgen: P's depth on a status boundary or one ulp below it; the oracle's statuses differ there, the FASTA does not."""
    on, off, spec = statusgen.case_pair(name)
    for c, want in ((on, spec["st_on"]), (off, spec["st_off"])):
        d = tmp_path / ("on" if c is on else "off")
        d.mkdir()
        fa, sams = c.write(d)
        exp = oracle.polish(fa, sams, debug=True, **c.opts)
        assert statusgen.status_at(exp["debug_tsv"], "probe", spec["P"]) == want
        out = d / "status.bed"
        assert ctx.polish_files(fa, sams, status=out, **c.opts) == exp["fasta"]
        assert out.read_bytes() == bed_from_debug_tsv(exp["debug_tsv"])


@pytest.mark.parametrize("eight", [False, True], ids=["4bit", "8bit"])
def test_status_contig_ends(ctx, oracle, tmp_path, eight):
    """endgen's contig ends: contigs of 1-9 bp, starts at every residue mod 32, contigs no read covers."""
    c = endgen.edges(41, eight_bit=eight)
    fa, sams = c.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **c.opts)
    out = tmp_path / "status.bed"
    assert ctx.polish_files(fa, sams, status=out, **c.opts) == exp["fasta"]
    assert out.read_bytes() == bed_from_debug_tsv(exp["debug_tsv"])


@pytest.mark.parametrize("min_depth,word", [(5, b"low_depth"), (0, b"multiple")])
def test_status_without_sam_files(ctx, oracle, tmp_path, min_depth, word):
    """No alignments: one run per contig, low_depth, or multiple with -d 0 (A, C, G and T all reach a valid threshold of 0)."""
    case = fuzzgen.make_case(101)
    fa, _ = case.write(tmp_path)
    exp = oracle.polish(fa, [], debug=True, min_depth=min_depth)
    out = tmp_path / "status.bed"
    assert ctx.polish_files(fa, [], status=out, min_depth=min_depth) == exp["fasta"]
    f = pp.load_fasta(fa)
    want = b"".join(b"%s\t0\t%d\t%s\n" % (n.encode(), int(f.off[i + 1] - f.off[i]), word) for i, n in enumerate(f.names))
    assert out.read_bytes() == want == bed_from_debug_tsv(exp["debug_tsv"])


def test_status_eight_bit_pool(ctx, oracle, tmp_path):
    """A read with a SEQ byte outside the 4-bit alphabet: the 8-bit pool and k_tile<8> in status mode."""
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
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == 8
    out = tmp_path / "status.bed"
    assert ctx.polish_files(fa, sams, status=out) == exp["fasta"]
    assert out.read_bytes() == bed_from_debug_tsv(exp["debug_tsv"])


def test_status_resident(ctx, oracle, tmp_path):
    """One resident dataset through the option grid, status on alternate calls and --changes on some of them; a failed call
    leaves nothing recording."""
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
            assert "status" not in r
            with pytest.raises(pp.PolypolishError):
                ctx.status_runs()
        else:
            r = ctx.polish_resident(status=True, changes=i % 4 == 0, **opts)
            assert bed_of_runs(f, r["status"]) == bed_from_debug_tsv(exp["debug_tsv"]), opts
            assert int((r["status"]["end"] - r["status"]["start"]).sum()) == int(f.off[-1])
            if i % 4 == 0:
                assert len(r["changes"]) == sum(r["changed"])
        assert [int(x) for x in r["changed"]] == exp["changed"], opts
    # a failed call, then a plain one: nothing to fetch
    with pytest.raises(pp.PolypolishError):
        ctx.polish_resident(status=True, fraction_valid=1.5)
    with pytest.raises(pp.PolypolishError):
        ctx.status_runs()
    ctx.polish_resident()
    with pytest.raises(pp.PolypolishError):
        ctx.status_runs()


def test_status_contexts(ctx, oracle, tmp_path):
    """Every context reports the runs of its own contigs; 1, 2, 3 and 8 contexts on one device write the same bytes."""
    syn = api.Synth(seed=9, n_contigs=8, contig_len=12_000, depth=50, draft_error_rate=2e-3)
    fa, sams = syn.write(tmp_path)
    one = tmp_path / "one.bed"
    exp = ctx.polish_files(fa, sams, status=one)
    assert one.read_bytes() == bed_from_debug_tsv(oracle.polish(fa, sams, debug=True)["debug_tsv"])
    for n in (2, 3, 8):
        for parser in (0, 1):
            out = tmp_path / ("multi%d_%d.bed" % (n, parser))
            assert api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser, status=out) == exp
            assert out.read_bytes() == one.read_bytes(), (n, parser)


@pytest.mark.parametrize("n_ctx", [1, 2, 3])
def test_status_filter_polish(oracle, tmp_path, n_ctx):
    """filter + polish in one call: the runs of the oracle's `filter`, then `polish --debug` of its output."""
    syn = api.Synth(seed=5, n_contigs=3, contig_len=30_000, depth=60, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    ef = oracle.filter(sams[0], sams[1])
    f1, f2 = tmp_path / "f1.sam", tmp_path / "f2.sam"
    f1.write_bytes(ef["out1"])
    f2.write_bytes(ef["out2"])
    exp = oracle.polish(fa, [f1, f2], debug=True)
    out = tmp_path / "status.bed"
    assert api.filter_polish_files_multi(fa, sams[0], sams[1], devices=[0] * n_ctx, status=out) == exp["fasta"]
    assert out.read_bytes() == bed_from_debug_tsv(exp["debug_tsv"])


def test_status_cli(oracle, tmp_path):
    """--debug, --changes and --status-bed together: the BED is the run-length encoding of the TSV written beside it; and the
    file-creation error."""
    syn = api.Synth(seed=4, n_contigs=2, contig_len=30_000, depth=40, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, min_depth=4)
    dbg, chg, bed = tmp_path / "debug.tsv", tmp_path / "changes.tsv", tmp_path / "status.bed"
    r = subprocess.run([EXE, "polish", "--min_depth", "4", "--debug", str(dbg), "--changes", str(chg), "--status-bed", str(bed), fa] + sams,
                       capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"] and dbg.read_bytes() == exp["debug_tsv"]
    assert bed.read_bytes() == bed_from_debug_tsv(dbg.read_bytes())
    r2 = subprocess.run([EXE, "polish", "--status-bed=" + str(tmp_path / "eq.bed"), "-d4", fa] + sams, capture_output=True)
    assert r2.returncode == 0 and r2.stdout == exp["fasta"]
    assert (tmp_path / "eq.bed").read_bytes() == bed.read_bytes()
    r = subprocess.run([EXE, "polish", "--status-bed", str(tmp_path / "no" / "x.bed"), fa] + sams, capture_output=True)
    assert r.returncode == 1 and r.stderr.endswith(b'Error: unable to create "%s"\n' % str(tmp_path / "no" / "x.bed").encode())
    with pytest.raises(pp.PolypolishError) as e:
        pp.polish(fa, sams, status=tmp_path / "no" / "y.bed")
    assert e.value.msg == 'unable to create "%s"' % (tmp_path / "no" / "y.bed")


def test_status_full_size(oracle):
    """BASELINE config 2 (5 Mbp x 100x): the BED is the run-length encoding of this build's own --debug TSV, covers every base, and
    its `changed` runs add up to the log's changed count."""
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_sts_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        syn = api.Synth(seed=2, contig_len=5_000_000, depth=100)
        fa, sams = syn.write(d)
        dbg, bed = os.path.join(d, "debug.tsv"), os.path.join(d, "status.bed")
        r1 = subprocess.run([EXE, "polish", "--debug", dbg, fa] + sams, capture_output=True)
        r2 = subprocess.run([EXE, "polish", "--status-bed", bed, fa] + sams, capture_output=True)
        assert r1.returncode == 0 and r2.returncode == 0, (r1.stderr.decode(), r2.stderr.decode())
        assert r2.stdout == r1.stdout
        got = open(bed, "rb").read()
        assert got == bed_from_debug_tsv(open(dbg, "rb").read())
        rows = [x.split(b"\t") for x in got.splitlines()]
        assert sum(int(c[2]) - int(c[1]) for c in rows) == int(pp.load_fasta(fa).off[-1])
        logged = sum(int(x.split()[0].replace(b",", b"")) for x in r2.stderr.split(b"\n") if b"changed (" in x)
        assert sum(int(c[2]) - int(c[1]) for c in rows if c[3] == b"changed") == logged > 0
    finally:
        shutil.rmtree(d, ignore_errors=True)
