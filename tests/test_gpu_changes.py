"""The change report (`polish --changes`, pp_polish_set_changes / pp_polish_changes_fetch) on the GPU: the --debug rows of the
changed positions, byte for byte the oracle's `changed` debug rows, whichever loader, shard count or entry point produced them."""
import os
import shutil
import subprocess
import tempfile

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import fuzzgen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def changed_rows(debug_tsv):
    lines = debug_tsv.split(b"\n")
    return b"\n".join([lines[0]] + [x for x in lines[1:] if x.split(b"\t")[7:8] == [b"changed"]]) + b"\n"


def n_rows(report):
    return report.count(b"\n") - 1


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
@pytest.mark.parametrize("seed", [100, 101, 104, 105, 300, 303])
def test_changes_parity(ctx, oracle, tmp_path, seed, parser):
    """The --debug parity seeds (4-bit and 8-bit pools, insertions, IUPAC drafts, deep multi-maps, --careful), both SAM parsers."""
    kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    out = tmp_path / "changes.tsv"
    ctx.set_parser(parser)
    try:
        assert ctx.polish_files(fa, sams, changes=out, **case.opts) == exp["fasta"]
    finally:
        ctx.set_parser(0)
    assert out.read_bytes() == changed_rows(exp["debug_tsv"])
    assert n_rows(out.read_bytes()) == sum(exp["changed"])


@pytest.fixture(scope="module")
def synth2(tmp_path_factory, oracle):
    d = tmp_path_factory.mktemp("synth2")
    syn = api.Synth(seed=6, n_contigs=2, contig_len=40_000, depth=60)
    fa, sams = syn.write(d)
    return fa, sams, oracle.polish(fa, sams, debug=True)


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
def test_changes_synth(ctx, synth2, tmp_path, parser):
    fa, sams, exp = synth2
    out = tmp_path / "changes.tsv"
    ctx.set_parser(parser)
    try:
        assert ctx.polish_files(fa, sams, changes=out) == exp["fasta"]
    finally:
        ctx.set_parser(0)
    assert out.read_bytes() == changed_rows(exp["debug_tsv"])
    assert n_rows(out.read_bytes()) > 0


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
def test_changes_shards(ctx, oracle, tmp_path, parser):
    """Every context reports its own contigs; the host merges them in the FASTA's contig order: same file as one context."""
    syn = api.Synth(seed=9, n_contigs=4, contig_len=30_000, depth=50, draft_error_rate=2e-3)
    fa, sams = syn.write(tmp_path)
    one = tmp_path / "one.tsv"
    exp = ctx.polish_files(fa, sams, changes=one)
    assert one.read_bytes() == changed_rows(oracle.polish(fa, sams, debug=True)["debug_tsv"])
    for devices in ([0, 0], [0, 0, 0, 0]):
        out = tmp_path / ("multi%d.tsv" % len(devices))
        assert api.polish_files_multi(fa, sams, devices=devices, parser=parser, changes=out) == exp
        assert out.read_bytes() == one.read_bytes(), devices


def test_changes_resident(ctx, oracle, tmp_path):
    """Several option sets on one resident dataset: each call's rows are the oracle's changed positions, as many as Σ changed."""
    syn = api.Synth(seed=3, n_contigs=3, contig_len=40_000, depth=80, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    f = syn.fasta()
    p = syn.pack(f)
    ctx.upload(f.view, p.view)
    for opts in (dict(), dict(careful=True), dict(min_depth=0), dict(max_errors=2), dict(fraction_invalid=0.05, fraction_valid=0.95), dict()):
        r = ctx.polish_resident(changes=True, **opts)
        assert len(r["changes"]) == sum(r["changed"]), opts
        exp = changed_rows(oracle.polish(fa, sams, debug=True, **opts)["debug_tsv"]).split(b"\n")[1:-1]
        got = []
        for x in exp:
            cols = x.split(b"\t")
            got.append((int(f.off[f.names.index(cols[0].decode())]) + int(cols[1]), cols[8].decode()))
        assert [(x["pos"], x["new_base"]) for x in r["changes"]] == got, opts
    # a call without the report records nothing
    r = ctx.polish_resident()
    assert "changes" not in r
    with pytest.raises(pp.PolypolishError):
        ctx.changes_rows()


def test_changes_filter_polish(ctx, oracle, tmp_path):
    """filter + polish in one call: the report of the oracle's `filter`, then `polish --debug` of its output, filtered."""
    syn = api.Synth(seed=5, contig_len=60_000, depth=60, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    ef = oracle.filter(sams[0], sams[1])
    f1, f2 = tmp_path / "f1.sam", tmp_path / "f2.sam"
    f1.write_bytes(ef["out1"])
    f2.write_bytes(ef["out2"])
    exp = oracle.polish(fa, [f1, f2], debug=True)
    out = tmp_path / "changes.tsv"
    assert ctx.filter_polish_files(fa, sams[0], sams[1], changes=out) == exp["fasta"]
    assert out.read_bytes() == changed_rows(exp["debug_tsv"])
    assert n_rows(out.read_bytes()) == sum(exp["changed"]) > 0


def test_changes_overflow(oracle, tmp_path):
    """A draft with about 5 % errors: more changed positions than the change list's first capacity (the call repeats itself with
    the exact size)."""
    syn = api.Synth(seed=12, contig_len=200_000, depth=40, draft_error_rate=0.05)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True)
    assert sum(exp["changed"]) > 4096
    out = tmp_path / "changes.tsv"
    with pp.Context(0) as c:                                   # a fresh context: the first capacity
        assert c.polish_files(fa, sams, changes=out) == exp["fasta"]
    assert out.read_bytes() == changed_rows(exp["debug_tsv"])


def test_failed_changes_call_stops_recording(ctx, oracle, tmp_path):
    """A --changes call that fails leaves nothing recording: a later plain call on the context has no rows to fetch."""
    syn = api.Synth(seed=7, contig_len=20_000, depth=30)
    fa, sams = syn.write(tmp_path)
    bad = tmp_path / "bad.sam"
    bad.write_bytes(open(sams[0], "rb").read() + b"zz\t0\tcontig_1\t1\t60\t4M\t*\t0\t0\tACGT\n")      # too few columns
    with pytest.raises(pp.PolypolishError):
        ctx.polish_files(fa, [bad], changes=tmp_path / "changes.tsv")
    with pytest.raises(pp.PolypolishError):
        ctx.changes_rows()
    assert ctx.polish_files(fa, sams) == oracle.polish(fa, sams)["fasta"]
    with pytest.raises(pp.PolypolishError):
        ctx.changes_rows()
    # and a file that cannot be created is reported like --debug's
    with pytest.raises(pp.PolypolishError) as e:
        ctx.polish_files(fa, sams, changes=tmp_path / "no" / "such" / "dir.tsv")
    assert e.value.msg == 'unable to create "%s"' % (tmp_path / "no" / "such" / "dir.tsv")


def test_cli_debug_and_changes_together(oracle, tmp_path):
    exe = os.path.join(ROOT, "build", "polypolish")
    syn = api.Synth(seed=4, contig_len=30_000, depth=40, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, min_depth=4)
    dbg, chg = tmp_path / "debug.tsv", tmp_path / "changes.tsv"
    r = subprocess.run([exe, "polish", "--min_depth", "4", "--debug", str(dbg), "--changes", str(chg), fa] + sams, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"]
    assert dbg.read_bytes() == exp["debug_tsv"]
    assert chg.read_bytes() == changed_rows(exp["debug_tsv"])
    r = subprocess.run([exe, "polish", "--changes", str(tmp_path / "no" / "x.tsv"), fa] + sams, capture_output=True)
    assert r.returncode == 1 and b'Error: unable to create "' in r.stderr


def test_changes_full_size(ctx, oracle):
    """BASELINE config 2 (5 Mbp x 100x): the rows are the oracle's changed debug rows, and as many as the log's changed count."""
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_chg_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        syn = api.Synth(seed=2, contig_len=5_000_000, depth=100)
        fa, sams = syn.write(d)
        exp = oracle.polish(fa, sams, debug=True)
        out = os.path.join(d, "changes.tsv")
        r = subprocess.run([os.path.join(ROOT, "build", "polypolish"), "polish", "--changes", out, fa] + sams, capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
        assert r.stdout == exp["fasta"]
        rows = open(out, "rb").read()
        assert rows == changed_rows(exp["debug_tsv"])
        logged = sum(int(x.split()[0].replace(b",", b"")) for x in r.stderr.split(b"\n") if b"changed (" in x)
        assert n_rows(rows) == logged == sum(exp["changed"]) > 0
    finally:
        shutil.rmtree(d, ignore_errors=True)
