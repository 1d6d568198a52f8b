"""The VCF (`polish --vcf`) on the GPU: the file is the model's (tests/vcfgen.py) from the oracle's --debug TSV, byte for byte, the
records applied to the draft give the FASTA the call returned, and that FASTA is the oracle's - whichever loader, context count or
entry point wrote it."""
import os
import shutil
import subprocess
import tempfile

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import endgen, indelgen, vcfgen
from tests.test_vcf_cpu import PARITY_SEEDS, fuzz_case

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


def check(fa, got_fasta, vcf_bytes, exp):
    """The three promises: the oracle's FASTA, the model's VCF, and the VCF rebuilding the FASTA."""
    assert got_fasta == exp["fasta"]
    assert vcf_bytes == vcfgen.vcf_from_debug(fa, exp["debug_tsv"])
    assert [s for _, s in vcfgen.apply_vcf(fa, vcf_bytes)] == [s for _, s in vcfgen.read_fasta(got_fasta)]


@pytest.mark.parametrize("parser", [0, 1], ids=["device", "host"])
@pytest.mark.parametrize("seed", PARITY_SEEDS)
def test_vcf_parity(ctx, oracle, tmp_path, seed, parser):
    """The --debug parity seeds (4-bit and 8-bit pools, insertions, IUPAC and '-' drafts, deep multi-maps), both SAM parsers."""
    case = fuzz_case(seed)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    out = tmp_path / "edits.vcf"
    ctx.set_parser(parser)
    try:
        got = ctx.polish_files(fa, sams, vcf=out, **case.opts)
    finally:
        ctx.set_parser(0)
    check(fa, got, out.read_bytes(), exp)


CASES = dict([("vcfgen-" + n, f) for n, f in vcfgen.CASES.items()] +
             [("indel-E", lambda: indelgen.edges(21)), ("indel-Q", lambda: indelgen.queue_general(22)),
              ("ends-E", lambda: endgen.edges(41)), ("ends-E8", lambda: endgen.edges(41, eight_bit=True)),
              ("ends-P", lambda: endgen.past_end(42))])


@pytest.mark.parametrize("name", list(CASES))
def test_vcf_cases(ctx, oracle, tmp_path, name):
    case = CASES[name]()
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    out = tmp_path / "edits.vcf"
    check(fa, ctx.polish_files(fa, sams, vcf=out, **case.opts), out.read_bytes(), exp)
    if name.startswith("vcfgen-"):
        vcfgen.check_claims(case, exp["debug_tsv"], out.read_bytes())


def test_vcf_without_sam_files(ctx, oracle, tmp_path):
    """No alignments: nothing changes, and the only records are the draft's '-' runs (vcfgen's whole-contig draft has a contig of
    '-' alone, fuzz seed 104's draft has '-' among its bases)."""
    for name, case in (("whole", vcfgen.whole_contig()), ("fuzz104", fuzz_case(104))):
        d = tmp_path / name
        d.mkdir()
        fa, _ = case.write(d)
        exp = oracle.polish(fa, [], debug=True)
        out = d / "edits.vcf"
        check(fa, ctx.polish_files(fa, [], vcf=out), out.read_bytes(), exp)
        recs = vcfgen.records_of(out.read_bytes())
        assert recs and all("-" in r[2] for r in recs)
        assert b"CHANGED=0\n" in out.read_bytes() and b"CHANGED=1" not in out.read_bytes()


def test_vcf_contexts(ctx, oracle, tmp_path):
    """Every context reports the change rows of its own contigs; 1, 2, 3 and 8 contexts through both parsers write the same bytes."""
    syn = api.Synth(seed=9, n_contigs=8, contig_len=12_000, depth=50, draft_error_rate=2e-3)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True)
    one = tmp_path / "one.vcf"
    check(fa, api.polish_files_multi(fa, sams, devices=[0], vcf=one), one.read_bytes(), exp)
    assert len(vcfgen.records_of(one.read_bytes())) > 8
    for n in (2, 3, 8):
        for parser in (0, 1):
            out = tmp_path / ("multi%d_%d.vcf" % (n, parser))
            assert api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser, vcf=out) == exp["fasta"]
            assert out.read_bytes() == one.read_bytes(), (n, parser)


@pytest.mark.parametrize("n_ctx,parser", [(1, 0), (2, 0), (3, 0), (2, 1)], ids=["1", "2", "3", "2-two-step"])
def test_vcf_filter_polish(oracle, tmp_path, n_ctx, parser):
    """filter + polish in one call: the VCF of the oracle's `filter`, then `polish --debug` of its output.  With host parsing the
    call takes the two-step path through temporary files."""
    syn = api.Synth(seed=5, n_contigs=3, contig_len=30_000, depth=60, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    ef = oracle.filter(sams[0], sams[1])
    f1, f2 = tmp_path / "f1.sam", tmp_path / "f2.sam"
    f1.write_bytes(ef["out1"])
    f2.write_bytes(ef["out2"])
    exp = oracle.polish(fa, [f1, f2], debug=True)
    out = tmp_path / "edits.vcf"
    got = api.filter_polish_files_multi(fa, sams[0], sams[1], devices=[0] * n_ctx, parser=parser, vcf=out)
    check(fa, got, out.read_bytes(), exp)


def test_vcf_cli(oracle, tmp_path):
    """--debug, --changes, --status-bed and --vcf together: each report is the one its flag writes alone; --vcf=FILE; and the
    file-creation error."""
    syn = api.Synth(seed=4, n_contigs=2, contig_len=30_000, depth=40, draft_error_rate=1e-3)
    fa, sams = syn.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, min_depth=4)
    flags = {"--debug": "debug.tsv", "--changes": "changes.tsv", "--status-bed": "status.bed", "--vcf": "edits.vcf"}
    both = []
    for f, n in flags.items():
        both += [f, str(tmp_path / ("all_" + n))]
    r = subprocess.run([EXE, "polish", "--min_depth", "4"] + both + [fa] + sams, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    check(fa, r.stdout, (tmp_path / "all_edits.vcf").read_bytes(), exp)
    for f, n in flags.items():
        one = subprocess.run([EXE, "polish", "--min_depth", "4", f, str(tmp_path / ("one_" + n)), fa] + sams, capture_output=True)
        assert one.returncode == 0 and one.stdout == r.stdout, f
        assert (tmp_path / ("one_" + n)).read_bytes() == (tmp_path / ("all_" + n)).read_bytes(), f
    r2 = subprocess.run([EXE, "polish", "--vcf=" + str(tmp_path / "eq.vcf"), "-d4", fa] + sams, capture_output=True)
    assert r2.returncode == 0 and r2.stdout == exp["fasta"]
    assert (tmp_path / "eq.vcf").read_bytes() == (tmp_path / "all_edits.vcf").read_bytes()
    bad = str(tmp_path / "no" / "x.vcf")
    r = subprocess.run([EXE, "polish", "--vcf", bad, fa] + sams, capture_output=True)
    assert r.returncode == 1 and r.stdout == b"" and r.stderr.endswith(b'Error: unable to create "%s"\n' % bad.encode())
    with pytest.raises(pp.PolypolishError) as e:
        pp.polish(fa, sams, vcf=tmp_path / "no" / "y.vcf")
    assert e.value.msg == 'unable to create "%s"' % (tmp_path / "no" / "y.vcf")


def test_vcf_full_size(oracle):
    """BASELINE config 2 (5 Mbp x 100x): the VCF is the model's from the oracle's TSV and rebuilds the FASTA."""
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_vcf_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        syn = api.Synth(seed=2, contig_len=5_000_000, depth=100)
        fa, sams = syn.write(d)
        exp = oracle.polish(fa, sams, debug=True)
        out = os.path.join(d, "edits.vcf")
        r = subprocess.run([EXE, "polish", "--vcf", out, fa] + sams, capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
        got = open(out, "rb").read()
        check(fa, r.stdout, got, exp)
        changed = sum(int(x.split(b"CHANGED=")[1].split(b";")[0]) for x in got.split(b"\n") if b"CHANGED=" in x and not x.startswith(b"#"))
        assert 0 < changed <= sum(exp["changed"])           # (a run whose edits undo each other has no record)
    finally:
        shutil.rmtree(d, ignore_errors=True)
