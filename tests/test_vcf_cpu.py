"""`polish --vcf` without a GPU: the model of tests/vcfgen.py rebuilds the oracle's FASTA from the oracle's own --debug TSV, the C++
record builder (polypolish_b200/csrc/vcf_records.h, through tests/vcf_harness.cpp) writes the model's bytes from the same rows, and
the flag's argument errors are clap's."""
import ctypes as C
import os
import subprocess

import pytest

import polypolish_b200 as pp
from tests import endgen, fuzzgen, indelgen, vcfgen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")
PARITY_SEEDS = [100, 101, 104, 105, 300, 303]


def fuzz_case(seed):
    """The --debug parity seeds' shapes (tests/test_gpu_status.py): exotic drafts and reads on every fourth seed, deep multi-maps
    from 300 on."""
    kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
    return fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)


CASES = dict([("fuzz%d" % s, (lambda s=s: fuzz_case(s))) for s in PARITY_SEEDS + list(range(1, 41))] +
             [("indel-E", lambda: indelgen.edges(21)), ("indel-Q", lambda: indelgen.queue_general(22)),
              ("ends-E", lambda: endgen.edges(41)), ("ends-E8", lambda: endgen.edges(41, eight_bit=True)),
              ("ends-P", lambda: endgen.past_end(42))] +
             [("vcfgen-" + n, f) for n, f in vcfgen.CASES.items()])


@pytest.fixture(scope="session", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


@pytest.fixture(scope="module")
def H():
    out = os.path.join(ROOT, "build", "vcf_harness.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "vcf_harness.cpp")])
    h = C.CDLL(out)
    h.h_vcf.restype = C.c_size_t
    return h


def polished(fasta_bytes):
    return [s for _, s in vcfgen.read_fasta(fasta_bytes)]


def run_oracle(oracle, tmp_path, name):
    case = CASES[name]()
    fa, sams = case.write(tmp_path)
    return case, fa, sams, oracle.polish(fa, sams, debug=True, **case.opts)


@pytest.mark.parametrize("name", list(CASES))
def test_model_rebuilds_the_oracle_fasta(oracle, tmp_path, name):
    """apply_vcf(vcf_from_debug(draft, TSV)) is the oracle's polished FASTA; the vcfgen cases make what they claim."""
    case, fa, sams, exp = run_oracle(oracle, tmp_path, name)
    vcf = vcfgen.vcf_from_debug(fa, exp["debug_tsv"])
    assert [s for _, s in vcfgen.apply_vcf(fa, vcf)] == polished(exp["fasta"])
    if name.startswith("vcfgen-"):
        vcfgen.check_claims(case, exp["debug_tsv"], vcf)
        f = pp.load_fasta(fa)
        p = pp.pack_sams(f, sams)
        assert p.view.seq_bits == (8 if case.facts["eight_bit"] else 4)
        p.close()


def builder_bytes(H, fa, debug_tsv):
    """The C++ builder's file for this draft, fed the oracle's change rows as (pos, allele, depth, support)."""
    contigs = vcfgen.read_fasta(fa)
    rows = vcfgen.changed_rows(debug_tsv)
    first, pos, allele, depth, support = [0], [], [], [], []
    for n, _ in contigs:
        for p, (a, dtext, sup) in sorted(rows.get(n, {}).items()):
            pos.append(p); allele.append(a.encode("latin-1")); depth.append(float(dtext)); support.append(sup)
        first.append(len(pos))
    k, m = len(contigs), max(1, len(pos))
    names = (C.c_char_p * k)(*[n.encode("latin-1") for n, _ in contigs])
    drafts = (C.c_char_p * k)(*[s.encode("latin-1") for _, s in contigs])
    args = [k, names, drafts, (C.c_uint64 * k)(*[len(s) for _, s in contigs]), (C.c_uint64 * (k + 1))(*first),
            (C.c_uint64 * m)(*pos), (C.c_char_p * m)(*allele), (C.c_double * m)(*depth), (C.c_uint32 * m)(*support)]
    size = H.h_vcf(*args, None, C.c_size_t(0))
    buf = C.create_string_buffer(size)
    assert H.h_vcf(*args, buf, C.c_size_t(size)) == size
    return buf.raw


@pytest.mark.parametrize("name", list(CASES))
def test_builder_matches_the_model(H, oracle, tmp_path, name):
    _, fa, _, exp = run_oracle(oracle, tmp_path, name)
    assert builder_bytes(H, fa, exp["debug_tsv"]) == vcfgen.vcf_from_debug(fa, exp["debug_tsv"])


def test_model_rules_by_hand():
    """The rules on drafts small enough to check by eye (allele, depth text, support per changed position)."""
    ch = lambda *xs: {p: (a, "9.0", 9) for p, a in xs}   # noqa: E731
    rec = lambda *xs: ["t\t%d\t.\t%s\t%s\t.\tPASS\t%s\n" % x for x in xs]   # noqa: E731
    info = lambda n: "CHANGED=%d" % n + (";DEPTH=%s;SUPPORT=%s" % (",".join(["9.0"] * n), ",".join(["9"] * n)) if n else "")  # noqa: E731
    assert vcfgen.contig_records("t", "ACGTA", ch((1, "T"), (2, "A"))) == rec((2, "CG", "TA", info(2)))
    assert vcfgen.contig_records("t", "ACGTA", ch((1, "CTT"))) == rec((2, "C", "CTT", info(1)))
    assert vcfgen.contig_records("t", "ACGTA", ch((2, "-"))) == rec((2, "CG", "C", info(1)))
    assert vcfgen.contig_records("t", "ACGTA", ch((0, "-"))) == rec((1, "AC", "C", info(1)))
    assert vcfgen.contig_records("t", "ACGTA", ch((0, "-"), (2, "-"))) == rec((1, "ACG", "C", info(2)))
    assert vcfgen.contig_records("t", "ACGTA", ch((0, "-"), (3, "-"))) == rec((1, "AC", "C", info(1)), (3, "GT", "G", info(1)))
    assert vcfgen.contig_records("t", "ACGTA", ch((1, "CG"), (2, "-"))) == []
    assert vcfgen.contig_records("t", "A-GTA", {}) == rec((1, "A-", "A", info(0)))
    assert vcfgen.contig_records("t", "-CGTA", {}) == rec((1, "-C", "C", info(0)))
    assert vcfgen.contig_records("t", "-C-TA", {}) == rec((1, "-C-", "C", info(0)))
    assert vcfgen.contig_records("t", "---", {}) == rec((1, "---", "<DEL>", info(0)))
    assert vcfgen.contig_records("t", "AC", ch((0, "-"), (1, "-"))) == rec((1, "AC", "<DEL>", info(2)))
    assert vcfgen.contig_records("t", "A-GTA", ch((2, "T"))) == rec((2, "-G", "T", info(1)))
    assert vcfgen.contig_records("t", "ACGT-", ch((4, "G"))) == rec((5, "-", "G", info(1)))


def test_apply_refuses_bad_records(tmp_path):
    fa = tmp_path / "d.fa"
    fa.write_bytes(b">t\nACGTA\n")
    head = vcfgen.header([("t", "ACGTA")])
    ok = head + "t\t2\t.\tCG\tTA\t.\tPASS\tCHANGED=0\n"
    assert vcfgen.apply_vcf(fa, ok.encode()) == [("t", "ATATA")]
    for body in ("t\t2\t.\tCG\tCG\t.\tPASS\tCHANGED=0\n",                                              # ALT == REF
                 "t\t2\t.\tGG\tTA\t.\tPASS\tCHANGED=0\n",                                              # REF not the draft
                 "t\t2\t.\tCG\tT\t.\tPASS\tCHANGED=0\nt\t3\t.\tG\tT\t.\tPASS\tCHANGED=0\n",             # overlap
                 "t\t3\t.\tG\tT\t.\tPASS\tCHANGED=0\nt\t2\t.\tC\tT\t.\tPASS\tCHANGED=0\n"):            # out of order
        with pytest.raises(AssertionError):
            vcfgen.apply_vcf(fa, (head + body).encode())


@pytest.mark.parametrize("args,msg", [
    (["polish", "--vcf"], "a value is required for '--vcf <FILE>' but none was supplied"),
    (["polish", "a.fa", "--vcf"], "a value is required for '--vcf <FILE>' but none was supplied"),
    (["filter-polish", "--in1", "a", "--in2", "b", "a.fa", "--vcf"], "a value is required for '--vcf <FILE>' but none was supplied"),
    # accepted, also as --vcf=FILE: the next error is the missing positional
    (["polish", "--vcf", "v.vcf"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["polish", "--vcf=v.vcf"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["filter-polish", "--vcf=v.vcf", "--gpu-count", "2"],
     "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["filter", "--vcf", "v.vcf"], "unexpected argument '--vcf' found"),
    (["filter", "--vcf=v.vcf"], "unexpected argument '--vcf' found"),
])
def test_vcf_usage_errors(args, msg):
    r = subprocess.run([EXE] + args, capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", f"error: {msg}\n\nFor more information, try '--help'.\n")


def test_help_names_vcf():
    r = subprocess.run([EXE, "polish", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--vcf <FILE>" in r.stdout
    r = subprocess.run([EXE, "filter", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--vcf" not in r.stdout
