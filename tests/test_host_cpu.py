"""CPU-side checks (no GPU): the library loads and exports the whole ABI, and the host text layer (FASTA loader,
SAM packer, synthetic generator) behaves like the reference's text handling as restated by the oracle."""
import gzip
import os
import re

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import fuzzgen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="session", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def test_abi_symbols_exported():
    """Every function include/pp_abi.h declares is exported by the shared library."""
    hdr = open(os.path.join(ROOT, "include", "pp_abi.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = sorted(set(re.findall(r"\b(pp_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) > 25
    L = pp.lib()
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    # ... and the other way round: no C-linkage pp_* entry point that the header does not declare
    import subprocess
    out = subprocess.run(["nm", "-D", "--defined-only", pp.lib()._name], capture_output=True, text=True, check=True).stdout
    exported = sorted({ln.split()[2] for ln in out.splitlines() if len(ln.split()) == 3 and ln.split()[1] == "T" and ln.split()[2].startswith("pp_")})
    undeclared = [n for n in exported if n not in names]
    assert not undeclared, undeclared


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    with pytest.raises(pp.PolypolishError):
        pp.Context(0)
    with pytest.raises(pp.PolypolishError):
        pp.polish("x.fasta", ["y.sam"])


FASTA_TXT = ">seq_1 123 456\nACGAT\n>seq_2 abc\nGGTA\n>seq_3\nCTCGCATCAG\n"
FASTA_EXP = [("seq_1", "123 456", "ACGAT"), ("seq_2", "abc", "GGTA"), ("seq_3", "", "CTCGCATCAG")]


def test_fasta_kat(tmp_path):   # misc.rs:246-267
    p = tmp_path / "a.fasta"
    p.write_text(FASTA_TXT)
    assert pp.load_fasta(p).records() == FASTA_EXP
    g = tmp_path / "a.fasta.gz"
    with gzip.open(g, "wt") as f:
        f.write(FASTA_TXT)
    assert pp.load_fasta(g).records() == FASTA_EXP


@pytest.mark.parametrize("text", [
    ">a\nACGT\n>a\nGG\n", "ACGT\n", ">\nACGT\n", ">a\n>b\nAC\n", "", "x", ">a desc\r\nacgtn\r\n\r\n>b\tq r\nAC\nGT",
    ">a x y\nAC\n", "\n\n>z\nA\n", ">a\n"])
def test_fasta_matches_oracle(oracle, tmp_path, text):
    p = tmp_path / "t.fasta"
    p.write_bytes(text.encode("utf-8"))
    try:
        exp = oracle.load_fasta(p)
    except Exception as e:
        with pytest.raises(pp.PolypolishError) as ei:
            pp.load_fasta(p)
        assert ei.value.msg == e.msg
        return
    assert [tuple(r) for r in pp.load_fasta(p).records()] == [tuple(r) for r in exp]


def _pack(tmp_path, fasta_text, sam_texts, careful=False):
    fa = tmp_path / "a.fasta"
    fa.write_text(fasta_text)
    f = pp.load_fasta(fa)
    p = api.Packed(f, careful)
    for i, t in enumerate(sam_texts):
        s = tmp_path / f"s{i}.sam"
        s.write_text(t)
        p.add_file(s)
    p.finish()
    return p


def test_pack_fields(tmp_path):
    sam = ("@HD\tVN:1\n"
           "r1\t0\tc1\t3\t60\t4M1I2M1D3M\t*\t0\t0\tacgtACGTNN\tIIIIIIIIII\tAS:i:3\tNM:i:2\tNM:i:5\n"
           "r1\t272\tc2\t1\t0\t10M\t*\t0\t0\t*\t*\tNM:i:0\tzp:z:FAIL\n"
           "r1\t4\t*\t0\t0\t*\t*\t0\t0\tAC\tII\n"
           "r1\t256\tc1\t0\t0\t0M10=\t*\t0\t0\t*\t*\tNM:i:1\n"
           "\n"
           "r2\t16\tzz\t7\t0\t3S7M\t*\t0\t0\tGGGGGGGGGG\t*\tNM:i:0\n")
    p = _pack(tmp_path, ">c1\nAAAAAAAAAAAAAAAAAAAA\n>c2\nCCCCCCCCCCCCCCCCCCCC\n", [sam])
    a = p.arrays()
    assert a["seq_bits"] == 4 and a["n_reads"] == 2
    assert a["contig"].tolist() == [0, 1, 0, 0xFFFFFFFF]
    assert a["ref_start"].tolist() == [2, 0, 0, 6]
    assert a["read_id"].tolist() == [0, 0, 0, 1]
    assert a["nm"].tolist() == [5, 0, 1, 0]                   # last NM wins (alignment.rs:68-71)
    assert a["n_cigar"].tolist() == [5, 1, 1, 2]              # zero-length op dropped
    fl = a["flags"].tolist()
    assert fl[0] == 0 and fl[1] == (api_flag("REVERSE") | api_flag("ZPFAIL") | api_flag("SEQSTAR") | api_flag("RC"))
    assert fl[2] == api_flag("SEQSTAR") and fl[3] == api_flag("REVERSE")
    assert a["seq_off"].tolist()[:3] == [0, 0, 0] and a["seq_len"].tolist() == [10, 10, 10, 10]
    ops = a["cigar_ops"].tolist()
    assert ops[:5] == [(4 << 4) | 0, (1 << 4) | 1, (2 << 4) | 0, (1 << 4) | 2, (3 << 4) | 0]
    nib = a["seq_pool"][:5].tolist()          # acgtACGTNN -> 1,2,4,8,1,2,4,8,15,15 (low nibble first)
    assert nib == [0x21, 0x84, 0x21, 0x84, 0xFF]
    assert p.read_name(3) == "r2"


def api_flag(n):
    return {"REVERSE": 1, "ZPFAIL": 2, "SEQSTAR": 4, "RC": 8, "NOSEQ": 16}[n]


BAD_SAMS = [
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\n",                                   # too few columns
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\n",                             # missing NM
    "r1\t0\tc1\t1\t60\t4Q\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",                     # invalid CIGAR
    "r1\t4\tc1\t1\t60\t4MM\t*\t0\t0\tACGT\tIIII\n",                            # invalid CIGAR on an unaligned line
    "@HD\n\nr1\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\tIIII\n",                          # no alignments
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\t*\t*\tNM:i:0\n",                           # no sequence in group
]


@pytest.mark.parametrize("sam", BAD_SAMS)
def test_pack_errors_match_oracle(oracle, tmp_path, sam):
    fa = tmp_path / "a.fasta"
    fa.write_text(">c1\nAAAAAAAAAAAAAAAAAAAA\n")
    s = tmp_path / "s0.sam"
    s.write_text(sam)
    with pytest.raises(Exception) as eo:
        oracle.polish(fa, [s])
    f = pp.load_fasta(fa)
    p = api.Packed(f, False)
    with pytest.raises(pp.PolypolishError) as ei:
        p.add_file(s)
        p.finish()
    assert ei.value.msg == eo.value.msg


def test_pack_eight_bit_fallback(tmp_path):
    sam = "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tAC.T\tIIII\tNM:i:0\nr2\t0\tc1\t1\t60\t4M\t*\t0\t0\tacgu\tIIII\tNM:i:0\n"
    p = _pack(tmp_path, ">c1\nAAAAAAAAAAAAAAAAAAAA\n", [sam])
    a = p.arrays()
    assert a["seq_bits"] == 8
    assert bytes(a["seq_pool"][:4]) == b"AC.T" and bytes(a["seq_pool"][32:36]) == b"ACGU"
    assert a["seq_off"].tolist() == [0, 1]


def test_pack_counts_match_oracle_on_fuzz(oracle, tmp_path):
    for seed in range(12):
        case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0)
        d = tmp_path / f"c{seed}"
        d.mkdir()
        fa, sams = case.write(d)
        r = oracle.polish(fa, sams, **case.opts)
        p = pp.pack_sams(pp.load_fasta(fa), sams, careful=case.opts["careful"])
        assert p.view.n_aln == r["alignment_total"]


def test_synth_deterministic_and_stream_equals_file(tmp_path):
    s1 = api.Synth(seed=7, contig_len=20000, depth=30, n_contigs=2)
    s2 = api.Synth(seed=7, contig_len=20000, depth=30, n_contigs=2)
    d1, d2 = tmp_path / "a", tmp_path / "b"
    d1.mkdir(); d2.mkdir()
    fa1, sams1 = s1.write(d1)
    fa2, sams2 = s2.write(d2)
    assert open(fa1, "rb").read() == open(fa2, "rb").read()
    for x, y in zip(sams1, sams2):
        assert open(x, "rb").read() == open(y, "rb").read()
    f1 = pp.load_fasta(fa1)
    p1, p2 = pp.pack_sams(f1, sams1), s1.pack()      # keep the owners alive: arrays() are views
    a1, a2 = p1.arrays(), p2.arrays()
    for k, v in a1.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, a2[k]), k
        else:
            assert v == a2[k], k
    # mates share names and order
    n1 = [l.split("\t")[0] for l in open(sams1[0]) if not l.startswith("@")]
    n2 = [l.split("\t")[0] for l in open(sams1[1]) if not l.startswith("@")]
    assert list(dict.fromkeys(n1)) == list(dict.fromkeys(n2))


def _pack_with(fa, sams, threads, chunk, careful=False):
    f = pp.load_fasta(fa)
    p = api.Packed(f, careful)
    p.set_threads(threads, chunk)
    for s in sams:
        p.add_file(s)
    p.finish()
    return f, p


@pytest.mark.parametrize("seed", range(40, 56))
def test_parallel_pack_equals_sequential(oracle, tmp_path, seed):
    """The multi-threaded file parser (chunks of ~2 KB here, so nearly every read group straddles a seam somewhere)
    must give exactly the sequential arrays, and the same error text on bad input."""
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, multimap=0.6)
    fa, sams = case.write(tmp_path)
    careful = case.opts["careful"]
    f1, p1 = _pack_with(fa, sams, 1, 1 << 30, careful)
    f2, p2 = _pack_with(fa, sams, 4, 2048, careful)
    a1, a2 = p1.arrays(), p2.arrays()
    for k, v in a1.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, a2[k]), k
        else:
            assert v == a2[k], k
    for i in range(0, len(a1["contig"]), 17):
        assert p1.read_name(i) == p2.read_name(i)


@pytest.mark.parametrize("sam", BAD_SAMS)
def test_parallel_pack_errors(oracle, tmp_path, sam):
    fa = tmp_path / "a.fasta"
    fa.write_text(">c1\nAAAAAAAAAAAAAAAAAAAA\n")
    good = "".join(f"g{i}\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n" for i in range(200))
    s = tmp_path / "s0.sam"
    s.write_text(good + sam + good if "no alignments" not in sam and "@HD" not in sam else sam)
    with pytest.raises(Exception) as eo:
        oracle.polish(fa, [s])
    f = pp.load_fasta(fa)
    p = api.Packed(f, False)
    p.set_threads(4, 512)
    with pytest.raises(pp.PolypolishError) as ei:
        p.add_file(s)
        p.finish()
    assert ei.value.msg == eo.value.msg


def test_cli_help_and_version_need_no_gpu():
    """`polypolish -h`, `polypolish polish -h`, `polypolish filter -h`, `-V` (main.rs:23-109): clap-style help with every
    reference option and its default; none of them touches CUDA."""
    import subprocess
    import __graft_entry__ as g
    g.build()
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "polypolish")
    top = subprocess.run([exe, "--help"], capture_output=True, text=True)
    assert top.returncode == 0 and "Usage: polypolish <COMMAND>" in top.stdout and "filter" in top.stdout and "polish" in top.stdout
    ph = subprocess.run([exe, "polish", "--help"], capture_output=True, text=True)
    assert ph.returncode == 0
    for frag in ["Usage: polypolish polish [OPTIONS] <ASSEMBLY> [SAM]...", "-i, --fraction_invalid <FRACTION_INVALID>", "[default: 0.2]",
                 "-v, --fraction_valid <FRACTION_VALID>", "[default: 0.5]", "-m, --max_errors <MAX_ERRORS>", "[default: 10]",
                 "-d, --min_depth <MIN_DEPTH>", "[default: 5]", "--careful", "--debug <DEBUG>"]:
        assert frag in ph.stdout, frag
    fh = subprocess.run([exe, "filter", "-h"], capture_output=True, text=True)
    assert fh.returncode == 0
    for frag in ["--in1 <IN1>", "--in2 <IN2>", "--out1 <OUT1>", "--out2 <OUT2>", "--orientation <ORIENTATION>", "[default: auto]",
                 "--low <LOW>", "[default: 0.1]", "--high <HIGH>", "[default: 99.9]"]:
        assert frag in fh.stdout, frag
    assert subprocess.run([exe, "-V"], capture_output=True, text=True).stdout.strip() == "Polypolish v0.6.1"
    bad = subprocess.run([exe, "polish", "--nope"], capture_output=True, text=True)
    assert bad.returncode == 2 and "unexpected argument '--nope'" in bad.stderr


CLI_USAGE_ERRORS = [
    # polish: <ASSEMBLY> required, positionals taken, --debug / --gpus accepted
    (["polish"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["polish", "--nope", "a.fa"], "unexpected argument '--nope' found"),
    (["polish", "--in1", "x", "a.fa"], "unexpected argument '--in1' found"),
    (["polish", "a.fa", "-m"], "a value is required for '--max_errors' but none was supplied"),
    (["polish", "a.fa", "--debug"], "a value is required for '--debug <DEBUG>' but none was supplied"),
    (["polish", "-i", "x", "a.fa"], "invalid value 'x' for '--fraction_invalid <FRACTION_INVALID>': invalid float literal"),
    (["polish", "-v=1e", "a.fa"], "invalid value '1e' for '--fraction_valid <FRACTION_VALID>': invalid float literal"),
    (["polish", "-m", "x", "a.fa"], "invalid value 'x' for '--max_errors <MAX_ERRORS>'"),
    (["polish", "-d", "-1", "a.fa"], "invalid value '-1' for '--min_depth <MIN_DEPTH>': invalid digit found in string"),
    (["polish", "--gpus", "x", "a.fa"], "invalid value 'x' for '--gpus'"),
    (["polish", "--device=4294967296", "a.fa"], "invalid value '4294967296' for '--device'"),
    # filter: no positionals, no --gpus, no polish options
    (["filter", "--in1", "a"], "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  --out1 <OUT1>\n  --out2 <OUT2>"),
    (["filter", "--nope"], "unexpected argument '--nope' found"),
    (["filter", "--gpus", "2"], "unexpected argument '--gpus' found"),
    (["filter", "-m5"], "unexpected argument '-m5' found"),
    (["filter", "--in1"], "a value is required for '--in1 <IN1>' but none was supplied"),
    (["filter", "--low", "x"], "invalid value 'x' for '--low <LOW>': invalid float literal"),
    (["filter", "--high="], "invalid value '' for '--high <HIGH>': invalid float literal"),
    (["filter", "--device", "x"], "invalid value 'x' for '--device'"),
    (["filter", "pos"], "unexpected argument 'pos' found"),
    (["filter", "--", "--in1"], "unexpected argument '--in1' found"),
    (["filter", "--quiet=1"], "unexpected argument '1' found"),
    # filter-polish: options of both, one <ASSEMBLY>, no -V / --debug / --gpus
    (["filter-polish", "--in1", "a", "--in2", "b"], "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["filter-polish", "a.fa"], "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["filter-polish", "--nope", "a.fa"], "unexpected argument '--nope' found"),
    (["filter-polish", "-V"], "unexpected argument '-V' found"),
    (["filter-polish", "--debug", "x", "a.fa"], "unexpected argument '--debug' found"),
    (["filter-polish", "--gpus", "2", "a.fa"], "unexpected argument '--gpus' found"),
    (["filter-polish", "a.fa", "--low"], "a value is required for '--low' but none was supplied"),
    (["filter-polish", "a.fa", "--orientation"], "a value is required for '--orientation <ORIENTATION>' but none was supplied"),
    (["filter-polish", "-v", "abc", "a.fa"], "invalid value 'abc' for '--fraction_valid <FRACTION_VALID>': invalid float literal"),
    (["filter-polish", "--high", "9x", "a.fa"], "invalid value '9x' for '--high <HIGH>': invalid float literal"),
    (["filter-polish", "-d", "x", "a.fa"], "invalid value 'x' for '--min_depth <MIN_DEPTH>'"),
    (["filter-polish", "--device", "-2", "a.fa"], "invalid value '-2' for '--device': invalid digit found in string"),
    (["frobnicate"], "unrecognized subcommand 'frobnicate'"),
]


def test_cli_usage_errors_need_no_gpu():
    """Every subcommand's argument errors, word for word with clap's exit code 2, and the `filter-polish` help: all of them are
    decided before a GPU context is created."""
    import subprocess
    exe = os.path.join(ROOT, "build", "polypolish")
    for args, msg in CLI_USAGE_ERRORS:
        r = subprocess.run([exe] + args, capture_output=True, text=True)
        assert (r.returncode, r.stdout, r.stderr) == (2, "", f"error: {msg}\n\nFor more information, try '--help'.\n"), args
    for flag in ("-h", "--help"):
        r = subprocess.run([exe, "filter-polish", flag], capture_output=True, text=True)
        assert (r.returncode, r.stderr) == (0, "")
        assert r.stdout == ("filter paired-end alignments based on insert size, then polish the assembly with the filtered alignments "
                            "(one pass, H100 build only)\n\nUsage: polypolish filter-polish [OPTIONS] --in1 <IN1> --in2 <IN2> <ASSEMBLY>\n\n"
                            "Options: those of `filter` (--out1 / --out2 optional: written only when given) and of `polish` (except --debug)\n")


@pytest.mark.parametrize("seed", range(6))
def test_sam_split_ranges_cut_between_read_groups(tmp_path, seed):
    """pp_sam_split_ranges (multi-GPU ingestion): every cut is a line start, and no read group as the reference forms them
    (tests/rangegen.py ref_groups) has aligned records on both sides of a cut."""
    import ctypes as C
    import random
    from polypolish_b200 import api
    from tests import rangegen
    rng = random.Random(seed)
    lines = ["@HD\tVN:1.6", "@SQ\tSN:c1\tLN:1000"] if seed % 2 == 0 else []
    for r in range(rng.randint(1, 400)):
        for _ in range(rng.choice([1, 1, 1, 2, 3, 8, 40] if seed != 3 else [200])):
            lines.append("read%d\t0\tc1\t%d\t60\t10M\t*\t0\t0\t%s\t*" % (r, rng.randint(1, 900), "ACGT" * rng.randint(1, 30)))
    text = "\n".join(lines) + ("\n" if seed != 5 else "")
    p = tmp_path / "x.sam"
    p.write_text(text)
    data = text.encode()
    L = api.lib()
    L.pp_sam_split_ranges.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_uint64)]
    for n in (1, 2, 3, 8, 32):
        cuts = (C.c_uint64 * (n + 1))()
        assert L.pp_sam_split_ranges(str(p).encode(), n, cuts) == 0
        cuts = list(cuts)
        assert cuts[0] == 0 and cuts[-1] == len(data) and cuts == sorted(cuts)
        for c in cuts[1:-1]:
            assert c == len(data) or data[c - 1:c] == b"\n"
        assert rangegen.split_groups(data, cuts) == [], n
    assert L.pp_sam_split_ranges(str(tmp_path / "missing.sam").encode(), 2, (C.c_uint64 * 3)()) != 0


def test_packer_reads_a_fifo_once(tmp_path):
    """pp_pack_add_sam_file maps regular files and streams anything else: a named pipe is opened exactly once (a second open
    would block for ever, or break the writer's pipe) and gives the same arrays as the file."""
    import threading
    syn = api.Synth(seed=3, n_contigs=1, contig_len=20_000, depth=20.0)
    fa, sams = syn.write(str(tmp_path))
    f = api.Fasta(fa)
    ref = api.pack_sams(f, sams)
    fifo = str(tmp_path / "reads.fifo")
    os.mkfifo(fifo)

    def writer():
        with open(fifo, "wb") as o:
            o.write(open(sams[0], "rb").read())
    t = threading.Thread(target=writer)
    t.start()
    p = api.Packed(f, False)
    p.add_file(fifo)
    t.join(timeout=30)
    assert not t.is_alive()
    p.add_file(sams[1])
    p.finish()
    a, b = api.view_arrays(ref.view), api.view_arrays(p.view)
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k]), k
