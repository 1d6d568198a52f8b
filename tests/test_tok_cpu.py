"""The device SAM tokeniser's per-item logic (tok_line.h) run on the CPU (tests/tok_harness.cpp), against the host packer.

The kernels of tok_kernels.cu call exactly these functions, one item per thread; here they run item by item in the same
pipeline order, so everything but the CUDA plumbing (line index, scans, launches) is covered without a GPU.
The GPU tests (test_gpu_tok.py) then compare the real device arrays with the host packer's."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from tests import fuzzgen
import polypolish_b200 as pp
from polypolish_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PP_OK, PP_TOK_HOST, PP_TOK_NEED8 = 0, 1, 2


@pytest.fixture(scope="module")
def H():
    out = os.path.join(ROOT, "build", "tok_harness.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "tok_harness.cpp")])
    return C.CDLL(out)


def tok_cpu(H, names, texts, careful=False, bits=4):
    """Runs the harness over the texts in order. Returns (rc, arrays)."""
    total = sum(len(t) for t in texts)
    cap_aln = total // 20 + 16
    cap_ops = total // 2 + 16
    cap_seq = total * (1 if bits == 4 else 2) + 64 * (cap_aln + 1)
    a = dict(contig=np.zeros(cap_aln, np.uint32), ref_start=np.zeros(cap_aln, np.uint32), read_id=np.zeros(cap_aln, np.uint32),
             seq_off=np.zeros(cap_aln, np.uint32), seq_len=np.zeros(cap_aln, np.uint16), cigar_off=np.zeros(cap_aln, np.uint32),
             n_cigar=np.zeros(cap_aln, np.uint16), nm=np.zeros(cap_aln, np.uint32), flags=np.zeros(cap_aln, np.uint8),
             cigar_ops=np.zeros(cap_ops, np.uint32), seq_pool=np.full(cap_seq, 0xEE, np.uint8))
    counts = (C.c_uint64 * 6)(0, 0, 0, 0, 0, 0)
    cn = (C.c_char_p * len(names))(*[n.encode("latin-1") for n in names])
    H.tok_cpu.restype = C.c_int
    order = ["contig", "ref_start", "read_id", "seq_off", "seq_len", "cigar_off", "n_cigar", "nm", "flags", "cigar_ops", "seq_pool"]
    for t in texts:
        rc = H.tok_cpu(C.c_char_p(t), C.c_uint64(len(t)), cn, C.c_uint32(len(names)), C.c_int(int(careful)), C.c_int(bits),
                       C.c_uint64(cap_aln), C.c_uint64(cap_ops), C.c_uint64(cap_seq),
                       *[a[k].ctypes.data_as(C.c_void_p) for k in order], counts)
        if rc != PP_OK:
            return rc, None, list(counts)
    n, no, nb, nr = counts[0], counts[1], counts[2], counts[3]
    out = {k: a[k][:n].copy() for k in order[:9]}
    out["cigar_ops"] = a["cigar_ops"][:no].copy()
    out["seq_pool"] = a["seq_pool"][:nb * (16 if bits == 4 else 32)].copy()
    out["n_reads"] = nr
    out["seq_bits"] = bits
    return PP_OK, out, list(counts)


def host_pack(tmp_path, fasta_text, texts, careful=False):
    fa = tmp_path / "a.fasta"
    fa.write_bytes(fasta_text if isinstance(fasta_text, bytes) else fasta_text.encode("latin-1"))
    f = pp.load_fasta(fa)
    p = api.Packed(f, careful)
    for i, t in enumerate(texts):
        p.add_text(t, f"s{i}.sam")
    p.finish()
    return f, p


def assert_same(dev, host):
    for k, v in host.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, dev[k]), k
        else:
            assert v == dev[k], k


@pytest.mark.parametrize("seed", range(60, 84))
def test_tok_logic_equals_host_packer_on_fuzz(H, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.0, multimap=0.5 if seed % 2 else 0.25)
    texts = [t.encode("latin-1") for t in case.sam_texts]
    careful = case.opts["careful"]
    f, p = host_pack(tmp_path, case.fasta_text, texts, careful)
    host = p.arrays()
    assert host["seq_bits"] == 4
    rc, dev, _ = tok_cpu(H, f.names, texts, careful, 4)
    assert rc == PP_OK
    assert_same(dev, host)


@pytest.mark.parametrize("seed", [200, 204, 208])
def test_tok_logic_eight_bit(H, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.5)
    texts = [t.encode("latin-1") for t in case.sam_texts]
    f, p = host_pack(tmp_path, case.fasta_text, texts, case.opts["careful"])
    host = p.arrays()
    rc4, _, _ = tok_cpu(H, f.names, texts, case.opts["careful"], 4)
    if host["seq_bits"] == 8:
        assert rc4 == PP_TOK_NEED8
    rc, dev, _ = tok_cpu(H, f.names, texts, case.opts["careful"], int(host["seq_bits"]))
    assert rc == PP_OK
    assert_same(dev, host)


FA = ">c1 first\nAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAA\n>c2\nCCCCCCCCCCCCCCCCCCCCCCCC\n>c10\nGGGGGGGGGGGG\n"
NAMES = ["c1", "c2", "c10"]


def line(name="r", flag=0, ref="c1", pos=1, cigar="4M", seq="ACGT", tags=("NM:i:0",), qual="IIII", mapq="60"):
    return "\t".join([name, str(flag), ref, str(pos), mapq, cigar, "*", "0", "0", seq, qual] + list(tags)) + "\n"


EDGE_TEXTS = [
    # headers, blank lines, CRLF, unaligned lines in the middle of a group, last line without newline
    "@HD\tVN:1.6\n\n" + line("a") + "\r\n" + line("a", 16, seq="*", qual="*").replace("\n", "\r\n") + line("u", 4, "*", 0, "*") + line("a", 0, "c2", 3, seq="*") + line("b", 16, "c10", 2)[:-1],
    # empty QNAME joins what follows; same-length different names; a name that is a prefix of the next
    line("") + line("x") + line("x") + line("y") + line("yy") + line("y") + line("") + line(""),
    # SEQ star before the source record; strands differ -> RC; source is reverse
    line("g", 0, seq="*", qual="*") + line("g", 16, seq="*", qual="*") + line("g", 16, "c2", 5, seq="ACGTACGTACGTACGTACGTACGTACGTACGTACG", cigar="35M") + line("g", 0, seq="*"),
    # tags: NM last wins, '+' sign, ZP:Z:fail any case, near misses, empty tag fields, a trailing tab
    line("t1", tags=("NM:i:3", "XS:i:1", "NM:i:+7")) + line("t2", tags=("zp:z:FAIL", "NM:i:1")) + line("t3", tags=("ZP:Z:failed", "NM:i:2", "ZP:Z:fai")) +
    line("t4", tags=("", "NM:i:4", "")) + line("t5", tags=("NM:i:5\t",)),
    # CIGAR shapes: zero-length ops vanish, every op letter, long numbers, '=' and 'X'
    line("c1r", cigar="0M4M0I", seq="ACGT") + line("c2r", cigar="1S2=1X1I1D1N1H1P", seq="ACGTA") + line("c3r", cigar="000004M", seq="ACGT") +
    line("c4r", cigar="268435455M", seq="ACGT"),
    # POS 0 stays 0; POS with '+'; unknown reference names (device leaves them to the polish step's error)
    line("p0", pos=0) + line("p1", pos="+5") + line("p2", ref="nope") + line("p3", ref="c1x") + line("p4", ref="c"),
    # sequences: empty SEQ field, lower case, every IUPAC code, 31/32/33/64/65 bases
    line("s0", seq="", cigar="1M") + line("s1", seq="acgtn", cigar="5M") + line("s2", seq="ACMGRSVTWYHKDBN", cigar="15M") +
    "".join(line(f"s{n}", seq=("ACGT" * 20)[:n], cigar=f"{n}M") for n in (31, 32, 33, 64, 65)),
]


@pytest.mark.parametrize("i", range(len(EDGE_TEXTS)))
@pytest.mark.parametrize("careful", [False, True])
def test_tok_logic_edge_texts(H, tmp_path, i, careful):
    t = EDGE_TEXTS[i].encode("latin-1")
    try:
        f, p = host_pack(tmp_path, FA, [t], careful)
    except pp.PolypolishError:
        rc, _, _ = tok_cpu(H, NAMES, [t], careful, 4)
        assert rc == PP_TOK_HOST
        return
    host = p.arrays()
    rc, dev, _ = tok_cpu(H, NAMES, [t], careful, int(host["seq_bits"]))
    assert rc == PP_OK
    assert_same(dev, host)


BAD_LINES = [
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\n",                        # too few columns
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\n",                  # missing NM
    "r1\t0\tc1\t1\t60\t4Q\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",          # invalid CIGAR
    "r1\t4\tc1\t1\t60\t4MM\t*\t0\t0\tACGT\tIIII\n",                 # invalid CIGAR on an unaligned line
    "r1\t0\tc1\t1\t60\t4\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",           # digits without an operation
    "r1\t0\tc1\t1\t60\t*\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",           # aligned with CIGAR *
    "r1\t0\tc1\t1\t60\t\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",            # aligned with empty CIGAR
    "r1\tx\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",          # FLAG not a number
    "r1\t4294967296\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",  # FLAG overflows u32
    "r1\t0\tc1\t-1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",         # POS negative
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:\n",           # NM without digits
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:1x\n",         # NM with junk
    "r1\t0\tc1\t1\t60\t268435456M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",  # operation longer than 2^28-1
    "r1\t0\tc1\t1\t60\t4294967296M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",  # operation length beyond u32
    "r1\t0\tc1\t1\t60\t4M\t*\t0\t0\t*\t*\tNM:i:0\n",                # group without sequence
    "r1\t0\tc1\t4294967297\t60\t4M\t*\t0\t0\tACGT\tIIII\tNM:i:0\n",  # start beyond 2^32
]


@pytest.mark.parametrize("bad", BAD_LINES)
def test_tok_logic_hands_bad_text_to_the_host(H, tmp_path, bad):
    good = "".join(line(f"g{i}") for i in range(30))
    t = (good + bad + good).encode("latin-1")
    with pytest.raises(pp.PolypolishError):
        host_pack(tmp_path, FA, [t])
    rc, _, counts = tok_cpu(H, NAMES, [t])
    assert rc == PP_TOK_HOST
    if "\t*\t*\tNM" not in bad:                # line-level problems are located exactly
        assert counts[5] == 30


def test_tok_logic_empty_and_header_only(H):
    assert tok_cpu(H, NAMES, [b""])[0] == PP_TOK_HOST
    assert tok_cpu(H, NAMES, [b"@HD\tVN:1\n\n"])[0] == PP_TOK_HOST
    assert tok_cpu(H, NAMES, [line("u", 4, "*", 0, "*").encode()])[0] == PP_TOK_HOST


def test_tok_logic_careful_group_without_sequence(H, tmp_path):
    """--careful drops multi-alignment reads before the sequence lookup (alignment.rs:277-279): no error, NOSEQ records."""
    t = (line("m", seq="*", qual="*") + line("m", 16, seq="*", qual="*") + line("n")).encode()
    f, p = host_pack(tmp_path, FA, [t], True)
    rc, dev, _ = tok_cpu(H, NAMES, [t], True, 4)
    assert rc == PP_OK
    assert_same(dev, p.arrays())
    assert tok_cpu(H, NAMES, [t], False, 4)[0] == PP_TOK_HOST


def test_tok_logic_random_bytes_never_disagree(H, tmp_path):
    """Mutated lines: wherever the harness says PP_OK the arrays equal the host packer's; wherever the host packer fails,
    the harness must have said PP_TOK_HOST (or NEED8, which ends in the host path too)."""
    rng = random.Random(5)
    base = [line(f"q{i // 2}", rng.choice([0, 16, 4, 256, 272] if i % 2 else [0, 16]), rng.choice(["c1", "c2", "c10", "zz"]), rng.randint(0, 30),
                 rng.choice(["4M", "2M1I1M", "1M1D3M", "2S2M", "4="]), rng.choice(["ACGT", "*", "acgn"] if i % 2 else ["ACGT", "acgn"]),
                 (f"NM:i:{rng.randint(0, 12)}",) + (("ZP:Z:fail",) if rng.random() < 0.1 else ())) for i in range(40)]
    alphabet = "\t\t\t0123456789MIDS=X*ACGTN:@+-\r zpZP\x08\x08\x01\x89\xff\x0a"   # \x08 = '\t' ^ 1: the word-wise tab search must stay exact
    n_ok = n_host = 0
    for trial in range(500):
        lines = list(base)
        for _ in range(rng.randint(1, 3)):
            j = rng.randrange(len(lines))
            s = list(lines[j])
            k = rng.randrange(len(s) - 1)
            op = rng.random()
            if op < 0.4:
                s[k] = rng.choice(alphabet)
            elif op < 0.7:
                del s[k]
            else:
                s.insert(k, rng.choice(alphabet))
            lines[j] = "".join(s)
        t = "".join(lines).encode("latin-1")
        try:
            f, p = host_pack(tmp_path, FA, [t])
            host = p.arrays()
        except pp.PolypolishError:
            host = None
        rc, dev, _ = tok_cpu(H, NAMES, [t], False, 4)
        if host is None:
            assert rc in (PP_TOK_HOST, PP_TOK_NEED8), t
            n_host += 1
        elif rc == PP_OK:
            assert host["seq_bits"] == 4
            assert_same(dev, host)
            n_ok += 1
        elif rc == PP_TOK_NEED8:
            assert host["seq_bits"] == 8
            rc8, dev8, _ = tok_cpu(H, NAMES, [t], False, 8)
            assert rc8 == PP_OK
            assert_same(dev8, host)
            n_ok += 1
        else:
            raise AssertionError(f"harness refused a text the host packer accepts: {t!r}")
    assert n_ok > 50 and n_host > 50


# ---- `polypolish filter`: the quick parse (parse_line_quick) against a Python model of load_alignments_one_file ---------
import re  # noqa: E402

CIGAR_TOKEN = re.compile(rb"\d+[MIDNSHP=X]")


def rust_parse_uint(b, maxv):
    if b.startswith(b"+"):
        b = b[1:]
    if not b or not b.isdigit() or not all(48 <= c <= 57 for c in b):
        return None
    v = int(b)
    return v if v <= maxv else None


def model_quick(line):
    """(kind, start, end, rev) for one line (bytes, no newline): filter.rs:122-137 + alignment.rs:102-149."""
    if line.startswith(b"@"):
        return (0, 0, 0, 0)
    f = line.split(b"\t")
    if len(f) < 11:
        return (2, 0, 0, 0)
    flag = rust_parse_uint(f[1], 0xFFFFFFFF)
    pos = rust_parse_uint(f[3], (1 << 64) - 1)
    if flag is None or pos is None:
        return (2, 0, 0, 0)
    if flag & 4:
        return (0, 0, 0, 0)
    start = pos - 1 if pos > 0 else 0
    end = start
    for m in CIGAR_TOKEN.finditer(f[5]):
        t = m.group()
        v = int(t[:-1])
        if v >= 1 << 64:
            return (2, 0, 0, 0)
        if t[-1:] in b"MDN=X":
            end = (end + v) & ((1 << 64) - 1)
    if end > 0xFFFFFFFE:
        return (2, 0, 0, 0)
    return (1, start & 0xFFFFFFFF, end, 1 if flag & 16 else 0)


def ftok_cpu(H, text, ref_hash=False):
    """The quick parse's columns per line; with ref_hash, the RNAME keys follow as a ninth array."""
    nl = text.count(b"\n") + 2
    kind = np.zeros(nl, np.uint8); rs = np.zeros(nl, np.uint32); re_ = np.zeros(nl, np.uint32); rev = np.zeros(nl, np.uint8)
    nlen = np.zeros(nl, np.uint32); rrel = np.zeros(nl, np.uint32); rlen = np.zeros(nl, np.uint32); nh = np.zeros(nl, np.uint64)
    rh = np.zeros(nl, np.uint64)
    n_out = C.c_uint64()
    H.ftok_cpu.restype = C.c_int
    rc = H.ftok_cpu(C.c_char_p(text), C.c_uint64(len(text)), C.c_uint64(nl),
                    *[a.ctypes.data_as(C.c_void_p) for a in (kind, rs, re_, rev, nlen, rrel, rlen, nh, rh)], C.byref(n_out))
    assert rc == 0
    n = n_out.value
    out = (kind[:n], rs[:n], re_[:n], rev[:n], nlen[:n], rrel[:n], rlen[:n], nh[:n])
    return out + (rh[:n],) if ref_hash else out


def split_lines(text):
    """str::lines(): split on \\n, strip one \\r before it, a final unterminated line is a line (and keeps its \\r)."""
    out = []
    parts = text.split(b"\n")
    for i, p in enumerate(parts):
        last = i == len(parts) - 1
        if last:
            if p:
                out.append(p)
        else:
            out.append(p[:-1] if p.endswith(b"\r") else p)
    return out


def test_ftok_quick_parse_matches_model(H):
    rng = random.Random(9)
    cigars = ["4M", "2M1I1M", "10M2D5M", "3S7M", "5=1X4=", "*", "", "12", "M", "4M5", "9999999999M", "4294967295M", "18446744073709551616M", "1M1N1H1P",
              "3Mjunk4D", "0M", "+4M", "4m"]
    flags = ["0", "16", "4", "20", "256", "272", "+16", "x", "", "4294967295", "4294967296", "-1"]
    poss = ["0", "1", "100", "+7", "4294967295", "4294967296", "18446744073709551615", "18446744073709551616", "a", ""]
    lines = ["@HD\tVN:1.6", "", "@", "\t", "a\tb"]
    for _ in range(600):
        n_extra = rng.choice([0, 0, 0, 1, 3])
        cols = [f"r{rng.randint(0, 50)}", rng.choice(flags), rng.choice(["c1", "c2", "", "*"]), rng.choice(poss), "60", rng.choice(cigars), "*", "0", "0",
                "ACGT", "IIII"] + ["NM:i:0"] * n_extra
        if rng.random() < 0.1:
            cols = cols[:rng.randint(1, 10)]
        lines.append("\t".join(cols))
    for ending in (b"\n", b"\r\n"):
        for final_newline in (True, False):
            text = ending.join(x.encode() for x in lines) + (ending if final_newline else b"")
            kind, rs, re_, rev, nlen, rrel, rlen, nh = ftok_cpu(H, text)
            want = split_lines(text)
            assert len(want) == len(kind)
            for i, ln in enumerate(want):
                k, s, e, r = model_quick(ln)
                assert kind[i] == k, (i, ln)
                if k == 1:
                    assert (rs[i], re_[i], rev[i]) == (s, e, r), (i, ln)
                    f = ln.split(b"\t")
                    assert nlen[i] == len(f[0]) and rlen[i] == len(f[2]) and ln[rrel[i]:rrel[i] + rlen[i]] == f[2]
    # equal names hash equal, different names (here) differ
    text = b"".join(("\t".join([nm, "0", "c1", "1", "60", "4M", "*", "0", "0", "ACGT", "IIII"]) + "\n").encode() for nm in ["a", "b", "a", "ab", ""])
    nh = ftok_cpu(H, text)[7]
    assert nh[0] == nh[2] and len({int(nh[0]), int(nh[1]), int(nh[3]), int(nh[4])}) == 4


# ---- upload-side QUAL stripping (tok_strip.h): the tokenised arrays must not notice -------------------------------------
def strip_cpu(H, text):
    out = C.create_string_buffer(len(text) + 1)
    H.strip_cpu.restype = C.c_uint64
    n = H.strip_cpu(C.c_char_p(text), C.c_uint64(len(text)), out)
    return out.raw[:n]


def test_strip_qual_keeps_everything_but_qual(H):
    rows = [line("a", qual="IIII"), line("b", qual="*"), line("c", qual=""), line("d", qual="I"), "@HD\tVN:1.6\n", "\n", "x\ty\n",
            line("e", qual="II", tags=()), line("f", qual="IIIIII", tags=()).replace("\n", "\r\n"), line("g", qual="!!!!", tags=("NM:i:1", "XX:Z:q\x08")),
            line("last", qual="ABCDEFG", tags=())[:-1]]
    text = "".join(rows).encode("latin-1")
    got = strip_cpu(H, text)
    want = []
    for r in rows:
        eol = "\r\n" if r.endswith("\r\n") else ("\n" if r.endswith("\n") else "")
        body = r[:len(r) - len(eol)]
        f = body.split("\t")
        if not body.startswith("@") and len(f) >= 11 and len(f[10]) >= 2:
            f[10] = "*"
            body = "\t".join(f)
        want.append(body + eol)
    assert got == "".join(want).encode("latin-1")
    assert len(got) <= len(text) and got.count(b"\n") == text.count(b"\n")


@pytest.mark.parametrize("seed", range(90, 102))
def test_stripped_text_tokenises_to_the_same_arrays(H, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 5 == 0 else 0.0, multimap=0.4)
    texts = [t.encode("latin-1") for t in case.sam_texts]
    if seed % 3 == 0:
        texts = [t.replace(b"\n", b"\r\n") for t in texts]
    if seed % 4 == 0:
        texts = [t[:-1] if t.endswith(b"\n") and not t.endswith(b"\r\n") else t for t in texts]
    careful = case.opts["careful"]
    f, p = host_pack(tmp_path, case.fasta_text, texts, careful)
    host = p.arrays()
    stripped = [strip_cpu(H, t) for t in texts]
    assert sum(map(len, stripped)) < 0.8 * sum(map(len, texts))
    rc, dev, _ = tok_cpu(H, f.names, stripped, careful, int(host["seq_bits"]))
    assert rc == PP_OK
    assert_same(dev, host)


def test_stripped_mutated_texts_agree_with_the_host_packer(H, tmp_path):
    """The stripping never turns a text the host packer rejects into one the tokeniser accepts, nor changes the arrays."""
    rng = random.Random(17)
    base = [line(f"q{i // 2}", rng.choice([0, 16, 4, 256, 272] if i % 2 else [0, 16]), rng.choice(["c1", "c2", "c10", "zz"]), rng.randint(0, 30),
                 rng.choice(["4M", "2M1I1M", "1M1D3M", "2S2M", "4="]), rng.choice(["ACGT", "*", "acgn"] if i % 2 else ["ACGT", "acgn"]),
                 (f"NM:i:{rng.randint(0, 12)}",) + (("ZP:Z:fail",) if rng.random() < 0.1 else ())) for i in range(30)]
    alphabet = "\t\t\t\t0123456789MIDS=X*ACGTN:@+-\r zpZP\x08\n"
    n_ok = 0
    for trial in range(400):
        lines = list(base)
        for _ in range(rng.randint(1, 3)):
            j = rng.randrange(len(lines))
            s = list(lines[j])
            k = rng.randrange(len(s) - 1)
            op = rng.random()
            if op < 0.4:
                s[k] = rng.choice(alphabet)
            elif op < 0.7:
                del s[k]
            else:
                s.insert(k, rng.choice(alphabet))
            lines[j] = "".join(s)
        t = "".join(lines).encode("latin-1")
        try:
            f, p = host_pack(tmp_path, FA, [t])
            host = p.arrays()
        except pp.PolypolishError:
            host = None
        rc, dev, _ = tok_cpu(H, NAMES, [strip_cpu(H, t)], False, 4)
        if host is None:
            assert rc in (PP_TOK_HOST, PP_TOK_NEED8), t
        elif rc == PP_OK:
            assert_same(dev, host)
            n_ok += 1
        else:
            assert rc == PP_TOK_NEED8 and host["seq_bits"] == 8, t
    assert n_ok > 50


def upload_emulate(H, text, S, look):
    out = C.create_string_buffer(len(text) + 1)
    last = C.c_uint8(10)
    sent = C.c_uint64()
    H.upload_emulate.restype = C.c_int
    rc = H.upload_emulate(C.c_char_p(text), C.c_uint64(len(text)), C.c_uint64(S), C.c_uint64(look), out, C.byref(last), C.byref(sent))
    return rc, out.raw[:len(text)], last.value, sent.value


@pytest.mark.parametrize("seed", range(110, 122))
@pytest.mark.parametrize("S,look", [(64, 512), (97, 300), (1000, 400), (4096, 4096)])
def test_stripping_upload_slices(H, tmp_path, seed, S, look):
    """Tiny slices, so that nearly every line straddles one: every byte of the device text is written exactly once, it has the size
    of the file, its last byte is the file's, and it tokenises to the host packer's arrays (the filler lines are skipped)."""
    case = fuzzgen.make_case(seed, exotic=0.0, multimap=0.4)
    texts = [t.encode("latin-1") for t in case.sam_texts]
    if seed % 3 == 0 and not any(b"\r" in t for t in texts):
        texts = [t.replace(b"\n", b"\r\n") for t in texts]
    if seed % 4 == 1 and not any(b"\r" in t for t in texts):
        texts = [t[:-1] for t in texts]
    careful = case.opts["careful"]
    f, p = host_pack(tmp_path, case.fasta_text, texts, careful)
    host = p.arrays()
    dev_texts = []
    for t in texts:
        rc, out, last, sent = upload_emulate(H, t, S, look)
        longest = max(len(x) for x in t.split(b"\n")) + 1
        if rc == 3:
            assert longest >= look - 1
            dev_texts.append(t)                       # the verbatim upload takes over
            continue
        assert rc == 0 and b"\xee" not in out and len(out) == len(t) and last == t[-1] and sent <= len(t)
        assert out.count(b"\n") >= t.count(b"\n")
        dev_texts.append(out)
    rc, dev, _ = tok_cpu(H, f.names, dev_texts, careful, int(host["seq_bits"]))
    assert rc == PP_OK
    assert_same(dev, host)
