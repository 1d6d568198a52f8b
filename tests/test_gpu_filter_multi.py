"""`filter` and `filter-polish` over several contexts (pp_filter_files_multi / pp_filter_polish_files_multi): every context filters a
byte range of both SAM files, the records meet on the context that owns their read name, the thresholds are reduced across
contexts.  Each case runs with 2, 3 and 8 contexts on one device (`devices=[0] * n`, so the whole suite runs on one H100) and is
compared, byte for byte, with the oracle and with the one-context call: both filtered SAM files, the log's numbers (pairs per
orientation, orientation, thresholds, pass / fail per file), and for the fused call the FASTA and the change report."""
import hashlib
import os
import pathlib
import random
import shutil
import subprocess
import tempfile
import threading

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api

pytestmark = pytest.mark.gpu

NS = (2, 3, 8)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctxs():
    import __graft_entry__ as g
    g.build()
    cs = [pp.Context(0) for _ in range(max(NS))]
    yield cs
    for c in cs:
        c.close()


def rec(name, flag, ref, pos, cigar="100M"):
    return "\t".join([name, str(flag), ref, str(pos), "60", cigar, "*", "0", "0", "ACGT", "IIII", "NM:i:0"])


FLAGS = {"fr": (0, 16), "rf": (16, 0), "ff": (0, 0), "rr": (16, 16)}


def pair_sams(seed, n_pairs=400, orient="fr", eol="\n", unterminated=False, bad_line_at=None):
    """Paired SAM text whose read names are spread over the byte ranges: file 1's lines are shuffled one by one (a name's
    alignments lie far apart), file 2's groups are shuffled; a read with its mate-1 record first in file 1 and its mate-2 record
    last in file 2; multi-mapped mates, mates in one file only, unaligned records, and pairs whose mates sit on different contigs
    at overlapping positions.  Range 0 of file 1 first meets contig c2 (headers name c2 first), later ranges meet c1 or c3 first."""
    rng = random.Random(seed)
    refs = ["c2", "c1", "c3"]
    fa, fb = FLAGS[orient]
    lines1, groups2 = [], []
    for i in range(n_pairs):
        name = f"r{i}"
        ref = rng.choice(refs)
        a = rng.randint(1, 90000)
        ins = max(150, int(rng.gauss(300, 8)))                 # narrow: many equal insert sizes, ranks fall on ties
        r1 = [rec(name, fa, ref, a, rng.choice(["100M", "50M2D50M", "40M3I57M", "5S95M"]))]
        r2 = [rec(name, fb, ref, a + ins - 100)]
        x = rng.random()
        if x < 0.2:
            r1 += [rec(name, 256 | rng.choice([0, 16]), rng.choice(refs), rng.randint(1, 90000)) for _ in range(rng.randint(1, 4))]
        elif x < 0.35:
            for _ in range(rng.randint(1, 3)):
                r1.append(rec(name, 256 | fa, ref, a + rng.choice([0, 1000, -50, 5])))
                r2.append(rec(name, 256 | fb, ref, a + ins - 100 + rng.choice([0, 1000, 3, 20000])))
        elif x < 0.42:
            r2 = []                                            # mate in one file only
        elif x < 0.47:
            r2 = [rec(name, 4, "*", 0, "*")]                   # mate unaligned
        elif x < 0.52:
            r1.append(rec(name, 4, "*", 0, "*"))
        elif x < 0.62:                                         # mates on different contigs, overlapping positions
            r2 = [rec(name, fb, refs[(refs.index(ref) + 1) % 3], a + ins - 100)]
        lines1 += r1
        groups2.append(r2)
    rng.shuffle(lines1)
    rng.shuffle(groups2)
    body2 = [x for g in groups2 for x in g]
    lines1.insert(0, rec("far", fa, "c2", 500))
    body2.append(rec("far", fb, "c2", 790))
    if bad_line_at is not None:
        lines1.insert(int(len(lines1) * bad_line_at), "broken\t0\tc1")
    head = ["@HD\tVN:1.6", "@SQ\tSN:c2\tLN:100000", "@SQ\tSN:c1\tLN:100000", "@SQ\tSN:c3\tLN:100000"]
    t1, t2 = eol.join(head + lines1) + eol, eol.join(head[:1] + body2) + eol
    if unterminated:
        t1, t2 = t1[:-len(eol)], t2[:-len(eol)]
    return t1, t2


def write_pair(d, t1, t2):
    i1, i2 = d / "i1.sam", d / "i2.sam"
    i1.write_bytes(t1.encode())
    i2.write_bytes(t2.encode())
    return i1, i2


def log_numbers(text):
    """The filter's log without the timing lines and the CLI's start line (those differ between one and several GPUs)."""
    return [x for x in text.splitlines() if x and not x.startswith(("device", "  phases", "Starting", "[timing]", "Finished"))]


def run_multi(ctxs, n, in1, in2, out1, out2, capfd, **kw):
    try:
        api.filter_files_multi(in1, in2, out1, out2, contexts=ctxs[:n], verbose=True, **kw)
        err = capfd.readouterr().err
        assert n == 1 or f"device text path over {n} GPUs" in err, err      # the n-context path ran, not the fallback
        return "ok", log_numbers(err)
    except pp.PolypolishError as e:
        capfd.readouterr()
        return "err", e.msg


def check_filter(ctxs, oracle, in1, in2, d, capfd, ns=NS, **kw):
    """Oracle, one context and n contexts agree: files, log numbers, or the error message."""
    try:
        exp = ("ok", oracle.filter(in1, in2, **kw))
    except Exception as e:
        exp = ("err", e.msg)
    one = run_multi(ctxs, 1, in1, in2, d / "one_1.sam", d / "one_2.sam", capfd, **kw)
    assert one[0] == exp[0], (exp, one)
    if exp[0] == "err":
        assert one[1] == exp[1]
    else:
        assert (d / "one_1.sam").read_bytes() == exp[1]["out1"] and (d / "one_2.sam").read_bytes() == exp[1]["out2"]
    for n in ns:
        o1, o2 = d / f"o1_{n}.sam", d / f"o2_{n}.sam"
        got = run_multi(ctxs, n, in1, in2, o1, o2, capfd, **kw)
        assert got == one, n
        if exp[0] == "ok":
            assert o1.read_bytes() == exp[1]["out1"] and o2.read_bytes() == exp[1]["out2"], n
    return exp


@pytest.mark.parametrize("seed,orient", [(1, "fr"), (2, "rf"), (3, "ff"), (4, "rr")])
def test_names_spread_over_ranges(ctxs, oracle, tmp_path, capfd, seed, orient):
    """One QNAME's alignments in several ranges, mate 1 in range 0 and mate 2 in the last range, mates in one file only, one
    alignment in one file and several in the other; contig ids that differ between contexts."""
    i1, i2 = write_pair(tmp_path, *pair_sams(seed, orient=orient))
    exp = check_filter(ctxs, oracle, i1, i2, tmp_path, capfd)
    assert exp[0] == "ok" and exp[1]["orientation"] == orient
    assert exp[1]["before_count"] > exp[1]["after_count"] > 0


@pytest.mark.parametrize("kw", [dict(orientation="auto"), dict(orientation="fr"), dict(orientation="rf"), dict(orientation="ff"),
                                dict(orientation="rr"), dict(orientation="bogus"), dict(low=5.0, high=95.0), dict(low=25.0, high=75.0),
                                dict(low=49.9, high=50.1), dict(low=0.01, high=99.99)])
def test_thresholds_and_orientations(ctxs, oracle, tmp_path, capfd, kw):
    """All five --orientation settings, ranks on ties and ranks whose values sit on different contexts; a user orientation
    without pairs gives the reference's error."""
    i1, i2 = write_pair(tmp_path, *pair_sams(11, n_pairs=600))
    check_filter(ctxs, oracle, i1, i2, tmp_path, capfd, **kw)


def test_auto_orientation_tie_and_no_unique_pairs(ctxs, oracle, tmp_path, capfd):
    fr = [(rec(f"p{i}", 0, "c1", 100 + 7 * i), rec(f"p{i}", 16, "c1", 400 + 7 * i)) for i in range(40)]
    ff = [(rec(f"q{i}", 0, "c1", 100 + 7 * i), rec(f"q{i}", 0, "c1", 400 + 7 * i)) for i in range(40)]
    both = fr + ff
    random.Random(5).shuffle(both)
    d = tmp_path / "tie"
    d.mkdir()
    i1, i2 = write_pair(d, "\n".join(a for a, _ in both) + "\n", "\n".join(b for _, b in both) + "\n")
    exp = check_filter(ctxs, oracle, i1, i2, d, capfd)
    assert exp[0] == "err" and exp[1].startswith("could not automatically determine")
    d = tmp_path / "multi"
    d.mkdir()
    multi = [rec(f"m{i}", 0, "c1", 100 + i) + "\n" + rec(f"m{i}", 256, "c1", 5000 + i) for i in range(30)]
    i1, i2 = write_pair(d, "\n".join(multi) + "\n", "\n".join(rec(f"m{i}", 16, "c1", 400 + i) for i in range(30)) + "\n")
    exp = check_filter(ctxs, oracle, i1, i2, d, capfd)
    assert exp[0] == "err" and exp[1].startswith("no one-alignment-per-read pairs")


@pytest.mark.parametrize("case", ["crlf", "unterminated", "tiny", "bad_late_line", "headers_only_range"])
def test_odd_text(ctxs, oracle, tmp_path, capfd, case):
    """CRLF, an unterminated last line, empty ranges (8 contexts on a file of a few lines), a malformed line in a later range (the
    one-context fallback's message with its line number), a range of headers only."""
    if case == "crlf":
        t = pair_sams(21, eol="\r\n")
    elif case == "unterminated":
        t = pair_sams(22, unterminated=True)
    elif case == "tiny":
        t = ("@HD\tVN:1.6\n" + "\n".join(rec(f"t{i}", 0, "c1", 100 + i) for i in range(3)) + "\n",
             "\n".join(rec(f"t{i}", 16, "c1", 400 + i) for i in range(3)) + "\n")
    elif case == "bad_late_line":
        t = pair_sams(23, bad_line_at=0.9)
    else:
        t1, t2 = pair_sams(24, n_pairs=100)
        t = ("".join(f"@CO\tcomment line {i:06d} padding padding padding padding\n" for i in range(2000)) + t1, t2)
    i1, i2 = write_pair(tmp_path, *t)
    exp = check_filter(ctxs, oracle, i1, i2, tmp_path, capfd)
    assert exp[0] == ("err" if case == "bad_late_line" else "ok")
    if case == "bad_late_line":
        assert "too few columns" in exp[1] and "(line " in exp[1]


def test_outputs_fifo_and_dev_null(ctxs, oracle, tmp_path):
    """A regular file, a FIFO read by another thread, /dev/null: the pieces of the contexts arrive in range order."""
    i1, i2 = write_pair(tmp_path, *pair_sams(31, n_pairs=3000))
    exp = oracle.filter(i1, i2)
    fifo = tmp_path / "out.fifo"
    os.mkfifo(fifo)
    for n in NS:
        got = {}

        def reader():
            with open(fifo, "rb") as f:
                got["data"] = f.read()
        t = threading.Thread(target=reader)
        t.start()
        api.filter_files_multi(i1, i2, fifo, "/dev/null", contexts=ctxs[:n])
        t.join(timeout=60)
        assert not t.is_alive() and got["data"] == exp["out1"], n
        t = threading.Thread(target=reader)
        t.start()
        api.filter_files_multi(i1, i2, tmp_path / "plain.sam", fifo, contexts=ctxs[:n])
        t.join(timeout=60)
        assert not t.is_alive() and got["data"] == exp["out2"], n
        assert (tmp_path / "plain.sam").read_bytes() == exp["out1"], n


def changed_rows(debug_tsv):
    lines = debug_tsv.split(b"\n")
    return b"\n".join([lines[0]] + [x for x in lines[1:] if x.split(b"\t")[7:8] == [b"changed"]]) + b"\n"


def with_8bit_seq(path):
    """One aligned record of the file gets a SEQ byte outside the 4-bit alphabet (the tokeniser starts again in 8-bit mode)."""
    lines = path.read_bytes().split(b"\n")
    for i, x in enumerate(lines):
        f = x.split(b"\t")
        if len(f) > 10 and not x.startswith(b"@") and not int(f[1]) & 4 and len(f[9]) > 10:
            f[9] = f[9][:5] + b"Z" + f[9][6:]
            lines[i] = b"\t".join(f)
            break
    path.write_bytes(b"\n".join(lines))


@pytest.mark.parametrize("seed,opts,eight_bit", [(41, {}, False), (42, dict(careful=True), False), (43, dict(min_depth=3), True)])
def test_filter_polish_multi(ctxs, oracle, tmp_path, capfd, seed, opts, eight_bit):
    """The fused call over n contexts: reads of repeat families (k != 1), --careful, an 8-bit SEQ byte; the FASTA, the change
    report and the filtered files are the oracle's `filter` then `polish`, and the one-context call's."""
    syn = api.Synth(seed=seed, n_contigs=3, contig_len=30_000, depth=40, repeat_fraction=0.1)
    fa, sams = syn.write(tmp_path)
    if eight_bit:
        with_8bit_seq(pathlib.Path(sams[0]))
    fo = oracle.filter(sams[0], sams[1])
    o1, o2 = tmp_path / "of1.sam", tmp_path / "of2.sam"
    o1.write_bytes(fo["out1"])
    o2.write_bytes(fo["out2"])
    exp = oracle.polish(fa, [o1, o2], debug=True, **opts)
    one = api.filter_polish_files_multi(fa, sams[0], sams[1], contexts=ctxs[:1], changes=tmp_path / "one.tsv", **opts)
    capfd.readouterr()
    assert one == exp["fasta"]
    assert (tmp_path / "one.tsv").read_bytes() == changed_rows(exp["debug_tsv"])
    for n in NS:
        chg = tmp_path / f"chg_{n}.tsv"
        assert api.filter_polish_files_multi(fa, sams[0], sams[1], contexts=ctxs[:n], changes=chg, verbose=True, **opts) == exp["fasta"], n
        # the n-context path ran, not the fallback (like `polish`, the fused call uses at most one context per contig)
        assert f"filter over {min(n, 3)} GPUs" in capfd.readouterr().err, n
        assert chg.read_bytes() == changed_rows(exp["debug_tsv"]), n
        f1, f2 = tmp_path / f"f1_{n}.sam", tmp_path / f"f2_{n}.sam"
        assert api.filter_polish_files_multi(fa, sams[0], sams[1], f1, f2, contexts=ctxs[:n], **opts) == exp["fasta"], n
        assert f1.read_bytes() == fo["out1"] and f2.read_bytes() == fo["out2"], n


def test_filter_polish_multi_errors(ctxs, oracle, tmp_path):
    """What the n-context path does not settle goes to the one-context call: its messages."""
    syn = api.Synth(seed=44, contig_len=20_000, depth=30)
    fa, sams = syn.write(tmp_path)
    bad = tmp_path / "bad_1.sam"
    bad.write_bytes(open(sams[0], "rb").read() + b"zz\t0\tcontig_1\t100\t60\t50M\t*\t0\t0\t*\t*\tNM:i:0\n")
    for n in NS:
        with pytest.raises(pp.PolypolishError) as e:
            api.filter_polish_files_multi(fa, bad, sams[1], contexts=ctxs[:n])
        assert "no alignments for read zz contain sequence" in e.value.msg
        with pytest.raises(pp.PolypolishError) as e:
            api.filter_polish_files_multi(fa, sams[0], sams[1], contexts=ctxs[:n], low=60.0)
        assert "--low must be greater than 0 and less than 50" in e.value.msg


def _sha_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def test_config3_full_size_multi(ctxs, oracle):
    """BASELINE config 3 (5 Mbp x 100x, `filter` then `polish`) with 8 contexts, and over every visible GPU when there are several:
    both filtered files and the FASTA (`polish` of the filtered files over the same contexts, and the fused call) have the oracle's
    SHA-256."""
    import torch
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_fmulti_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > (8 << 30) else None)
    try:
        syn = api.Synth(seed=2, contig_len=5_000_000, depth=100)
        fa, sams = syn.write(d)
        fo = oracle.filter(sams[0], sams[1])
        o1, o2 = os.path.join(d, "o1.sam"), os.path.join(d, "o2.sam")
        open(o1, "wb").write(fo["out1"])
        open(o2, "wb").write(fo["out2"])
        del fo
        exp = hashlib.sha256(oracle.polish(fa, [o1, o2])["fasta"]).hexdigest()
        runs = [dict(contexts=ctxs[:8])]
        if torch.cuda.device_count() > 1:
            runs.append(dict(devices=list(range(torch.cuda.device_count()))))
        f1, f2 = os.path.join(d, "f1.sam"), os.path.join(d, "f2.sam")
        for kw in runs:
            api.filter_files_multi(sams[0], sams[1], f1, f2, **kw)
            assert _sha_file(f1) == _sha_file(o1) and _sha_file(f2) == _sha_file(o2)
            assert hashlib.sha256(api.polish_files_multi(fa, [f1, f2], **kw)).hexdigest() == exp
            assert hashlib.sha256(api.filter_polish_files_multi(fa, sams[0], sams[1], **kw)).hexdigest() == exp
    finally:
        shutil.rmtree(d, ignore_errors=True)


def test_cli_gpus(ctxs, oracle, tmp_path):
    """`polypolish filter --gpu-count K` and `filter-polish --gpu-count K` (K = the visible GPUs) against K = 1: same files, FASTA and
    log numbers."""
    import torch
    exe = os.path.join(ROOT, "build", "polypolish")
    k = str(max(1, torch.cuda.device_count()))
    syn = api.Synth(seed=45, n_contigs=2, contig_len=25_000, depth=40)
    fa, sams = syn.write(tmp_path)
    out = {}
    for g in ("1", k):
        o1, o2 = tmp_path / f"a1_{g}.sam", tmp_path / f"a2_{g}.sam"
        r = subprocess.run([exe, "filter", "--gpu-count", g, "--in1", sams[0], "--in2", sams[1], "--out1", o1, "--out2", o2], capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
        fp = subprocess.run([exe, "filter-polish", "--gpu-count", g, "--in1", sams[0], "--in2", sams[1], fa], capture_output=True)
        assert fp.returncode == 0, fp.stderr.decode()
        out[g] = (o1.read_bytes(), o2.read_bytes(), log_numbers(r.stderr.decode()), fp.stdout)
    assert out[k] == out["1"]
    fo = oracle.filter(sams[0], sams[1])
    assert out["1"][:2] == (fo["out1"], fo["out2"])
