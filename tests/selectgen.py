"""FASTA + SAM cases for read selection (process_one_read, alignment.rs:275-305): which records are good, k of every read group and
the errors only good records raise, under every option set of OPTS (seeded, deterministic, in the style of tests/limitgen.py).

Each generator returns a fuzzgen.Case with a `facts` dict of what it was built to reach; tests assert the facts before they trust a
pass.  The model every case is checked with is limitgen.record_good(..., detail=True).
  * option_grid (A): NM on both sides of every max_errors of OPTS and around the 255 the per-alignment summary holds, CIGAR ends
    from M = X S H I D, ZP tags in several casings, groups of 1, 2, 3 and 9 records whose k takes every value 0-9, SEQ="*"
    records whose group's source record is not good, unaligned records inside groups, a QNAME that ends one file and starts the
    next, and probe loci whose vote flips with max_errors and with --careful.
  * block_edges (B): multi-record groups starting -3 .. +3 records from 256-alignment block edges (k_goodk's blocks), groups of
    257 and 513 records, and optionally a group across the alignment index where k_goodk's grid-stride loop wraps.
  * global_k (C): A plus a group past SC_GROUP_SCAN_LIMIT (limitgen.read_groups), so the grid runs in global-k mode.
  * errors (D): unknown RNAME, CIGAR / SEQ length mismatch, N and P inside the CIGAR, an overrun past a contig's end, each on a
    record whose goodness depends on the options; which one the reference names depends on the option set.
  * careful_noseq (E): groups without any SEQ, kept by a load with --careful and raised by a call without it.
"""
import random

from tests import limitgen as lg
from tests.fuzzgen import Case
from tests.limitgen import rand_seq, sam

U32 = 2 ** 32
# the option grid, in the order the resident tests run it: every neighbour pair differs in max_errors or --careful
OPTS = [dict(), dict(max_errors=0), dict(max_errors=1, careful=True), dict(max_errors=254), dict(max_errors=U32 - 1),
        dict(max_errors=255), dict(max_errors=256, careful=True), dict(max_errors=256), dict(max_errors=65535), dict(max_errors=U32 - 2),
        dict(max_errors=65536, careful=True), dict(careful=True)]
MAXERRS = sorted({o.get("max_errors", 10) for o in OPTS})
NMS = sorted({x for m in MAXERRS for x in (m - 1, m, m + 1) if 0 <= x <= U32 - 2} | {254, 255, 256, 257, 1000, 65535, 65536, U32 - 2})
ENDS = "M=XSHID"
ZPS = [None, "ZP:Z:fail", "zp:z:FAIL", "ZP:Z:pass", "ZP:Z:failx"]
END_LEN = {"=": 3, "X": 1, "S": 4, "H": 4, "I": 2, "D": 2}      # length of a non-M first / last op
READ = 60


def shaped(rng, ref, pos0, first="M", last="M", n=READ):
    """(CIGAR, SEQ) of a read at pos0 of `ref` whose first and last CIGAR ops are `first` / `last` around a match run; n read
    bases in all (hard clips excepted)."""
    ends = [(END_LEN[o], o) for o in (first, last) if o != "M"]
    mid = n - sum(l for l, o in ends if o in "=XSI")
    ops = ([(END_LEN[first], first)] if first != "M" else []) + [(mid, "M")] + ([(END_LEN[last], last)] if last != "M" else [])
    seq, r = [], pos0
    for l, o in ops:
        if o in "M=":
            seq.append(ref[r:r + l])
            r += l
        elif o == "X":
            seq.append("".join(lg._mutate(rng, b) for b in ref[r:r + l]))
            r += l
        elif o in "SI":
            seq.append(rand_seq(rng, l))
        elif o == "D":
            r += l
    return "".join("%d%s" % (l, o) for l, o in ops), "".join(seq)


class Builder:
    """Read groups on a set of contigs, kept as groups of SAM lines until they are laid out into files."""

    def __init__(self, rng, contigs):
        self.rng = rng
        self.contigs = dict(contigs)
        self.n = 0

    def qname(self, tag):
        self.n += 1
        return "%s%d" % (tag, self.n)

    def read(self, q, ctg, flag=0, first="M", last="M", nm=0, zp=None, star=False, pos=None, seq=None):
        ref = self.contigs[ctg]
        pos = self.rng.randint(0, len(ref) - READ - 10) if pos is None else pos
        cig, s = shaped(self.rng, ref, pos, first, last)
        return sam(q, flag, ctg, pos, cig, "*" if star else (seq or s), nm, [zp] if zp else [])

    def unaligned(self, q):
        return "\t".join([q, "4", "*", "0", "0", "*", "*", "0", "0", rand_seq(self.rng, 30), "*"])

    def probe_reads(self, ctg, P, y, pos, nm, q, flag=0):
        """A 60M read over position P of contig `ctg` carrying base y there."""
        ref = self.contigs[ctg]
        s = ref[pos:P] + y + ref[P + 1:pos + READ]
        return sam(q, flag, ctg, pos, "%dM" % READ, s, nm)


def layout(groups, n_files=2, split=None):
    """SAM texts of the groups in order, cut into n_files at group boundaries; `split` = a group whose records are cut between
    file 1 and file 2 (the same QNAME ends one and starts the next)."""
    texts = [[] for _ in range(n_files)]
    cut = len(groups) // 2
    for i, g in enumerate(groups):
        texts[0 if i < cut else min(n_files - 1, 1)].extend(g)
    if split:
        texts[0].extend(split[:len(split) // 2])
        texts[1][:0] = split[len(split) // 2:]
    return ["\n".join(t) + "\n" for t in texts]


def probes(b, ctg, rng):
    """Loci of contig `ctg` whose vote flips between option sets: for every max_errors m > 0 of OPTS, four reads of NM 0 and one of
    NM m carry base Y (changed iff max_errors >= m, with min_depth 5); and ten two-record groups of NM 0 (each read counts 1/2)
    carry Y at another locus (changed unless --careful)."""
    ref = b.contigs[ctg]
    out = []
    P = 100
    for m in [x for x in MAXERRS if 0 < x < U32 - 1]:
        y = lg._mutate(rng, ref[P])
        for j, nm in enumerate([0, 0, 0, 0, m]):
            out.append([b.probe_reads(ctg, P, y, P - 20 - 3 * j, nm, b.qname("p"), 16 if j % 2 else 0)])
        P += 150
    y = lg._mutate(rng, ref[P])
    for j in range(10):
        q = b.qname("pc")
        out.append([b.probe_reads(ctg, P, y, P - 15 - 2 * j, 0, q, 16 if j % 2 else 0), b.read(q, "ga", 256, star=True)])
    assert P + 100 < len(ref)
    return out


def option_grid(seed):
    rng = random.Random(seed)
    n_probe = 150 * (len(MAXERRS) + 1) + 200
    b = Builder(rng, [("ga", rand_seq(rng, 3000)), ("gb", rand_seq(rng, 3000)), ("probe", rand_seq(rng, n_probe))])
    groups = []
    # single records: every NM, every ZP tag, every pair of end ops
    for nm in NMS:
        groups.append([b.read(b.qname("n"), rng.choice("ga gb".split()), rng.choice([0, 16]), nm=nm)])
    for zp in ZPS:
        for nm in (0, 255, 256):
            groups.append([b.read(b.qname("z"), "ga", rng.choice([0, 16]), nm=nm, zp=zp)])
    for f in ENDS:
        for l in ENDS:
            groups.append([b.read(b.qname("e"), "gb", rng.choice([0, 16]), first=f, last=l, nm=rng.choice([0, 10, 11, 256]))])
    # groups of 2, 3 and 9 with mixed goodness: secondaries with and without SEQ, on both strands
    for size in (2, 3, 9):
        for _ in range(12):
            q = b.qname("g%d_" % size)
            g = []
            for j in range(size):
                r = rng.random()
                f, l = ("S", "M") if r < 0.1 else ("M", "X") if r < 0.15 else ("M", "M")
                zp = rng.choice(ZPS) if rng.random() < 0.2 else None
                g.append(b.read(q, rng.choice(["ga", "gb"]), (256 if j else 0) | rng.choice([0, 16]), f, l, rng.choice(NMS), zp,
                                star=j > 0 and rng.random() < 0.6))
            groups.append(g)
    # 9-record groups with exactly j always-good records (k = j under every set without --careful)
    for j in range(10):
        q = b.qname("k")
        g = [b.read(q, "ga", 0, nm=0) if i < j else b.read(q, "gb", 256 if i else 0, "S", "M", 0) for i in range(9)]
        rng.shuffle(g)
        groups.append(g)
    # a 9-record group whose k changes with every max_errors
    q = b.qname("kx")
    groups.append([b.read(q, "ga", 256 if i else 0, nm=nm, star=i > 0) for i, nm in enumerate([0, 1, 9, 10, 11, 255, 256, 65536, U32 - 2])])
    # SEQ="*" records on both strands whose group's source record (the first with SEQ) is not good
    for src_ends, src_nm, src_zp in ((("S", "M"), 0, None), (("M", "M"), 257, None), (("M", "M"), 0, "zp:z:FAIL")):
        q = b.qname("src")
        g = [b.read(q, "ga", 16, *src_ends, src_nm, src_zp)]
        g += [b.read(q, rng.choice(["ga", "gb"]), 256 | s, nm=rng.choice([0, 1, 11]), star=True) for s in (0, 16, 16, 0)]
        groups.append(g)
    # unaligned records inside groups: the group's own QNAME and another one (neither ends the group nor counts in it)
    for other in (False, True):
        q = b.qname("u")
        groups.append([b.read(q, "ga", 0, nm=0), b.unaligned(b.qname("x") if other else q), b.read(q, "gb", 256, nm=1, star=True)])
        groups.append([b.read(b.qname("s"), "gb", 0, nm=0), b.unaligned(b.qname("x"))])
    groups += probes(b, "probe", rng)
    rng.shuffle(groups)
    q = b.qname("split")
    split = [b.read(q, "ga", 0, nm=0), b.read(q, "gb", 256, nm=11, star=True), b.read(q, "gb", 16, nm=0), b.read(q, "ga", 272, nm=2, star=True)]
    texts = layout(groups, split=split)
    c = Case(lg.fasta(list(b.contigs.items())), texts, dict())
    c.contigs = {k: len(v) for k, v in b.contigs.items()}
    c.facts = dict(split=q)
    return c


def block_edges(seed, wrap=None, big=(257, 513)):
    """Single records as filler and groups of 2-8 records whose first record sits -3 .. +3 records from a 256-alignment block edge,
    groups of the `big` sizes starting one record before an edge (a block holds only their middle), and with `wrap`, a group across
    alignment index `wrap` (where k_goodk's grid-stride loop starts its second round).  Every record has its own SEQ, so a group can
    be split by renaming.  facts: per multi-record group its QNAME, first alignment and size."""
    rng = random.Random(seed)
    b = Builder(rng, [("ba", rand_seq(rng, 5000)), ("bb", rand_seq(rng, 5000))])
    recs, groups = [], []

    def single():
        recs.append(b.read(b.qname("s"), rng.choice(["ba", "bb"]), rng.choice([0, 16]), nm=rng.choice([0, 0, 1, 2, 11])))

    def group(size, at):
        while len(recs) < at:
            single()
        q = b.qname("G")
        groups.append(dict(qname=q, start=len(recs), size=size))
        for j in range(size):
            r = rng.random()
            if j == 0 or j == size - 1:
                nm, f = 0, "M"                                       # a good record on either side of any edge
            else:
                nm, f = rng.choice([0, 1, 10, 11, 255, 256, 1000, 65536, U32 - 2]), "S" if r < 0.1 else "M"
            recs.append(b.read(q, rng.choice(["ba", "bb"]), (256 if j else 0) | rng.choice([0, 16]), f, "M", nm,
                               "ZP:Z:fail" if r > 0.93 and 0 < j < size - 1 else None))

    edge = 256
    for off in range(-3, 4):
        for size in (2, 6):
            group(size, edge + off)
            edge += 256
    for size in big:
        group(size, edge - 1)
        edge = (len(recs) // 256 + 2) * 256
    group(7, 512 * ((len(recs) + 600) // 512) - 3)                  # across a multiple of 512: the emulator's grid of 2 wraps there
    if wrap:
        group(7, wrap - 3)
    for _ in range(40):
        single()
    c = Case(lg.fasta(list(b.contigs.items())), ["\n".join(recs) + "\n"], dict())
    c.contigs = {k: len(v) for k, v in b.contigs.items()}
    c.facts = dict(groups=groups, n_aln=len(recs), wrap=wrap)
    return c


def split_group(case, g, at):
    """The case's text with the records of group g from alignment index `at` on renamed (the group split in two there)."""
    lines = case.sam_texts[0].split("\n")
    for i in range(at, g["start"] + g["size"]):
        lines[i] = "%s_far\t" % g["qname"] + lines[i].split("\t", 1)[1]
    return ["\n".join(lines)]


def global_k(seed):
    """A's text followed by a read_groups file with a group of 9,000 records (global-k mode whenever one of its records is good)."""
    a = option_grid(seed)
    rg = lg.read_groups(seed + 1, [9000], offset=0, where="last", filler=300)
    c = Case(a.fasta_text + rg.fasta_text, a.sam_texts + rg.sam_texts, dict())
    c.contigs = dict(a.contigs)
    for line in rg.fasta_text.split("\n"):
        if line.startswith(">"):
            name = line[1:]
        elif line:
            c.contigs[name] = len(line)
    c.facts = dict(big=rg.facts["groups"][0])
    return c


def errors(seed):
    """Error records whose goodness depends on the options, in this SAM order (NM, group): P inside the CIGAR (65536, two records),
    N inside (256, two records), an overrun past contig `da`'s end (11, single), an unknown RNAME (1, single), a CIGAR / SEQ length
    mismatch (0, two records); between them reads that polish `da`.  facts["expect"]: the error kind the reference names under each
    option set of ERR_OPTS, None where the call succeeds."""
    rng = random.Random(seed)
    L = 4000
    b = Builder(rng, [("da", rand_seq(rng, L)), ("db", rand_seq(rng, 2000))])
    ref = b.contigs["da"]
    out = []

    def filler(n):
        for _ in range(n):
            P = rng.randint(200, 1100)                          # (clear of the variant loci)
            out.append(b.read(b.qname("f"), "da", rng.choice([0, 16]), nm=rng.choice([0, 1]), pos=P))

    def two(first_line, q):
        out.append(first_line)
        out.append(b.read(q, "db", 272, nm=0, star=True))

    filler(60)
    q = b.qname("eP")
    two(sam(q, 0, "da", 500, "20M1P40M", ref[500:560], 65536), q)
    filler(60)
    q = b.qname("eN")
    two(sam(q, 0, "da", 700, "30M2N30M", ref[700:730] + ref[732:762], 256), q)
    filler(60)
    # ends 8 bases past the end of `da` with no homopolymer at its end: the trim keeps entries past the end
    s = ref[L - 52:] + "ACGTACGT"
    out.append(sam(b.qname("eO"), 0, "da", L - 52, "60M", s, 11))
    filler(60)
    out.append(sam(b.qname("eR"), 16, "nowhere", 10, "60M", rand_seq(rng, 60), 1))
    filler(60)
    q = b.qname("eL")
    two(sam(q, 0, "da", 900, "60M", ref[900:959], 0), q)
    filler(60)
    # varied-depth variant loci so that the calls that succeed change the draft
    for k in range(6):
        P = 1200 + 300 * k
        y = lg._mutate(rng, ref[P])
        for j in range(5 + k % 3):
            out.append(b.probe_reads("da", P, y, P - 10 - 3 * j, j % 2, b.qname("v"), 16 if j % 2 else 0))
    c = Case(lg.fasta(list(b.contigs.items())), ["\n".join(out) + "\n"], dict())
    c.contigs = {k: len(v) for k, v in b.contigs.items()}
    c.facts = dict(expect=list(ERR_EXPECT))
    return c


# errors(): the option sets it runs and what the reference names under each: ok -> unknown RNAME -> ok -> N -> ok -> P -> overrun ->
# length mismatch -> ok (only max_errors 0 with --careful leaves every error record out)
_OK = dict(max_errors=0, careful=True)
ERR_OPTS = [_OK, dict(), dict(_OK, min_depth=3), dict(max_errors=256), dict(_OK, fraction_valid=0.8), dict(max_errors=65536),
            dict(max_errors=65536, careful=True), dict(max_errors=0), _OK]
ERR_EXPECT = [None, "unknown_contig", None, "bad_op", None, "bad_op", "oob", "seq_mismatch", None]


def careful_noseq(seed, variant):
    """A dataset to load with --careful that holds two-record groups without any SEQ (kept, PP_FLAG_NOSEQ):
    "none": its records are never good under max_errors <= 19 (NM 20);  "good": one of its records is good (NM 0);
    "after": an earlier single record on an unknown contig is good, so its error comes first under every set without --careful;
    "unknown": the group's first record is on an unknown contig (the group's error still wins).  Plus reads that polish `ea`."""
    rng = random.Random(seed)
    b = Builder(rng, [("ea", rand_seq(rng, 3000))])
    ref = b.contigs["ea"]
    out = []

    def filler(n):
        for _ in range(n):
            out.append(b.read(b.qname("f"), "ea", rng.choice([0, 16]), nm=rng.choice([0, 1])))

    filler(40)
    if variant == "after":
        out.append(sam(b.qname("bad"), 0, "nowhere", 5, "60M", rand_seq(rng, 60), 0))
        filler(10)
    nm = {"none": (20, 20), "good": (20, 0), "after": (0, 0), "unknown": (0, 0)}[variant]
    q = "zz"
    out.append(sam(q, 256, "nowhere" if variant == "unknown" else "ea", 100, "60M", "*", nm[0]))
    out.append(sam(q, 272, "ea", 400, "60M", "*", nm[1]))
    filler(40)
    for k in range(3):
        P = 800 + 400 * k
        y = lg._mutate(rng, ref[P])
        for j in range(6):
            out.append(b.probe_reads("ea", P, y, P - 10 - 3 * j, 0, b.qname("v"), 16 if j % 2 else 0))
    c = Case(lg.fasta(list(b.contigs.items())), ["\n".join(out) + "\n"], dict())
    c.contigs = {k: len(v) for k, v in b.contigs.items()}
    c.facts = dict(variant=variant, expect="unknown_contig" if variant == "after" else "noseq")
    return c


NOSEQ_VARIANTS = ["none", "good", "after", "unknown"]
