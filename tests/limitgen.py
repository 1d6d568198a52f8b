"""FASTA + SAM cases that cross the size limits of the polish path (seeded, deterministic, in the style of tests/fuzzgen.py).

Each generator returns a fuzzgen.Case with an extra `facts` dict: what the case was built to reach, so that a test can assert the
limit was crossed before it trusts a pass.  The limits (polypolish_b200/csrc/polish_dev.cuh unless noted):
  * long_alleles: other alleles longer than the exact signature (15 symbols 4-bit, 7 bytes 8-bit), hashed and compared against
    the reads; alleles inserted by the one-indel fast walk (aM bI cM, read <= 192); two equal-length alleles one base apart.
  * output_growth: a 2048-position chunk that emits more than CP_STAGE = 4096 bytes (the unstaged path of compact_body) and
    a polished length above the first output capacity G + G/16 + 2^20 (and the callers' G + 2^20).
  * node_pool: more distinct (position, allele) pairs than the first node capacity max(65536, n_aln/8 + G/64).
  * read_groups: QNAME groups that cross 256-alignment blocks and SC_GROUP_SCAN_LIMIT (global-k mode), a QNAME that ends one
    SAM file and starts the next (two groups).
  * boundary_case: a position covered by alignments of given k whose reference depth is an exact vote boundary.
"""
import random
import re

from tests.fuzzgen import Case, revcomp

ACGT = "ACGT"
SCAN_LIMIT = 8192          # SC_GROUP_SCAN_LIMIT
PR_BLOCK = 256             # PR_THREADS: alignments per k_goodk block
CP_STAGE = 4096            # bytes one compaction chunk stages in shared memory
CHUNK = 2048               # positions per tile / compaction chunk


def rand_seq(rng, n):
    return "".join(rng.choice(ACGT) for _ in range(n))


def sam(qname, flag, rname, pos0, cigar, seq, nm=0, extra=()):
    return "\t".join([qname, str(flag), rname, str(pos0 + 1), "60", cigar, "*", "0", "0", seq, "*", "NM:i:%d" % nm] + list(extra))


def fasta(contigs):
    return "".join(">%s\n%s\n" % (n, s) for n, s in contigs)


def _mutate(rng, b):
    return rng.choice([x for x in ACGT if x != b])


# ---- A. long other alleles -------------------------------------------------------------------------------------------------
def long_alleles(seed, lengths, eight_bit=False, reads_per_locus=16, huge=False):
    """One locus per allele length L (anchor base + L - 1 inserted bases) on contig `long`, carried by reads with SEQ on both strands;
    every read has a SEQ="*" secondary of the opposite strand on contig `mirror` (the reverse complement of `long`), which takes the
    read's sequence reverse-complemented and so carries the reverse-complemented allele there.  Read shapes vary: a = 1 (the allele
    starts at the read's first base), c = 9 (the shortest last run the one-indel fast walk takes) and c = 8 (one too short).
    Then equal-length alleles one base apart (first / middle / last inserted base) at 6 : 1 and 5 : 5; with eight_bit, alleles that
    hold '-' bytes and one read whose SEQ has a byte outside the 4-bit alphabet (the batch goes to the 8-bit pool).  huge: a read
    of 65,535 bases whose allele is longer than 65,000."""
    rng = random.Random(seed)
    spacing = 200
    n_pair = 6
    pair_len = 40
    lpos = []
    P = 100
    for L in lengths:
        lpos.append(P)
        P += spacing
    pair_pos = []
    for j in range(n_pair):
        pair_pos.append(P)
        P += spacing
    glen = P + 100
    long_seq = rand_seq(rng, glen)
    lines = []
    shapes = [(30, 30), (1, 30), (30, 9), (30, 8), (20, 12), (1, 9), (40, 8), (25, 25)]
    n = 0
    facts = dict(allele_lengths=[], fast_walk_reads=0, hashed_reads=0)
    exact_max = 7 if eight_bit else 15

    def add_read(P, ins, a, c, flag, with_secondary=True):
        nonlocal n
        s0 = P - a + 1
        read = long_seq[s0:P + 1] + ins + long_seq[P + 1:P + 1 + c]
        q = "q%d" % n
        n += 1
        cig = "%dM%dI%dM" % (a, len(ins), c) if ins else "%dM" % (a + c)
        lines.append(sam(q, flag, "long", s0, cig, read, 0))
        if with_secondary:
            m0 = glen - 1 - (P + c)
            cig2 = "%dM%dI%dM" % (c, len(ins), a) if ins else "%dM" % (a + c)
            lines.append(sam(q, (flag ^ 16) | 256, "mirror", m0, cig2, "*", 0))
        if ins and len(read) <= 192 and c >= 9 and a <= 255 and not eight_bit:
            facts["fast_walk_reads"] += 1
        if len(ins) + 1 > exact_max:
            facts["hashed_reads"] += 1

    for L, P in zip(lengths, lpos):
        ins = rand_seq(rng, L - 1)
        if eight_bit and L >= 9:
            ins = "".join("-" if i % 7 == 3 else ch for i, ch in enumerate(ins))      # '-' bytes: kept in --debug, dropped from FASTA
        facts["allele_lengths"].append(L)
        for r in range(reads_per_locus):
            a, c = shapes[r % len(shapes)]
            add_read(P, ins, a, c, 16 if r % 2 else 0)
    # equal-length alleles one base apart, first / middle / last inserted base, counts 6 : 1 and 5 : 5
    for j, P in enumerate(pair_pos):
        ins = rand_seq(rng, pair_len - 1)
        at = [0, (pair_len - 1) // 2, pair_len - 2][j % 3]
        alt = ins[:at] + _mutate(rng, ins[at]) + ins[at + 1:]
        na, nb = (6, 1) if j < 3 else (5, 5)
        for r in range(na + nb):
            add_read(P, ins if r < na else alt, 30, 30, 16 if r % 2 else 0, with_secondary=False)
    contigs = [("long", long_seq), ("mirror", revcomp(long_seq))]
    if eight_bit:                                                       # a byte outside "=ACMGRSVTWYHKDBN": 8-bit pool
        s0 = 20
        read = long_seq[s0:s0 + 30] + "." + long_seq[s0 + 31:s0 + 60]
        lines.append(sam("q8bit", 0, "long", s0, "60M", read, 1))
    if huge:
        a = c = 200
        hseq = rand_seq(rng, 1000)
        ins = rand_seq(rng, 65535 - a - c)
        for r in range(6):
            lines.append(sam("h%d" % r, 16 if r % 2 else 0, "huge", 300 - a + 1, "%dM%dI%dM" % (a, len(ins), c),
                             hseq[301 - a:301] + ins + hseq[301:301 + c], 0))
        contigs.append(("huge", hseq))
        facts["allele_lengths"].append(len(ins) + 1)
        facts["hashed_reads"] += 6
    facts["seq_bits"] = 8 if eight_bit else 4
    c = Case(fasta(contigs), ["\n".join(lines) + "\n"], dict(min_depth=5))
    c.facts = facts
    return c


# ---- B. output growth ------------------------------------------------------------------------------------------------------
def output_growth(seed, n_ins=300, ins_len=4000, depth=5, contig_lens=(21_504, 19_000)):
    """n_ins insertions of ins_len bases, `depth` reads each, spread over two contigs; contig 1 ends in the middle of a
    2048-position chunk that emits more than 4096 bytes.  facts: the designed output bytes per chunk and in total."""
    rng = random.Random(seed)
    contigs = [("grow%d" % (i + 1), rand_seq(rng, L)) for i, L in enumerate(contig_lens)]
    G = sum(contig_lens)
    spacing = (G - 200 * len(contigs)) // n_ins
    lines = []
    growth = {}
    n = 0
    g0 = 0
    per = [n_ins * L // G for L in contig_lens]
    per[-1] = n_ins - sum(per[:-1])
    for (name, s), k in zip(contigs, per):
        for j in range(k):
            P = 100 + j * spacing
            assert P + 60 < len(s)
            ins = rand_seq(rng, ins_len)
            for r in range(depth):
                a, c = 40, 40
                lines.append(sam("g%d" % n, 16 if r % 2 else 0, name, P - a + 1, "%dM%dI%dM" % (a, ins_len, c),
                                 s[P - a + 1:P + 1] + ins + s[P + 1:P + 1 + c], 0))
                n += 1
            growth[(g0 + P) // CHUNK] = growth.get((g0 + P) // CHUNK, 0) + ins_len
        g0 += len(s)
    chunk_bytes = {ch: min(CHUNK, G - ch * CHUNK) + extra for ch, extra in growth.items()}
    boundary_chunk = contig_lens[0] // CHUNK
    c = Case(fasta(contigs), ["\n".join(lines) + "\n"], dict())
    c.facts = dict(G=G, total=G + sum(growth.values()), chunk_bytes=chunk_bytes, boundary_chunk=boundary_chunk)
    return c


# ---- C. node pool ----------------------------------------------------------------------------------------------------------
def node_pool(seed, length=100_000, depth=30, read_len=150, n_ins=5):
    """Every read carries n_ins random insertions of 3-6 bases: about length * depth / read_len * n_ins distinct other alleles."""
    rng = random.Random(seed)
    ref = rand_seq(rng, length)
    lines = []
    n_reads = length * depth // read_len
    for i in range(n_reads):
        st = rng.randint(0, length - read_len - 1)
        cuts = sorted(rng.sample(range(10, read_len - 10), n_ins))
        ops, read, p = [], [], st
        prev = 0
        for cut in cuts:
            ops.append("%dM" % (cut - prev))
            read.append(ref[st + prev:st + cut])
            ins = rand_seq(rng, rng.randint(3, 6))
            ops.append("%dI" % len(ins))
            read.append(ins)
            prev = cut
        ops.append("%dM" % (read_len - prev))
        read.append(ref[st + prev:st + read_len])
        lines.append(sam("n%d" % i, 16 if i % 2 else 0, "nodes", st, "".join(ops), "".join(read), 0))
    c = Case(fasta([("nodes", ref)]), ["\n".join(lines) + "\n"], dict())
    c.facts = dict(n_aln=n_reads, G=length, node_cap=max(65536, n_reads // 8 + length // 64))
    return c




# ---- D. read groups --------------------------------------------------------------------------------------------------------
def read_groups(seed, sizes, offset=0, where="first", contig_len=20_000, n_contigs=3, filler=1200):
    """QNAME groups of the given sizes: one aligned record with SEQ, the rest SEQ="*" secondaries spread over every contig, some of
    them bad (NM above max_errors, a soft-clipped end, ZP:Z:fail) so that k != size.  Each starts at alignment index == offset
    (mod 256) among single-record reads; the first of them is the first group of the list (where="first") or the last of them the
    last (where="last").  Also groups of k = 32 and k = 33 good records, and the QNAME `split`, whose 3 records end reads_1.sam and
    whose 4 records start reads_2.sam (two groups).  facts: per big group its QNAME, size and first alignment index."""
    rng = random.Random(seed)
    names = ["ctg%d" % (i + 1) for i in range(n_contigs)]
    refs = {nm: rand_seq(rng, contig_len) for nm in names}
    recs = []                                    # SAM order; every line is an aligned record
    n_single = [0]

    def single():
        c = rng.choice(names)
        st = rng.randint(0, contig_len - 61)
        read = list(refs[c][st:st + 60])
        nm = 0
        if rng.random() < 0.3:
            i = rng.randint(0, 59)
            read[i] = _mutate(rng, read[i])
            nm = 1
        recs.append(sam("s%d" % n_single[0], 16 if rng.random() < 0.5 else 0, c, st, "60M", "".join(read), nm))
        n_single[0] += 1

    def group(q, size, all_good=False):
        c = rng.choice(names)
        st = rng.randint(0, contig_len - 61)
        src = list(refs[c][st:st + 60])
        for i in rng.sample(range(60), 2):
            src[i] = _mutate(rng, src[i])
        recs.append(sam(q, 16 if rng.random() < 0.5 else 0, c, st, "60M", "".join(src), 2))
        for j in range(size - 1):
            cig, nm, extra = "60M", rng.randint(0, 3), []
            r = 1.0 if all_good else rng.random()
            if r < 0.05:
                nm = 20
            elif r < 0.08:
                cig = "5S55M"
            elif r < 0.10:
                extra = ["ZP:Z:fail"]
            recs.append(sam(q, 256 | (16 if rng.random() < 0.5 else 0), rng.choice(names), rng.randint(0, contig_len - 61), cig, "*", nm,
                            extra))

    def split_group():
        c = names[0]
        for j in range(3):
            recs.append(sam("split", 256 if j else 0, c, 100 + 40 * j, "60M", "*" if j else refs[c][100:160], 0))
        cut = len(recs)
        for j in range(4):
            recs.append(sam("split", 272 if j else 16, c, 300 + 40 * j, "60M", "*" if j else refs[c][300:360], 0))
        return cut

    def small_groups():
        group("k32", 32, True)
        group("k33", 33, True)

    big = []

    def big_groups():
        for i, size in enumerate(sizes):
            while len(recs) % PR_BLOCK != offset % PR_BLOCK:
                single()
            big.append(dict(qname="big%d" % i, size=size, start=len(recs)))
            group("big%d" % i, size)

    if where == "first":
        big_groups()
        small_groups()
        for _ in range(filler):
            single()
        cut = split_group()
        for _ in range(filler // 4):
            single()
    else:
        for _ in range(filler):
            single()
        cut = split_group()
        small_groups()
        for _ in range(filler // 4):
            single()
        big_groups()
    texts = ["\n".join(recs[:cut]) + "\n", "\n".join(recs[cut:]) + "\n"]
    c = Case(fasta([(nm, refs[nm]) for nm in names]), texts, dict())
    c.facts = dict(groups=big, n_aln=len(recs), split_cut=cut)
    return c


def group_records(read_id):
    """(first alignment, size) of every read group of a packed batch, from its read_id array."""
    out = []
    start = 0
    for i in range(1, len(read_id) + 1):
        if i == len(read_id) or read_id[i] != read_id[i - 1]:
            out.append((start, i - start))
            start = i
    return out


def expect_global_k(read_id, good):
    """Whether k_goodk gives up its in-block count (FL_BIGGROUP) and the call repeats in global-k mode: some good record of a
    multi-record group sees more than SC_GROUP_SCAN_LIMIT records of its group outside its 256-alignment block.  This restates the
    rule of goodk_body (polish_dev.cuh: the backward and forward scans past the block, `if (++steps > SC_GROUP_SCAN_LIMIT)`);
    change the two together."""
    for start, size in group_records(read_id):
        if size < 2:
            continue
        for b0 in range(start - start % PR_BLOCK, start + size, PR_BLOCK):
            lo, hi = max(start, b0), min(start + size, b0 + PR_BLOCK)
            if size - (hi - lo) > SCAN_LIMIT and any(good[lo:hi]):
                return True
    return False


def record_good(sam_texts, max_errors=10, careful=False, **_):
    """alignment.rs goodness of every aligned record, in SAM order (the records these generators write: NM tag, M ends, ZP:Z:fail).
    --careful drops every record of a multi-record group."""
    rows = [l.split("\t") for t in sam_texts for l in t.split("\n") if l and not l.startswith("@")]
    good = []
    for i, r in enumerate(rows):
        nm = int([x for x in r[11:] if x.startswith("NM:i:")][0][5:])
        ops = re.findall(r"\d+([MIDNSHP=X])", r[5])
        ends = ops[0] in "M=" and ops[-1] in "M="
        g = ends and nm <= max_errors and "ZP:Z:fail" not in r[11:]
        if careful:
            multi = (i > 0 and rows[i - 1][0] == r[0]) or (i + 1 < len(rows) and rows[i + 1][0] == r[0])
            g = g and not multi
        good.append(g)
    return good


# ---- E. depth on a vote boundary -------------------------------------------------------------------------------------------
def seq_sum(ks):
    s = 0.0
    for k in ks:
        s += 1.0 / k
    return s


def boundary_orders(seed, ks, target, tries=20000):
    """Two SAM orders of the multiset ks: one whose sequential f64 sum of 1/k is exactly `target`, one whose sum is one ulp below."""
    import math
    rng = random.Random(seed)
    below = math.nextafter(target, 0.0)
    on = lo = None
    ks = list(ks)
    for _ in range(tries):
        rng.shuffle(ks)
        s = seq_sum(ks)
        if s == target and on is None:
            on = list(ks)
        elif s == below and lo is None:
            lo = list(ks)
        if on and lo:
            return on, lo
    raise AssertionError("no such pair of orders for %r" % (target,))


def boundary_case(d, ks, x_reads=0):
    """Like tests/test_emu_depth_boundary.write_case, with room for k > 32: position P of contig `probe` is covered by len(ks) reads,
    read i with ks[i] good alignments (the others on contig `filler`); every read over P carries base Y != draft, the first
    `x_reads` base X."""
    rng = random.Random(11)
    probe = rand_seq(rng, 400)
    flen = 20_000
    filler = rand_seq(rng, flen)
    P = 200
    others = [b for b in ACGT if b != probe[P]]
    y, x = others[0], others[1]
    fa = d / "a.fasta"
    fa.write_text(">probe\n" + probe + "\n>filler\n" + filler + "\n")
    lines = []
    j = 0
    for i, k in enumerate(ks):
        s = P - 30 + (i % 7)
        lines.append(sam("r%d" % i, 0, "probe", s, "60M", probe[s:P] + (x if i < x_reads else y) + probe[P + 1:s + 60], 1))
        for _ in range(k - 1):
            fpos = 10 + (37 * j) % (flen - 100)
            j += 1
            lines.append(sam("r%d" % i, 256, "filler", fpos, "60M", filler[fpos:fpos + 60], 0))
    s = d / "a.sam"
    s.write_text("\n".join(lines) + "\n")
    return fa, s, P
