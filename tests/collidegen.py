"""Strings whose 64-bit keys collide, and the FASTA + SAM cases that put them where the device path compares keys before bytes.

The device path takes two strings as equal when their keys are equal, then confirms the bytes:
  * polish tokeniser: RNAME -> contig through the FNV-1a 64 table of the contig names (tok_line.h parse_line, tok_table.h);
  * `filter` on one context: QNAMEs and RNAMEs (RNAME keys xor REF_DOMAIN) interned in one table, confirmed by k_ftok_verify;
  * `filter` over N contexts: every QNAME goes to the context its key picks and is interned there again, confirmed by k_fx_verify;
  * k_tile's other alleles: make_sig (polish_dev.cuh), 60 bits (4-bit bases) or 56 bits (8-bit) of FNV-1a over the allele's
    symbols xor its length, confirmed by allele_equal.
Random strings never collide in 64 bits, so without these pairs the byte checks never see two different strings.  Each pair was
found by tests/manual/fnv_collide.c (a rho search with distinguished points, deterministic for a seed); the command beside each
constant prints it again.  FNV-1a keeps a collision when the same bytes follow, so NAME_A + s and NAME_B + s collide for any s.

Every case has a twin in which the colliding string is replaced by its partner, so the two are really one string; the tests check
that the oracle's answer for the twin differs from the case's, so a case would fail if the byte check it targets were skipped.
"""
import random

from tests.fuzzgen import Case
from tests.limitgen import fasta, rand_seq, sam

FNV_BASIS, FNV_PRIME, MASK = 14695981039346656037, 1099511628211, (1 << 64) - 1
REF_DOMAIN = 0x9E3779B97F4A7C15          # tok_kernels.cu: RNAME keys live in the filter's intern table xor this

# name pair                                           gcc -O3 -pthread -o fnv_collide tests/manual/fnv_collide.c
NAME_A, NAME_B = "PmxVHU8Ar4H", "W0y7AQw62nK"        # ./fnv_collide name
JOUX_C, JOUX_D = "rC2dP8X5IH5", "8TEJ8yD3Zz3"        # ./fnv_collide name PmxVHU8Ar4H  (the pair that follows NAME_A: a 4-way set)
CLAW_Q, CLAW_R = "TK1YMlSORMI", "YGJsCo1hTAD"        # ./fnv_collide claw      fnv(CLAW_Q) == fnv(CLAW_R) ^ REF_DOMAIN
SIG4 = ("ACAATCCCCCGGCGAAAATATTTATAGAGTT", "AAGCTGTCACCTTTTACCCGTCTGAAGTGCA")    # ./fnv_collide sig 4 A    31 bases (4-bit)
SIG8 = ("ACCCGAACCGTTCCCGCACGGCGAGTCTT", "ATGCTTCACGGATAAGGTTGAATTTCTAT")       # ./fnv_collide sig 8 A    29 bytes (8-bit)
SIG8_LEN = ("AAAACGCCACGGGCCGACTTCGCCTGTGT", "ATTACGTCAGCGGGGGATTACAGGCTGTCA")  # ./fnv_collide sig 8 A 1  29 and 30 bytes
REGEN = {"name": "fnv_collide name", "joux": "fnv_collide name " + NAME_A, "claw": "fnv_collide claw", "sig4": "fnv_collide sig 4 A",
         "sig8": "fnv_collide sig 8 A", "sig8_len": "fnv_collide sig 8 A 1"}
JOUX = [NAME_A + JOUX_C, NAME_A + JOUX_D, NAME_B + JOUX_C, NAME_B + JOUX_D]


def fnv1a(b):
    h = FNV_BASIS
    for c in b.encode() if isinstance(b, str) else b:
        h = ((h ^ c) * FNV_PRIME) & MASK
    return h


def sig(allele, bits):
    """make_sig of an allele longer than the exact limit (4-bit symbols: the BAM codes A=1 C=2 G=4 T=8; 8-bit: the bytes)."""
    code = {"A": 1, "C": 2, "G": 4, "T": 8}
    h = FNV_BASIS
    for c in allele:
        h = ((h ^ (code[c] if bits == 4 else ord(c))) * FNV_PRIME) & MASK
    return ((h ^ len(allele)) << (4 if bits == 4 else 8)) & MASK


def rc(s):
    return s[::-1].translate(str.maketrans("ACGTN", "TGCAN"))


def _draft(rng, truth, step=97):
    d = list(truth)
    for p in range(40, len(d) - 40, step):
        d[p] = rng.choice([x for x in "ACGT" if x != d[p]])
    return "".join(d)


# ---- A. contig names ------------------------------------------------------------------------------------------------------------
def contig_case(order="ab", only=None, twin=False, seed=1, length=2000, depth=12):
    """Contigs NAME_A and NAME_B (in FASTA order `order`), reads on each that turn its draft errors back into its truth.  only="a":
    the assembly holds NAME_A alone and the reads of NAME_B name a contig it does not have (the reference's error).  The twin's
    reads of NAME_B name NAME_A."""
    rng = random.Random(seed)
    truth = {"a": rand_seq(rng, length), "b": rand_seq(rng, length)}
    names = {"a": NAME_A, "b": NAME_B}
    contigs = [(names[k], _draft(rng, truth[k])) for k in order if only in (None, k)]
    lines, n = [], 0
    for k in "ab":
        rname = NAME_A if (twin and k == "b") else names[k]
        for start in range(0, length - 100, 100 // depth * 1 + 7):
            s = truth[k][start:start + 100]
            lines.append(sam("r%d" % n, 16 if n % 2 else 0, rname, start, "100M", s, 1))
            n += 1
    order_lines = list(range(len(lines)))
    rng.shuffle(order_lines)
    case = Case(fasta(contigs), ["\n".join(lines[i] for i in order_lines) + "\n"], {})
    case.facts = dict(order=order, only=only)
    return case


# ---- B - D. filter ---------------------------------------------------------------------------------------------------------------
FILTER_KINDS = ("one_file", "two_files", "rname", "claw", "joux")
C1_LEN, SMALL_LEN = 60_000, 3_000


def filter_case(kind, twin=False, seed=7, n_pairs=300):
    """Paired SAM files on contig c1 (pairs fr, insert about 300) with records of colliding strings: the first colliding QNAME is the
    first record of file 1, its partner the last record of file 1 (one_file) or of file 2 (two_files, joux), so that over N contexts
    they lie in the first and the last byte range.  Separate strings and merged ones give different verdicts:
      one_file   A is a good pair (A1, A2); B1 alone far away.  Merged, B1 is a second alignment of A in file 1 and fails.
      two_files  A has two alignments in file 1, B one in file 2: reads without mates pass.  Merged, A's fail (no good pair with B).
      rname      mate 1 on contig NAME_A and on c1, mate 2 on NAME_B: no pair on one contig, both mate-1 records fail.  Merged, the
                 NAME_A record and mate 2 are a good pair.
      claw       a read named CLAW_Q next to a contig named CLAW_R: one intern slot, a QNAME and an RNAME.
      joux       the four names of the 4-way set, two alone in file 1, two alone in file 2.
    The assembly (for filter-polish) holds c1, NAME_A, NAME_B and CLAW_R.  twin: every colliding string replaced by the first of its set."""
    rng = random.Random(seed)
    truth = {"c1": rand_seq(rng, C1_LEN), NAME_A: rand_seq(rng, SMALL_LEN), NAME_B: rand_seq(rng, SMALL_LEN), CLAW_R: rand_seq(rng, SMALL_LEN)}

    def rec(name, flag, ref, pos, length=100):
        return sam(name, flag, ref, pos, "%dM" % length, truth[ref][pos:pos + length], 1)

    l1, l2 = [], []
    for i in range(n_pairs):
        a = rng.randint(0, C1_LEN - 800)
        ins = max(150, int(rng.gauss(300, 8)))
        l1.append(rec("p%d" % i, 0, "c1", a))
        l2.append(rec("p%d" % i, 16, "c1", a + ins - 100))
    rng.shuffle(l2)
    same = (lambda x: NAME_A) if twin else (lambda x: x)
    first1, last1, first2, last2 = [], [], [], []
    if kind == "one_file":
        first1.append(rec(NAME_A, 0, "c1", 1000))
        first2.append(rec(NAME_A, 16, "c1", 1200))
        last1.append(rec(same(NAME_B), 0, "c1", 40_000))
    elif kind == "two_files":
        first1 += [rec(NAME_A, 0, "c1", 1000), rec(NAME_A, 256, "c1", 45_000)]
        last2.append(rec(same(NAME_B), 0, "c1", 30_000))
    elif kind == "rname":
        first1 += [rec("x1", 0, NAME_A, 1000), rec("x1", 256, "c1", 20_000)]
        last2.append(rec("x1", 16, same(NAME_B), 1200))
    elif kind == "claw":
        first1.append(rec(CLAW_Q, 0, "c1", 1000))
        last1.append(rec("x2", 0, CLAW_R, 500))
        last2.append(rec("x2", 16, CLAW_R, 700))
    elif kind == "joux":
        j = [JOUX[0]] * 4 if twin else JOUX
        first1.append(rec(j[0], 0, "c1", 1000))
        last1.append(rec(j[3], 0, "c1", 50_000))
        first2.append(rec(j[1], 0, "c1", 20_000))
        last2.append(rec(j[2], 16, "c1", 10_000))
    head = "@HD\tVN:1.6\n@SQ\tSN:c1\tLN:%d\n" % C1_LEN
    t1 = head + "\n".join(first1 + l1 + last1) + "\n"
    t2 = head + "\n".join(first2 + l2 + last2) + "\n"
    contigs = [(k, _draft(rng, v)) for k, v in truth.items()]
    case = Case(fasta(contigs), [t1, t2], {})
    case.facts = dict(kind=kind, first=t1.index("\n", len(head)) if first1 else None)
    return case


def verdicts(text):
    """Per record of a filtered SAM file: did it fail (the filter's ZP:Z:fail tag)?"""
    return [x.endswith(b"\tZP:Z:fail") for x in text.split(b"\n") if x and not x.startswith(b"@")]


# ---- E. other alleles ------------------------------------------------------------------------------------------------------------
P, CONTIG_LEN = 1500, 3200
KINDS = ("fast", "staged", "long", "escape")


def allele_case(counts, pair, bits=4, twin=False, seed=3, multi=()):
    """One contig; position P (draft base A) covered only by reads whose insertion after P makes the allele pair[0] (counts[0]
    reads) or pair[1] (counts[1] reads), in SAM order A, B, A, B, ...  Read i is walked as KINDS[i % 4] (the fast one-indel walk; a
    second indel and an X, so the staged general walk; more than 192 bases, so the queue; an N far from P, so an escape), on
    strand i % 2.  Reads whose index is in `multi` have a SEQ=* secondary far from P (k = 2).  bits=8: one read elsewhere carries a
    byte outside the 4-bit alphabet, so the dataset is 8-bit.  twin: every read carries pair[0]."""
    rng = random.Random(seed)
    truth = list(rand_seq(rng, CONTIG_LEN))
    truth[P] = "A"
    truth = "".join(truth)
    assert pair[0][0] == pair[1][0] == "A"
    lines = []
    order = []
    na, nb = counts
    i = j = 0
    while i < na or j < nb:
        if i < na:
            order.append(0); i += 1
        if j < nb:
            order.append(1); j += 1
    for n, which in enumerate(order):
        ins = (pair[0] if twin else pair[which])[1:]
        kind = KINDS[n % 4]
        left = rng.randint(30, 90) if kind != "long" else rng.randint(120, 160)
        right = rng.randint(30, 90) if kind != "long" else rng.randint(60, 100)
        s0 = P + 1 - left
        pre = truth[s0:P + 1]
        post = truth[P + 1:P + 1 + right]
        if kind == "staged":
            cut = right // 2
            post = post[:cut] + truth[P + 1 + cut + 2:P + 1 + right + 2]
            xs = list(pre)
            xs[5] = rng.choice([c for c in "ACGT" if c != xs[5]])
            pre = "".join(xs)
            cigar = "5=1X%d=%dI%dM2D%dM" % (left - 6, len(ins), cut, right - cut)
        else:
            cigar = "%dM%dI%dM" % (left, len(ins), right)
        if kind == "escape":
            post = post[:-10] + "N" + post[-9:]
        seq = pre + ins + post
        assert kind != "long" or len(seq) > 192
        flag = 16 if n % 2 else 0
        lines.append(sam("q%d" % n, flag, "ctg", s0, cigar, seq, 1))
        if n in multi:
            lines.append(sam("q%d" % n, flag | 256, "ctg", s0 + 1400, cigar, "*", 1))
    if bits == 8:
        s = truth[200:300]
        lines.append(sam("z8", 0, "ctg", 200, "100M", s[:50] + "Z" + s[51:], 1))
    case = Case(fasta([("ctg", _draft(rng, truth))]), ["\n".join(lines) + "\n"], {})
    case.facts = dict(P=P, order=order)
    return case


def row(debug_tsv, pos):
    """The --debug row of a position (header first)."""
    return debug_tsv.split(b"\n")[1 + pos].split(b"\t")
