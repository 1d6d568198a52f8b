"""FASTA + SAM cases for the one-indel fast walk of k_tile (seeded, deterministic, in the style of tests/ringgen.py).

A read whose CIGAR is aM bI cM or aM bD cM is walked in the chunk loop as two segments of one read, each at its own draft offset
(polypolish_b200/csrc/polish_dev.cuh fast_walk): A = bases [0, a - 1) (I) or [0, a) (D) at the read's start, B = the last run, b
positions back (I) or on (D).  The walk hands the read to the general walk when the homopolymer tail is longer than the last run c.

E (edges) covers, with one substitution in each segment so that a wrong draft offset changes a count:
  * boundaries a = 1 .. 72: every nibble of a word and both sides of 4-word group boundaries, for I and for D;
  * insertions of 1 to 20 bases (signature alleles up to 15 bases, compared alleles beyond), some at one locus on 6 reads;
  * deletions across a tile border, reads whose segment A ends before the tile (they start in the look-back bin) and reads
    whose segment B lies past the tile's end;
  * last runs c = 1 .. 8 with homopolymer tails of c - 1, c and c + 1 bases (the last one goes to the general walk);
  * reads with 2 and 3 alignments (k > 1), and a tile dense with 192-base one-indel reads (several per chunk, lane 31 among them).
Q (queue): a tile with more general-walk reads (two indels) than the queue holds, among one-indel and plain reads.

Each builder returns a fuzzgen.Case with `facts`: the kind of every alignment (SAM order), its start and its read length.
"""
import random

from tests.fuzzgen import Case
from tests.limitgen import fasta, rand_seq, sam

BIN = 256                  # PP_BIN
TILE = 2048                # TL_T
QCAP = 1024                # TL_QCAP


def _mutate(rng, b):
    return rng.choice([x for x in "ACGT" if x != b])


def tail_run(seq):
    """How many of the last bases equal the last one."""
    n = 1
    while n < len(seq) and seq[-1 - n] == seq[-1]:
        n += 1
    return n


class _Builder:
    def __init__(self, rng, truth):
        self.rng, self.truth = rng, truth
        self.groups = []                                  # (kind, [(start, cigar, seq, nm)])

    def plain(self, kind, start, length):
        s = list(self.truth[start:start + length])
        i = self.rng.randint(0, length - 12)
        s[i] = _mutate(self.rng, s[i])
        self.groups.append((kind, [(start, "%dM" % length, "".join(s), 1)]))

    def one_indel(self, kind, start, a, b, c, is_del, ins=None, tail=None, others=()):
        """aM bI cM (ins: the inserted bases) / aM bD cM at `start`, one substitution in each segment; tail = r: the last r bases
        equal, the base before them not; others: starts of more alignments of the same read (k > 1)."""
        rng, t = self.rng, self.truth
        if is_del:
            s = list(t[start:start + a] + t[start + a + b:start + a + b + c])
            b_lo = a                                      # segment B in read bases
        else:
            ins = ins if ins is not None else rand_seq(rng, b)
            assert len(ins) == b
            s = list(t[start:start + a] + ins + t[start + a:start + a + c])
            b_lo = a + b
        nm = b
        for lo, hi in ((0, a - (0 if is_del else 1)), (b_lo, len(s) - 9 if c >= 12 else b_lo + 1)):
            if hi > lo and not (tail and hi > len(s) - tail - 1):
                i = rng.randint(lo, hi - 1)
                s[i] = _mutate(rng, s[i])
                nm += 1
        if tail:
            x = rng.choice("ACGT")
            s[len(s) - tail:] = x * tail
            if tail < len(s):
                s[len(s) - tail - 1] = _mutate(rng, x)
            assert tail_run(s) == tail
        cig = "%dM%d%s%dM" % (a, b, "D" if is_del else "I", c)
        self.groups.append((kind, [(p, cig, "".join(s), min(nm, 10)) for p in (start,) + tuple(others)]))

    def two_indel(self, kind, start):
        """aM bI cM dD eM: the general walk."""
        rng, t = self.rng, self.truth
        a, b, c, d, e = rng.randint(5, 40), rng.randint(1, 3), rng.randint(5, 40), rng.randint(1, 3), rng.randint(9, 40)
        s = t[start:start + a] + rand_seq(rng, b) + t[start + a:start + a + c] + t[start + a + c + d:start + a + c + d + e]
        self.groups.append((kind, [(start, "%dM%dI%dM%dD%dM" % (a, b, c, d, e), s, b + d)]))


def _genome(rng, n_tiles):
    truth = rand_seq(rng, n_tiles * TILE)
    draft = list(truth)
    for p in range(30, len(draft) - 30, 97):
        q = p + rng.randint(0, 40)
        draft[q] = _mutate(rng, draft[q])
    return truth, "".join(draft)


def _background(B, n_tiles, depth=8):
    rng = B.rng
    n = n_tiles * TILE * depth // 120
    for _ in range(n):
        length = rng.randint(60, 180)
        B.plain("plain", rng.randint(0, n_tiles * TILE - length - 1), length)


def _emit(B, rng, facts):
    order = list(range(len(B.groups)))
    rng.shuffle(order)                                    # SAM order within a bin is the slot order: not position order
    lines, kinds, starts, lens = [], [], [], []
    for gi, g in enumerate(order):
        kind, recs = B.groups[g]
        for j, (start, cig, seq, nm) in enumerate(recs):
            flag = (16 if (gi + j) % 2 else 0) | (256 if j else 0)
            lines.append(sam("r%d" % gi, flag, "indel", start, cig, seq, nm))
            kinds.append(kind)
            starts.append(start)
            lens.append(len(seq))
    facts.update(kinds=kinds, starts=starts, lens=lens)
    case = Case(fasta([("indel", B.draft)]), ["\n".join(lines) + "\n"], {})
    case.facts = facts
    return case


def edges(seed):
    """E: eight tiles; see the module's docstring."""
    rng = random.Random(seed)
    n_tiles = 8
    truth, draft = _genome(rng, n_tiles)
    B = _Builder(rng, truth)
    B.draft = draft
    # tile 1: the boundary at every base of the first three words and around the group boundaries (32 and 64 bases)
    for a in range(1, 73):
        for is_del in (False, True):
            b = rng.randint(1, 3) if rng.random() < 0.7 else rng.randint(4, 12)
            c = rng.randint(9, 190 - a - b) if not is_del else rng.randint(9, 192 - a)
            B.one_indel("boundary", TILE + rng.randint(0, TILE - BIN - 1), a, b, c, is_del)
    # tile 2: insertions of 1 .. 20 bases; three of them on 6 reads at one locus each (an allele that reaches the vote)
    for n in range(1, 21):
        for _ in range(3):
            a = rng.randint(1, 90)
            B.one_indel("ins_len", 2 * TILE + rng.randint(0, TILE - BIN - 1), a, n, rng.randint(9, 190 - a - n), False)
    for n in (3, 15, 20):
        locus = 2 * TILE + rng.randint(0, TILE - BIN - 200)
        ins = rand_seq(rng, n)
        for _ in range(6):
            a = rng.randint(2, 60)
            B.one_indel("ins_locus", locus - a, a, n, rng.randint(20, 100), False, ins=ins)
    # deletions that cross the border of tiles 2 | 3 (its end, and tile 3's start) at every offset
    P = 3 * TILE
    for b in (1, 2, 5, 12):
        for x in range(b):
            a = rng.randint(1, 100)
            B.one_indel("del_border", P - x - a, a, b, rng.randint(9, 90), True)
    # segment A before tile 4's start (the read starts in the look-back bin), segment B past tile 3's end (the same reads), and
    # segment B past tile 5's end
    P = 4 * TILE
    for i in range(24):
        is_del = i % 2 == 1
        a, b = rng.randint(10, 120), rng.randint(1, 6)
        # A ends at P - 1 or before; B starts at P or just before it (I), or the deletion reaches P or past it (D)
        start = P - a - rng.randint(0, b) if is_del else P - a - rng.randint(0, 2)
        B.one_indel("a_before", start, a, b, rng.randint(9, 60), is_del)
    P = 6 * TILE
    for i in range(16):
        a = rng.randint(20, 100)
        B.one_indel("b_past", P - a - rng.randint(0, 3), a, rng.randint(1, 4), rng.randint(9, 60), i % 2 == 1)
    # tile 4: last runs c = 1 .. 8 with tails of c - 1, c and c + 1 equal bases
    for c in range(1, 9):
        for tail in (c - 1, c, c + 1):
            if tail < 1:
                continue
            for is_del in (False, True):
                for _ in range(2):
                    a = rng.randint(20, 150)
                    B.one_indel("tail_c%d_r%d" % (c, tail), 4 * TILE + rng.randint(0, TILE - BIN - 1), a, rng.randint(1, 4), c, is_del,
                                tail=tail)
    # tile 4: reads with 2 or 3 alignments (the others in tiles 6 and 7)
    for i in range(30):
        a, b, c = rng.randint(1, 80), rng.randint(1, 5), rng.randint(9, 80)
        others = tuple(t * TILE + rng.randint(0, TILE - BIN - 1) for t in ((6,) if i % 2 else (6, 7)))
        B.one_indel("multi%d" % (1 + len(others)), 4 * TILE + rng.randint(0, TILE - BIN - 1), a, b, c, i % 3 == 0, others=others)
    # tile 5: dense with 192-base one-indel reads
    for i in range(160):
        is_del = i % 2 == 0
        a = rng.randint(1, 180)
        b = rng.randint(1, min(11, 191 - a)) if not is_del else rng.randint(1, 30)
        c = 192 - a - (0 if is_del else b)
        B.one_indel("len192", 5 * TILE + rng.randint(0, TILE - BIN - 1 - 40), a, b, c, is_del)
    _background(B, n_tiles)
    return _emit(B, rng, dict(n_tiles=n_tiles))


def queue_general(seed, n_two=1100):
    """Q: three tiles; the middle one has n_two two-indel reads (the general walk: more than TL_QCAP, so the rest are walked in
    place) among one-indel and plain reads."""
    rng = random.Random(seed)
    truth, draft = _genome(rng, 3)
    B = _Builder(rng, truth)
    B.draft = draft
    for _ in range(n_two):
        B.two_indel("indel2", TILE + rng.randint(0, TILE - BIN - 1))
    for _ in range(300):
        a = rng.randint(1, 60)
        B.one_indel("indel", TILE + rng.randint(0, TILE - BIN - 1), a, rng.randint(1, 3), rng.randint(9, 100), rng.random() < 0.5)
    _background(B, 3)
    return _emit(B, rng, dict(n_tiles=3, n_two=n_two))
