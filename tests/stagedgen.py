"""FASTA + SAM cases for the staged general walk of k_tile (seeded, deterministic, in the style of tests/indelgen.py).

A 4-bit read of at most 192 bases that the fast walk does not take (two or more indels, X ops, long homopolymer tails) is walked
by the general walk in the chunk loop, from the slot's copy of its bases in the chunk ring (polypolish_b200/csrc/polish_dev.cuh,
TR_STAGED / StagedBases).  Only longer reads and the 8-bit pool still go to the queue after the chunk loop.

S (staged) covers, with one substitution in every match run so that a wrong draft offset changes a count:
  * reads with 2 - 6 indels in random orders, I right after D and D right after I among them, and X / = ops mixed with M;
  * the first indel after a = 1 .. 72 bases: every nibble of a word and both sides of 4-word group boundaries;
  * insertions of 1 to 20 bases (signature alleles up to 15 bases, compared alleles beyond), some at one locus on 6 reads;
  * deletions across the border of tiles 2 | 3, and reads that start in the bin before tile 4 (the look-back);
  * plain reads with homopolymer tails of 8 - 20 bases, and tails that cross one or more indels: through an `xD 1I` pair (the
    trim counts the inserted base on the deletion's last entry) and stopped by an I or a D;
  * reads of exactly 192 bases (staged) and of 193 (queued), a tile dense with 192-base many-indel reads (several per chunk,
    lane 31 among them, one warp drawing many);
  * reads with 2 and 3 alignments (k > 1).
Q (queue): a tile with more 193 - 200-base two-indel reads (not staged: the queue) than the queue holds.
B (8-bit): a smaller S whose batch goes to the 8-bit pool (one read carries a byte outside the 16 BAM codes): everything queued.
"""
import random

from tests.fuzzgen import Case
from tests.indelgen import BIN, QCAP, TILE, _background, _genome, _mutate, tail_run  # noqa: F401
from tests.limitgen import fasta, rand_seq, sam

STAGED_LEN = 192           # TL_FAST_LEN


class _Builder:
    def __init__(self, rng, truth):
        self.rng, self.truth = rng, truth
        self.groups = []                                  # (kind, [(start, cigar, seq, nm)])

    def read(self, kind, start, ops, tail=None, others=(), ins=None):
        """ops = [(op, n)] with op in M = X I D: the read the truth gives at `start` (X: a mismatch, I: random bases or `ins`), one
        substitution in every M / = run outside the tail; tail = r: the last r bases equal, the base before them not; others:
        starts of more alignments of the same read (k > 1).  Returns the reference span."""
        rng, t = self.rng, self.truth
        s, runs, p, nm = [], [], start, 0
        for op, n in ops:
            if op in "M=X":
                seg = list(t[p:p + n])
                if op == "X":
                    seg = [_mutate(rng, b) for b in seg]
                    nm += n
                else:
                    runs.append((len(s), len(s) + n))
                s += seg
                p += n
            elif op == "I":
                s += list(ins if ins is not None else rand_seq(rng, n))
                nm += n
            else:
                p += n
                nm += n
        keep = len(s) - (tail + 1 if tail else 0)
        for lo, hi in runs:
            hi = min(hi, keep)
            if hi - lo >= 2:
                i = rng.randint(lo, hi - 1)
                s[i] = _mutate(rng, s[i])
                nm += 1
        if tail:
            x = rng.choice("ACGT")
            s[len(s) - tail:] = x * tail
            if tail < len(s):
                s[len(s) - tail - 1] = _mutate(rng, x)
            assert tail_run(s) == tail
        cig = "".join("%d%s" % (n, op) for op, n in ops)
        self.groups.append((kind, [(q, cig, "".join(s), min(nm, 10)) for q in (start,) + tuple(others)]))
        return p - start

    def plain(self, kind, start, length):                 # (indelgen's background reads)
        self.read(kind, start, [("M", length)])


def _indels(rng, n, length, first=None, first_op=None, adjacent=False, max_ins=3):
    """ops of a read of `length` bases with n indels between match runs (the first after `first` bases when given); adjacent: one
    D right before an I or one I right before a D, with no match run between them."""
    kinds = [first_op or rng.choice("ID")] + [rng.choice("ID") for _ in range(n - 1)]
    glue = -1                                             # indel `glue` is followed directly by indel glue + 1
    if adjacent and n >= 2:
        glue = rng.randint(0, n - 2)
        kinds[glue + 1] = "I" if kinds[glue] == "D" else "D"
    sizes = [rng.randint(1, max_ins) for _ in kinds]
    m = length - sum(z for k, z in zip(kinds, sizes) if k == "I")
    n_runs = n + 1 - (glue >= 0)
    if first is not None:
        first = min(first, m - (n_runs - 1))
        cuts = [first] + sorted(first + c for c in rng.sample(range(1, m - first), n_runs - 2))
    else:
        cuts = sorted(rng.sample(range(1, m), n_runs - 1))
    runs = [b - a for a, b in zip([0] + cuts, cuts + [m])]
    ops, r = [("M", runs[0])], 1
    for j, (k, z) in enumerate(zip(kinds, sizes)):
        ops.append((k, z))
        if j != glue:
            ops.append(("M", runs[r]))
            r += 1
    return ops


def _span(ops):
    return sum(n for op, n in ops if op in "M=XD")


def _mixed_ops(rng, ops):
    """Some M runs split into M / = / X pieces."""
    out = []
    for op, n in ops:
        if op == "M" and n >= 6 and rng.random() < 0.6:
            a = rng.randint(1, n - 4)
            b = rng.randint(1, 2)
            out += [("M", a), ("X", b), ("=", n - a - b)]
        else:
            out.append((op, n))
    return out


def _emit(B, rng, name, facts, eight_bit=False):
    order = list(range(len(B.groups)))
    rng.shuffle(order)                                    # SAM order within a bin is the slot order: not position order
    lines, kinds, starts, lens, cigars = [], [], [], [], []
    for gi, g in enumerate(order):
        kind, recs = B.groups[g]
        for j, (start, cig, seq, nm) in enumerate(recs):
            flag = (16 if (gi + j) % 2 else 0) | (256 if j else 0)
            lines.append(sam("r%d" % gi, flag, name, start, cig, seq, nm))
            kinds.append(kind)
            starts.append(start)
            lens.append(len(seq))
            cigars.append(cig)
    if eight_bit:                                         # a byte outside "=ACMGRSVTWYHKDBN": the batch goes to the 8-bit pool
        a = kinds.index("plain")
        f = lines[a].split("\t")
        f[9] = f[9][:5] + "." + f[9][6:]
        lines[a] = "\t".join(f)
    facts.update(kinds=kinds, starts=starts, lens=lens, cigars=cigars, seq_bits=8 if eight_bit else 4)
    case = Case(fasta([(name, B.draft)]), ["\n".join(lines) + "\n"], {})
    case.facts = facts
    return case


def staged(seed, eight_bit=False, scale=1):
    """S (and B with eight_bit, scale < 1: fewer reads of each kind); see the module's docstring."""
    rng = random.Random(seed)
    n_tiles = 8
    truth, draft = _genome(rng, n_tiles)
    B = _Builder(rng, truth)
    B.draft = draft
    cnt = lambda n: max(1, int(n * scale))
    # tile 1: the first indel after every base of the first three words and around the group boundaries (32 and 64 bases)
    for a in range(1, 73):
        for op in "ID":
            if scale < 1 and a % 4:
                continue
            n = rng.randint(2, 6)
            length = rng.randint(max(a + 40, 60), STAGED_LEN)
            ops = _indels(rng, n, length, first=a, first_op=op)
            B.read("boundary", TILE + rng.randint(0, TILE - BIN - 1), ops)
    # tile 2: 2 - 6 indels in random orders, adjacent D / I pairs, X and = ops, insertions of 1 .. 20 bases (three at one locus)
    for _ in range(cnt(120)):
        n = rng.randint(2, 6)
        ops = _indels(rng, n, rng.randint(60, STAGED_LEN), adjacent=rng.random() < 0.5)
        B.read("order", 2 * TILE + rng.randint(0, TILE - BIN - 1), ops)
    for _ in range(cnt(40)):
        ops = _mixed_ops(rng, _indels(rng, rng.randint(1, 4), rng.randint(60, STAGED_LEN)))
        B.read("xeq", 2 * TILE + rng.randint(0, TILE - BIN - 1), ops)
    for n in range(1, 21):
        for _ in range(cnt(3)):
            op2, z = rng.choice("ID"), rng.randint(1, 3)
            m = rng.randint(30, STAGED_LEN - n - (z if op2 == "I" else 0))
            x, y = sorted(rng.sample(range(1, m), 2))
            ops = [("M", x), ("I", n), ("M", y - x), (op2, z), ("M", m - y)]
            B.read("ins_len", 2 * TILE + rng.randint(0, TILE - BIN - 1), ops)
    for n in (3, 15, 20):
        locus = 2 * TILE + rng.randint(200, TILE - BIN - 200)
        ins = rand_seq(rng, n)
        for _ in range(6):
            a = rng.randint(2, 60)
            ops = [("M", a), ("I", n), ("M", rng.randint(20, 60)), ("D", rng.randint(1, 3)), ("M", rng.randint(9, 40))]
            B.read("ins_locus", locus - a, ops, ins=ins)
    # deletions that cross the border of tiles 2 | 3 at every offset, in reads with more indels
    P = 3 * TILE
    for b in (1, 2, 5, 12):
        for x in range(b):
            a = rng.randint(10, 80)
            ops = [("M", a), ("D", b), ("M", rng.randint(10, 40)), (rng.choice("ID"), rng.randint(1, 3)), ("M", rng.randint(9, 40))]
            B.read("del_border", P - x - a, ops)
    # tile 4: reads that start in the bin before it; plain reads with tails of 8 - 20 bases; tails that cross indels
    P = 4 * TILE
    for _ in range(cnt(24)):
        ops = _indels(rng, rng.randint(2, 4), rng.randint(80, STAGED_LEN))
        span = _span(ops)
        B.read("lookback", P - rng.randint(1, min(BIN - 1, span - 1)), ops)
    for tail in range(8, 21):
        for _ in range(cnt(3)):
            length = rng.randint(tail + 20, STAGED_LEN)
            B.read("tail_plain", P + rng.randint(0, TILE - BIN - 1), [("M", length)], tail=tail)
    for c in range(1, 7):
        for _ in range(cnt(2)):
            a = rng.randint(20, 100)
            # through an xD 1I pair (one or two of them): the trim takes the inserted base and goes on into the run before
            ops = [("M", a), ("D", 1), ("I", 1), ("M", c)]
            B.read("tail_di", P + rng.randint(0, TILE - BIN - 1), ops, tail=c + 1 + rng.randint(1, 5))
            ops = [("M", a), ("D", 1), ("I", 1), ("M", 3), ("D", 1), ("I", 1), ("M", c)]
            B.read("tail_di2", P + rng.randint(0, TILE - BIN - 1), ops, tail=c + 5 + rng.randint(1, 5))
            # stopped by a D of 2+ bases before the inserted base, by a plain I, by a plain D
            ops = [("M", a), ("D", 2), ("I", 1), ("M", c)]
            B.read("tail_d2i", P + rng.randint(0, TILE - BIN - 1), ops, tail=c + 1 + rng.randint(1, 5))
            for op in "ID":
                ops = [("M", a), (op, rng.randint(1, 3)), ("M", rng.randint(10, 30)), (op, rng.randint(1, 3)), ("M", c)]
                B.read("tail_" + op, P + rng.randint(0, TILE - BIN - 1), ops, tail=min(c + rng.randint(1, 8), 30))
    # tile 4: reads with 2 or 3 alignments (the others in tiles 6 and 7)
    for i in range(cnt(30)):
        ops = _indels(rng, rng.randint(2, 4), rng.randint(60, STAGED_LEN))
        others = tuple(t * TILE + rng.randint(0, TILE - BIN - 1) for t in ((6,) if i % 2 else (6, 7)))
        B.read("multi%d" % (1 + len(others)), P + rng.randint(0, TILE - BIN - 1), ops, others=others)
    # tile 5: dense with 192-base many-indel reads, and some of 193 bases (the queue)
    for i in range(cnt(200)):
        ops = _indels(rng, rng.randint(2, 6), STAGED_LEN, adjacent=i % 3 == 0)
        B.read("len192", 5 * TILE + rng.randint(0, TILE - BIN - 1 - 60), ops)
    for i in range(cnt(12)):
        ops = _indels(rng, rng.randint(1, 3), STAGED_LEN + 1)
        B.read("len193", 5 * TILE + rng.randint(0, TILE - BIN - 1 - 60), ops)
    _background(B, n_tiles)
    kinds = [k for k, _ in B.groups]
    assert all(sum(n for op, n in _ops(recs[0][1]) if op in "MI=X") == len(recs[0][2]) for _, recs in B.groups), kinds
    return _emit(B, rng, "staged", dict(n_tiles=n_tiles), eight_bit=eight_bit)


def _ops(cig):
    out, n = [], ""
    for ch in cig:
        if ch.isdigit():
            n += ch
        else:
            out.append((ch, int(n)))
            n = ""
    return out


def queue_long(seed, n_long=1100):
    """Q: three tiles; the middle one has n_long two-indel reads of 193 - 200 bases (not staged: more than TL_QCAP, so the rest are
    walked in place from the pool) among staged many-indel reads and plain reads."""
    rng = random.Random(seed)
    truth, draft = _genome(rng, 3)
    B = _Builder(rng, truth)
    B.draft = draft
    for _ in range(n_long):
        ops = _indels(rng, 2, rng.randint(STAGED_LEN + 1, 200))
        B.read("long2", TILE + rng.randint(0, TILE - BIN - 1), ops)
    for _ in range(300):
        ops = _indels(rng, rng.randint(2, 5), rng.randint(60, STAGED_LEN))
        B.read("staged", TILE + rng.randint(0, TILE - BIN - 1), ops)
    _background(B, 3)
    return _emit(B, rng, "staged", dict(n_tiles=3, n_long=n_long))
