"""FASTA + SAM cases for the 2-bit staged reads of k_tile (seeded, deterministic, in the style of tests/stagedgen.py).

The chunk loop reads a staged read's bases as 2-bit codes (k_permute_seq: the effective read, reverse complement applied, 16 bases per
32-bit word) and compares them with a 2-bit copy of the draft plus a mask of the draft positions that are not A/C/G/T; a read with a
base other than A/C/G/T is an escape, walked in place from the 4-bit pool (polypolish_b200/csrc/polish_dev.cuh: TR_ESC, `dn2`).

T covers, with the polished output and every count of --debug depending on each of them:
  * tile 1: plain reads of 150 and 192 bases with one substitution at read index i for every i < 192 (every field of a 16-base word,
    both sides of the 64-base group boundaries), starting at every residue mod 16 of the tile; one-indel reads with insertions of
    1 - 20 bases and deletions; reads with 2 - 6 indels.  Every other read is a reverse-strand primary whose `SEQ=*` secondary lies
    on tile 3, a reverse-complement copy of tile 1's region: there the effective read is the primary's reverse complement, and the
    secondaries alone carry the votes that turn tile 3's draft errors back into the truth (a wrong complement or shift flips them);
  * tile 4: draft positions with IUPAC codes, N, `-` and lower case under plain, one-indel and many-indel reads;
  * tile 5: escape reads (an N or IUPAC base) of every walk kind, dense enough for several per chunk and lane 31, with k = 2 and 3,
    192-base reads among them; and 192-base plain reads (lane 31).
No read is longer than 192 bases: nothing goes to the queue.
"""
import random

from tests.fuzzgen import Case
from tests.indelgen import BIN, TILE, _mutate
from tests.limitgen import fasta, rand_seq, sam
from tests.stagedgen import STAGED_LEN, _indels

N_TILES = 7
IUPAC = "NRYSWKMBDHV"
_COMP = str.maketrans("ACGTNRYSWKMBDHV", "TGCANYRSWMKVHDB")
R1, W = TILE + 64, 1400                                  # tile 1's region and its reverse-complement copy on tile 3
R3 = 3 * TILE + 64


def rc(s):
    return s[::-1].translate(_COMP)


def _ops_str(ops):
    return "".join("%d%s" % (n, op) for op, n in ops)


def _span(ops):
    return sum(n for op, n in ops if op in "MD")


class _Reads:
    def __init__(self, rng, truth):
        self.rng, self.truth, self.groups = rng, truth, []   # groups: (kind, [(start, cigar, seq, nm, flag)])

    def seq(self, start, ops, subs=(), esc=None):
        """The read the truth gives at `start` under ops (M / I / D; I: random bases), substitutions at read indices `subs`, and
        `esc` = (index, base) written over one base."""
        s, p = [], start
        for op, n in ops:
            if op == "M":
                s += self.truth[p:p + n]
                p += n
            elif op == "I":
                s += rand_seq(self.rng, n)
            else:
                p += n
        for i in subs:
            s[i] = _mutate(self.rng, s[i])
        if esc:
            s[esc[0]] = esc[1]
        return "".join(s)

    def add(self, kind, start, ops, subs=(), esc=None, reverse=False, mirror=False, others=()):
        """One read group.  mirror: a reverse-strand primary and its SEQ=* forward secondary on the reverse-complement copy (tile 1 ->
        tile 3); others: starts of further records of the read (own SEQ, same strand)."""
        s = self.seq(start, ops, subs, esc)
        nm = min(len(subs) + sum(n for op, n in ops if op in "ID"), 10)
        flag = 16 if (reverse or mirror) else 0
        recs = [(start, _ops_str(ops), s, nm, flag)]
        if mirror:
            q = R3 + (R1 + W) - (start + _span(ops))
            recs.append((q, _ops_str(ops[::-1]), "*", nm, 256))
        recs += [(o, _ops_str(ops), s, 10, flag | 256) for o in others]
        self.groups.append((kind, recs))


def _genome(rng):
    truth = list(rand_seq(rng, N_TILES * TILE))
    truth[R3:R3 + W] = list(rc("".join(truth[R1:R1 + W])))
    draft = list(truth)
    for p in range(30, len(draft) - 30, 61):
        q = p + rng.randint(0, 30)
        draft[q] = _mutate(rng, draft[q])
    return truth, draft


def _one_indel(rng, length, op, n):
    a = rng.randint(1, length - 20)
    m = length - (n if op == "I" else 0)
    a = min(a, m - 9)
    return [("M", a), (op, n), ("M", m - a)]


def twobit(seed):
    rng = random.Random(seed)
    truth, draft = _genome(rng)
    B = _Reads(rng, truth)
    k = 0
    # tile 1: a substitution at every read index, every start residue mod 16, half of the reads mirrored onto tile 3
    for i in range(STAGED_LEN):
        for length in (150, STAGED_LEN):
            if i >= length:
                continue
            r = (i + length) % 16
            start = R1 + r + 16 * rng.randint(0, (W - length - 16) // 16)
            B.add("sub", start, [("M", length)], subs=(i,), mirror=k % 2 == 0)
            k += 1
    for n in range(1, 21):
        for op in "ID":
            length = rng.randint(100, STAGED_LEN)
            ops = _one_indel(rng, length, op, n)
            B.add("indel1", R1 + rng.randint(0, W - _span(ops) - 1), ops, subs=(rng.randrange(length),), mirror=k % 2 == 0)
            k += 1
    for _ in range(120):
        ops = _indels(rng, rng.randint(2, 6), rng.randint(80, STAGED_LEN))
        B.add("staged", R1 + rng.randint(0, W - _span(ops) - 1), ops, mirror=k % 2 == 0)
        k += 1
    # tile 4: draft bytes that are not A/C/G/T under every kind of walk
    P = 4 * TILE + 300
    specials = [P + 23 * j + rng.randint(0, 9) for j in range(40)]
    for j, p in enumerate(specials):
        draft[p] = (IUPAC + "-acgtn")[j % (len(IUPAC) + 6)]
    for _ in range(60):
        for kind in ("plain4", "indel14", "staged4"):
            length = rng.randint(120, STAGED_LEN)
            if kind == "plain4":
                ops = [("M", length)]
            elif kind == "indel14":
                ops = _one_indel(rng, length, rng.choice("ID"), rng.randint(1, 12))
            else:
                ops = _indels(rng, rng.randint(2, 5), length)
            B.add(kind, P - 100 + rng.randint(0, 1000 - _span(ops)), ops, reverse=rng.random() < 0.5)
    # tile 5: escape reads of every kind, several per chunk, k = 2 and 3; 192-base plain reads
    P = 5 * TILE
    for j in range(240):
        kind = ("esc_plain", "esc_indel1", "esc_staged")[j % 3]
        length = STAGED_LEN if j % 4 == 0 else rng.randint(60, STAGED_LEN)
        if kind == "esc_plain":
            ops = [("M", length)]
        elif kind == "esc_indel1":
            ops = _one_indel(rng, length, rng.choice("ID"), rng.randint(1, 20))
        else:
            ops = _indels(rng, rng.randint(2, 6), length)
        esc = (rng.choice([0, length - 1, rng.randrange(length)]), rng.choice(IUPAC))
        others = () if j % 3 == 0 else tuple(6 * TILE + rng.randint(0, TILE - BIN - 200) for _ in range(1 + j % 2))
        B.add(kind, P + rng.randint(0, TILE - BIN - 200), ops, subs=(rng.randrange(length),), esc=esc, reverse=j % 2 == 1,
              others=others)
    for _ in range(200):
        B.add("len192", P + rng.randint(0, TILE - BIN - 200), [("M", STAGED_LEN)], subs=(rng.randrange(STAGED_LEN),),
              reverse=rng.random() < 0.5)
    # background
    for _ in range(N_TILES * TILE * 6 // 120):
        length = rng.randint(60, 180)
        B.add("plain", rng.randint(0, N_TILES * TILE - length - 1), [("M", length)], reverse=rng.random() < 0.5)
    return _emit(B, rng, "".join(draft), specials)


def _emit(B, rng, draft, specials):
    order = list(range(len(B.groups)))
    rng.shuffle(order)                                    # SAM order within a bin is the slot order: not position order
    lines, kinds = [], []
    for gi, g in enumerate(order):
        kind, recs = B.groups[g]
        for start, cig, seq, nm, flag in recs:
            lines.append(sam("r%d" % gi, flag, "twobit", start, cig, seq, nm))
            kinds.append(kind)
    case = Case(fasta([("twobit", draft)]), ["\n".join(lines) + "\n"], {})
    case.facts = dict(kinds=kinds, n_tiles=N_TILES, specials=specials,
                      n_esc=sum(len(recs) for kind, recs in B.groups if kind.startswith("esc")))
    return case
