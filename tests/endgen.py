"""FASTA + SAM cases at contig ends (seeded, deterministic, in the style of tests/stagedgen.py).

The reference indexes the pileup only for the entries the homopolymer trim keeps (pileup.rs:189-200, alignment.rs:364-378): an
alignment overruns its contig only if a KEPT entry lies past the end, and it checks the CIGAR ops and the CIGAR / SEQ length before
it indexes anything.  A read whose tail has r equal bases (the base before them differs) keeps E - r - 1 of its E entries, so one
placed at start = end - E + over has `over` untrimmed entries past the end: legal for over <= r + 1 (the last kept entry is then at
most the contig's last base), an overrun for over = r + 2.

E (edges, legal): an assembly of many contigs whose starts fall at every residue mod 32, on and next to bin borders (256 b - 1,
256 b, 256 b + 1) and tile borders (2048 t - 1, 2048 t, 2048 t + 1), contigs of 1, 2, 7, 8 and 9 bp (several starts inside one
8-position k_compact item and one 128-position warp vote), and contigs no read covers.  At contig ends, a bundle of reads of one walk
kind with tails r and every over in 1 .. r + 1 (and at r + 1 twice, so the last base has depth for the vote):
  * plain: the fast walk, r <= 7;   fast1I / fast1D: aM bI cM / aM bD cM, segment B ending on the last base;
  * gen: two or three indels;  xeq: X and = ops;  short: reads of 3 - 7 bases;  tail8: tails of 8 - 12 bases (the general walk);
  * queued: 193 - 200 bases;  long: more than 512 entries (the long list), on the first contig (700 bp);
  * insend / delend: the last base carries an insertion / is deleted (segment B trimmed whole past the end);
  * first, firstins, firstdel: reads that start on a contig's first base, which is a mismatch / followed by an insertion /
    followed by a deletion.
The draft differs from the truth at the last base of every bundle's contig and at the first base of the `first` ones, so the vote
changes them.  With eight_bit, one read carries a byte outside the 4-bit alphabet: the whole batch goes to the 8-bit pool (queued).

P (starts at or past the end, legal): records whose entries all trim away - 1M, CAAAAA-like (xM yA) and pure homopolymers - at
POS = length + 1 and far past the end, on a middle contig and on the last one, as primaries with SEQ and as SEQ="*" secondaries (same
strand and opposite strand as the SEQ record).  Each is the second good alignment of a read whose other alignment (xM 1D yM: the trim
stops at the "-") covers a probe position whose vote flips between k = 1 and k = 2; a 1-base read cannot have such a partner.

Errors (`errors`): every walk kind of E with one read at over = r + 2; an overrun before and after an unknown RNAME, a CIGAR / SEQ
mismatch and a bad op, in other tiles; a start past the end with a bad op (N, S, H, P between M runs) or with a CIGAR / SEQ mismatch.

Every case is a fuzzgen.Case with `facts`: per alignment (SAM order) its kind, contig, start and kept entries (the trim modelled
here), and what the case was built to reach.
"""
import random

from tests.fuzzgen import Case, revcomp
from tests.indelgen import BIN, TILE, _mutate
from tests.limitgen import fasta, rand_seq, sam

FAST_LEN = 192             # TL_FAST_LEN
LONG_E = 512               # TL_LONG_E
KINDS = ["plain", "fast1I", "fast1D", "gen", "xeq", "short", "tail8", "queued", "long"]


def parse_cigar(cig):
    out, n = [], ""
    for ch in cig:
        if ch.isdigit():
            n += ch
        else:
            out.append((ch, int(n)))
            n = ""
    return out


def kept_entries(ops, seq):
    """The reference's entries (alignment.rs:175-201) after its trim (:364-378): how many survive."""
    ent, i = [], 0
    for op, n in ops:
        for _ in range(n):
            if op in "M=X":
                ent.append((i, i + 1))
                i += 1
            elif op == "I":
                ent[-1] = (ent[-1][0], i + 1)
                i += 1
            else:
                ent.append((i, i))
    last = seq[ent[-1][0]:ent[-1][1]]
    while ent and seq[ent[-1][0]:ent[-1][1]] == last:
        ent.pop()
    if ent:
        ent.pop()
    return len(ent)


def span(ops):
    return sum(n for op, n in ops if op in "M=XD")


class _Asm:
    """Contig layout: starts at every residue mod 32, at bin and tile borders, a cluster of tiny contigs."""

    def __init__(self, rng, n_tiles=5, tail_len=400):
        targets = set()
        for t in range(1, n_tiles):
            targets |= {TILE * t - 1, TILE * t, TILE * t + 1}
        for b in (3, 11):                                  # bin borders that are not tile borders
            targets |= {BIN * b - 1, BIN * b, BIN * b + 1}
        lens = [700, 1, 2, 7, 8, 9]                        # starts 700, 701, 703, 710, 718: one 8-position item, one 128-position warp
        pos = sum(lens)
        seen = {p % 32 for p in self.starts_of(lens)}
        end = TILE * n_tiles - tail_len - 1000
        while pos < end:
            nxt = min([t for t in targets if t > pos] or [end])
            if nxt - pos <= 260:
                L = nxt - pos
            else:
                want = [L for L in range(210, 261) if (pos + L) % 32 not in seen] or [233]
                L = rng.choice(want)
            lens.append(L)
            pos += L
            seen.add(pos % 32)
        lens.append(1000)                                  # the probe contig (P)
        lens.append(tail_len)                              # the last contig
        self.lens = lens
        self.starts = self.starts_of(lens)
        self.names = ["ctg%d" % i for i in range(len(lens))]
        self.G = sum(lens)

    @staticmethod
    def starts_of(lens):
        out, p = [], 0
        for L in lens:
            out.append(p)
            p += L
        return out

    def span_of(self, c):
        return self.starts[c], self.starts[c] + self.lens[c]


class _Builder:
    def __init__(self, rng, asm):
        self.rng, self.asm = rng, asm
        self.truth = rand_seq(rng, asm.G)
        self.draft = list(self.truth)
        self.groups = []                                   # [(kind, [(contig, local start, cigar, seq, nm, flag, extra)])]

    def edit(self, g):                                     # the draft differs from the truth at global position g
        self.draft[g] = _mutate(self.rng, self.truth[g])

    def read(self, kind, c, start, ops, r, ins=None):
        """A read of contig c at local `start` from the truth, tail r (the last r bases equal, the one before them not), one
        substitution per match run away from the contig's ends and the tail.  Returns the SAM record tuple."""
        rng, t = self.rng, self.truth
        cs, ce = self.asm.span_of(c)
        g, s, ref = cs + start, [], []
        for op, n in ops:
            if op in "M=X":
                for j in range(n):
                    b = t[g + j] if g + j < len(t) else rng.choice("ACGT")
                    s.append(_mutate(rng, b) if op == "X" else b)
                    ref.append(g + j)
                g += n
            elif op == "I":
                s += list(ins if ins is not None else rand_seq(rng, n))
                ref += [None] * n
            else:
                g += n
        tail = r + 1
        assert ops[-1][0] in "M=" and ops[-1][1] >= tail, (ops, r)
        x = rng.choice("ACGT")
        s[len(s) - r:] = x * r
        s[len(s) - tail] = _mutate(rng, x)
        ok = [i for i in range(len(s) - tail) if ref[i] is not None and cs + 3 <= ref[i] < ce - 3]
        nm = sum(n for op, n in ops if op in "XID")
        if ok and len(s) >= 12:
            i = rng.choice(ok)
            s[i] = _mutate(rng, s[i])
            nm += 1
        return (c, start, "".join("%d%s" % (n, op) for op, n in ops), "".join(s), min(nm, 10))

    def add(self, kind, recs):
        self.groups.append((kind, [rec + (None,) * (7 - len(rec)) if len(rec) < 7 else rec for rec in recs]))


def _ops_for(rng, kind, r, room):
    """CIGAR ops of a read of `kind` with tail r whose reference span fits `room` bases (None: it does not fit)."""
    last = r + 4                                           # the last match run holds the tail and three kept bases
    if kind == "plain":
        L = rng.randint(max(12, last), min(FAST_LEN, room))
        return [("M", L)]
    if kind in ("fast1I", "fast1D"):
        a, b = rng.randint(1, 60), rng.randint(1, 12)
        c = rng.randint(last, last + 40)
        if kind == "fast1I":
            c = min(c, FAST_LEN - a - b)
            return [("M", a), ("I", b), ("M", c)]
        return [("M", a), ("D", b), ("M", min(c, FAST_LEN - a))]
    if kind == "gen":
        runs = [rng.randint(3, 30) for _ in range(rng.randint(2, 3))] + [rng.randint(last, last + 30)]
        ops = [("M", runs[0])]
        for n in runs[1:]:
            ops += [(rng.choice("ID"), rng.randint(1, 3)), ("M", n)]
        return ops
    if kind == "xeq":
        return [("M", rng.randint(3, 30)), ("X", rng.randint(1, 2)), ("=", rng.randint(3, 30)), (rng.choice("ID"), rng.randint(1, 3)),
                (rng.choice("M="), rng.randint(last, last + 30))]
    if kind == "short":
        return [("M", rng.randint(max(r + 2, 3), 7))]
    if kind == "tail8":
        return [("M", rng.randint(max(40, last), min(FAST_LEN, room)))]
    if kind == "queued":
        L = rng.randint(FAST_LEN + 1, 200)
        if rng.random() < 0.5:
            return [("M", L)]
        a = rng.randint(20, 150)
        return [("M", a), ("D", rng.randint(1, 3)), ("M", L - a)]
    if kind == "long":
        return [("M", rng.randint(LONG_E + 8, 600))]
    raise ValueError(kind)


TAILS = {"plain": [1, 2, 3, 4, 5, 6, 7], "fast1I": [1, 3, 5, 7], "fast1D": [1, 2, 4, 6], "gen": [1, 2, 3, 5], "xeq": [1, 3, 4],
         "short": [1, 2, 3], "tail8": [8, 9, 10, 12], "queued": [1, 3, 8], "long": [1, 2, 9]}


def _end_read(B, kind, c, r, over):
    """A read of `kind` with tail r on contig c with `over` untrimmed entries past the end (start = end - E + over)."""
    rng = B.rng
    L = B.asm.lens[c]
    for _ in range(200):
        ops = _ops_for(rng, kind, r, L + over)
        E = span(ops)
        start = L - E + over
        if start >= 0:
            rec = B.read(kind, c, start, ops, r)
            assert kept_entries(ops, rec[3]) == E - r - 1
            return rec
    raise AssertionError((kind, c, r, over))


def _bundle(B, kind, c, twice=True):
    """Reads of `kind` at the end of contig c: every tail of TAILS[kind], every over in 1 .. r + 1 (r + 1 twice)."""
    for r in TAILS[kind]:
        for over in range(1, r + 2):
            for _ in range(2 if (twice and over == r + 1) else 1):
                B.add(kind, [_end_read(B, kind, c, r, over)])
    cs, ce = B.asm.span_of(c)
    B.edit(ce - 1)


def _first(B, kind, c, n=6):
    """n reads that start on contig c's first base: a mismatch there (first), an insertion after it (firstins: 1M bI cM, one allele)
    or a deletion after it (firstdel: 1M bD cM)."""
    rng = B.rng
    cs, ce = B.asm.span_of(c)
    ins, b = rand_seq(rng, rng.randint(1, 4)), rng.randint(1, 3)
    for _ in range(n):
        r = rng.randint(1, 5)
        room = min(B.asm.lens[c] - 4, 150)
        if kind == "first":
            ops = [("M", rng.randint(20, room))]
        elif kind == "firstins":
            ops = [("M", 1), ("I", len(ins)), ("M", rng.randint(20, room))]
        else:
            ops = [("M", 1), ("D", b), ("M", rng.randint(20, room - b))]
        B.add(kind, [B.read(kind, c, 0, ops, r, ins=ins if kind == "firstins" else None)])
    if kind == "first":
        B.edit(cs)


def _insdel_end(B, kind, c, n=6):
    """n reads whose kept entries end on contig c's last base, which carries an insertion (insend: aM bI cM with c = r + 1 bases past
    the end, all trimmed) or is deleted with the b - 1 bases before it (delend: aM bD cM, the D ends on the last base)."""
    rng = B.rng
    L = B.asm.lens[c]
    ins, b = rand_seq(rng, rng.randint(1, 5)), rng.randint(1, 3)
    for _ in range(n):
        r = rng.randint(1, 6)
        a = rng.randint(20, min(120, L - b - 1))
        if kind == "insend":
            ops = [("M", a), ("I", len(ins)), ("M", r + 1)]
            start = L - a
        else:
            ops = [("M", a), ("D", b), ("M", r + 1)]
            start = L - a - b
        rec = B.read(kind, c, start, ops, r, ins=ins if kind == "insend" else None)
        assert start + kept_entries(ops, rec[3]) == L
        B.add(kind, [rec])


def _kept_of(line):
    """Kept entries of a SAM record with its own SEQ and a CIGAR of M = X I D (None otherwise)."""
    f = line.split("\t")
    ops = parse_cigar(f[5])
    if f[9] == "*" or any(op not in "M=XID" for op, _ in ops) or sum(n for op, n in ops if op in "M=XI") != len(f[9]):
        return None
    return kept_entries(ops, f[9].upper())


def _emit(B, name_facts, eight_bit=False, extra_lines=()):
    """SAM text: groups in a shuffled order, then `extra_lines` = [(index in the output, kind, record line, contig)] put in place."""
    rng, asm = B.rng, B.asm
    order = list(range(len(B.groups)))
    rng.shuffle(order)
    rows = []                                               # (kind, contig, start, line, ops, seq)
    for gi, g in enumerate(order):
        kind, recs = B.groups[g]
        for j, (c, start, cig, seq, nm, flag, qname) in enumerate(recs):
            if flag is None:
                flag = (16 if (gi + j) % 2 else 0) | (256 if j else 0)
            rows.append((kind[j] if isinstance(kind, list) else kind, c, start, sam(qname or "r%d" % gi, flag, asm.names[c], start, cig, seq, nm)))
    for at, kind, line, c in sorted(extra_lines, key=lambda x: x[0]):
        rows.insert(at, (kind, c, int(line.split("\t")[3]) - 1, line))
    if eight_bit:                                          # a byte outside "=ACMGRSVTWYHKDBN": the batch goes to the 8-bit pool
        a = next(i for i, x in enumerate(rows) if x[0] == "marker")
        f = rows[a][3].split("\t")
        f[9] = f[9][:5] + "." + f[9][6:]
        rows[a] = rows[a][:3] + ("\t".join(f),)
    facts = dict(name_facts)
    facts.update(kinds=[x[0] for x in rows], contigs=[x[1] for x in rows], starts=[x[2] for x in rows], lens=asm.lens,
                 cstarts=asm.starts, n_tiles=-(-asm.G // TILE), seq_bits=8 if eight_bit else 4,
                 lines=[x[3] for x in rows], kept=[_kept_of(x[3]) for x in rows])
    draft = "".join(B.draft)
    case = Case(fasta([(asm.names[c], draft[asm.starts[c]:asm.starts[c] + asm.lens[c]]) for c in range(len(asm.lens))]),
                ["\n".join(x[3] for x in rows) + "\n"], {})
    case.facts = facts
    return case


def _sites(B):
    """Contigs of the E bundles (one kind each), the first-base contigs and the uncovered ones."""
    asm = B.asm
    mids = [c for c in range(6, len(asm.lens) - 2) if asm.lens[c] >= 210]
    # contigs that end on or next to a tile border first
    near = [c for c in mids if any(abs(asm.starts[c] + asm.lens[c] - TILE * t) <= 1 for t in range(1, 8))]
    mids = near + [c for c in mids if c not in near]
    plan = {}
    kinds = ["plain", "fast1I", "fast1D", "gen", "xeq", "tail8", "queued", "short", "insend", "delend", "first", "firstins", "firstdel",
             "plain", "gen", "queued", "fast1D", "tail8"]
    for c, k in zip(mids, kinds):
        plan[c] = k
    uncovered = [c for c in mids if c not in plan]
    return plan, uncovered


def edges(seed, eight_bit=False):
    """E; see the module's docstring."""
    rng = random.Random(seed)
    asm = _Asm(rng)
    B = _Builder(rng, asm)
    plan, uncovered = _sites(B)
    for c, k in plan.items():
        if k in ("insend", "delend"):
            _insdel_end(B, k, c)
        elif k.startswith("first"):
            _first(B, k, c)
        else:
            _bundle(B, k, c)
    _bundle(B, "long", 0)
    _first(B, "first", 0)
    # the tiny contigs: short reads ending on the last base of the 7, 8 and 9 bp ones; 1 and 2 bp: a 3-base read keeps one entry
    for c in (3, 4, 5):
        for r in (1, 2):
            for over in range(1, r + 2):
                B.add("short", [_end_read(B, "short", c, r, over)])
    for c in (1, 2):
        s = B.read("tiny", c, asm.lens[c] - 1, [("M", 3)], 1)
        B.add("tiny", [s])
    # a plain read far from every end (the 8-bit marker)
    B.add("marker", [B.read("marker", 0, 200, [("M", 100)], 1)])
    facts = dict(plan=plan, uncovered=uncovered)
    return _emit(B, facts, eight_bit=eight_bit)


# ---- P: starts at or past the end -------------------------------------------------------------------------------------------------
P_SEQS = {"1M": "G", "xMyA": "CAAAAA", "homo": "TTTTT"}


def _probe_partner(eff):
    """The partner alignment of a P record, whose effective read is `eff`: ops 1M 1D yM and the probe's base (its first entry, always
    kept: the trim stops at the "-")."""
    ops = [("M", 1), ("D", 1), ("M", len(eff) - 1)]
    assert kept_entries(ops, eff) >= 1
    return ops, eff[0]


def past_end(seed):
    """P; see the module's docstring."""
    rng = random.Random(seed)
    asm = _Asm(rng)
    B = _Builder(rng, asm)
    plan, _ = _sites(B)
    for c, k in list(plan.items())[:4]:                    # a few legal bundles around them
        _bundle(B, k, c)
    c_probe, c_last = len(asm.lens) - 2, len(asm.lens) - 1
    c_mid = sorted(plan)[len(plan) // 2]
    probe_cs, _ = asm.span_of(c_probe)
    probes, n_probe = [], 0
    for c in (c_mid, c_last):
        for far in (False, True):
            for pk, eff in P_SEQS.items():
                for star in (False, True):
                    for opposite in (False, True):
                        L = asm.lens[c]
                        pos = L + (rng.randint(1000, 100_000) if far else 0)
                        q = "p%d_%s_%s%s%s" % (c, pk, "far" if far else "end", "_star" if star else "", "_opp" if opposite else "")
                        sP = 16 if rng.random() < 0.5 else 0
                        sQ = sP ^ 16 if opposite else sP
                        p_rec = (c, pos, "%dM" % len(eff), eff, 0)          # (SAM's SEQ is what the trim reads)
                        if pk == "1M":
                            # (a 1-base read keeps nothing anywhere: its partner is another past-the-end record)
                            part = (c_mid, asm.lens[c_mid], "1M", eff if sQ == sP else revcomp(eff), 0)
                            probe = None
                        else:
                            # the partner's read: a SEQ="*" record takes the group's SEQ, reverse complemented if the strands differ
                            q_eff = eff if sQ == sP else revcomp(eff)
                            p0 = 20 + 30 * n_probe
                            n_probe += 1
                            ops, base = _probe_partner(q_eff)
                            g = probe_cs + p0
                            B.draft[g] = _mutate(rng, base)
                            for i in range(4):               # four k = 1 reads carry `base` at the probe
                                s0 = p0 - 8 - i
                                seq = list("".join(B.draft[probe_cs + s0:probe_cs + s0 + 20]))
                                seq[p0 - s0] = base
                                if seq[-1] == seq[-2]:
                                    seq[-2] = _mutate(rng, seq[-1])
                                B.add("support", [(c_probe, s0, "20M", "".join(seq), 1)])
                            cig = "".join("%d%s" % (n, op) for op, n in ops)
                            part = (c_probe, p0, cig, q_eff, 2)
                            probe = (g, base)
                        # which of the two carries SEQ, and which comes first in the group
                        seq_on_p = not star
                        recs = []
                        for kind, rec, strand in (("past", p_rec, sP), ("partner", part, sQ)):
                            has_seq = (kind == "past") == seq_on_p
                            flag = strand | (0 if has_seq else 256)
                            recs.append((kind, rec[:3] + (rec[3] if has_seq else "*", rec[4], flag, q)))
                        if rng.random() < 0.5:
                            recs.reverse()
                        B.groups.append(([x[0] if x[0] != "partner" or probe else "past" for x in recs], [x[1] for x in recs]))
                        probes.append(dict(qname=q, kind=pk, star=star, far=far, contig=c, probe=probe, partner_seq=part[3]))
    return _emit(B, dict(probes=probes, c_probe=c_probe, c_mid=c_mid, c_last=c_last))
    return case


# ---- errors ---------------------------------------------------------------------------------------------------------------------
def _oob_line(B, kind, c, qname, r=None):
    """One read of `kind` on contig c whose first trimmed-in entry past the end is kept: over = r + 2."""
    r = r if r is not None else B.rng.choice(TAILS[kind])
    rec = _end_read(B, kind, c, r, r + 2)
    c, start, cig, seq, nm = rec
    return sam(qname, 0, B.asm.names[c], start, cig, seq, nm)


def error_cases(seed):
    """{name: Case}; facts["expect"] = ("oob", qname) or ("msg", qname of the record whose message wins)."""
    out = {}
    rng = random.Random(seed)
    asm = _Asm(rng)

    def base():
        B = _Builder(random.Random(rng.random()), asm)
        plan, _ = _sites(B)
        for c, k in list(plan.items())[:3]:
            _bundle(B, k, c, twice=False)
        return B, plan

    def tile_of(c):
        return (asm.starts[c] + asm.lens[c] - 1) // TILE

    # every walk kind, one read one entry too far
    for kind in KINDS:
        for eight in ((False, True) if kind == "queued" else (False,)):
            B, plan = base()
            B.add("marker", [B.read("marker", 0, 200, [("M", 100)], 1)])
            c = 0 if kind == "long" else (next(c for c in plan if asm.lens[c] >= 210 and c not in list(plan)[:3]) if kind != "short" else 5)
            line = _oob_line(B, kind, c, "oob")
            n = sum(len(r) for _, r in B.groups)
            case = _emit(B, dict(expect=("oob", "oob")), eight_bit=eight, extra_lines=[(n // 2, "oob", line, c)])
            out["oob_" + kind + ("8" if eight else "")] = case
    # error order: an overrun and another error, each first in SAM order, in different tiles
    mids = [c for c in range(6, len(asm.lens) - 2) if asm.lens[c] >= 210]
    c_lo = next(c for c in mids if tile_of(c) == 0)
    c_hi = next(c for c in reversed(mids) if tile_of(c) >= 2)
    for other in ("unknown", "mismatch", "badop"):
        for oob_first in (True, False):
            B, plan = base()
            c_oob, c_other = (c_lo, c_hi) if oob_first else (c_hi, c_lo)
            oob = _oob_line(B, "plain", c_oob, "oob")
            o_rec = B.read("x", c_other, 30, [("M", 40)], 1)
            name = B.asm.names[c_other]
            cig, seq = o_rec[2], o_rec[3]
            if other == "unknown":
                name = "no_such_contig"
            elif other == "mismatch":
                seq = seq[:-1]
            else:
                cig = "20M2N20M"
            oth = sam("other", 0, name, 30, cig, seq, 1)
            n = sum(len(r) for _, r in B.groups)
            a, b = (oob, oth) if oob_first else (oth, oob)
            extra = [(n // 3, "first", a, c_oob if oob_first else c_other), (n // 3 + 1 + n // 3, "second", b, c_hi if oob_first else c_lo)]
            case = _emit(B, dict(expect=("oob", "oob") if oob_first else ("msg", name if other == "unknown" else "other")), extra_lines=extra)
            out["order_%s_%s" % (other, "oobfirst" if oob_first else "oobsecond")] = case
    # a start past the end with a bad op or a CIGAR / SEQ mismatch: the reference's message, not an overrun
    c_last = len(asm.lens) - 1
    for bad in ("N", "S", "H", "P", "len"):
        B, plan = base()
        L = asm.lens[c_last]
        if bad == "len":
            line = sam("pbad", 0, asm.names[c_last], L + 7, "10M", "ACGTACGTA", 0)
        else:
            cig = "4M2%s4M" % bad
            seq = "ACGTACGT" if bad in "NHP" else "ACGTACGTAC"
            line = sam("pbad", 0, asm.names[c_last], L + 7, cig, seq, 0)
        n = sum(len(r) for _, r in B.groups)
        out["pastbad_" + bad] = _emit(B, dict(expect=("msg", "pbad")), extra_lines=[(n // 2, "pbad", line, c_last)])
    return out
