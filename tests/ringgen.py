"""FASTA + SAM cases that drive every shape of k_tile's chunk ring (seeded, deterministic, in the style of tests/limitgen.py).

A tile reads the slots [lo, hi) of the binned dataset: the alignments that start in its 8 bins and in the `lb` bins before it
(lb = 1 here: no binned alignment has more than 256 entries).  Warp w takes the 32-slot chunks at lo + 32 w + 512 j, and lane 0 of the
warp copies chunk j into stage j % 2 of the warp's two-stage ring one chunk ahead (polypolish_b200/csrc/polish_dev.cuh tile_body).
The cases set the number of slots of every tile, hi - lo, from a schedule that reaches each edge of that loop: empty tiles, a partial
chunk for warp 0 only, counts that are 0, 1 and 31 mod 32, warps with 1 to 4 chunks, and neighbours in the heaviest-first tile order
whose warps end on odd and even chunk counts, which is how the parity of a warp's stages carries from one tile to the next.

Every read has its own substitutions, so that a read walked from the wrong stage, or a stage read one round stale, changes some
position's counts in the --debug TSV.  The mix: 192-base reads (some in lane 31 of a full chunk, whose trim may load word 24 of the
stage's bases, which is rec[0]), reads of 8-15 bases and shorter than 8 (queued), homopolymer tails of 7 and 8 bases (the second is
queued), one-indel reads aM bI cM / aM bD cM (queued, walked from stage 0), reads that start in the bin before a tile and reads that
cross a tile's end, reads that map to 2 or 3 places (k > 1, carried in the queue entry), and ZP:Z:fail records (k = 0).

Each builder returns a fuzzgen.Case with a `facts` dict: the schedule, the kind of every alignment (SAM order = alignment index) and
what the case was built to reach, for the tests to check against the emulator's layout readouts before they trust a pass.
"""
import random

from tests.fuzzgen import Case
from tests.limitgen import fasta, rand_seq, sam

BIN = 256                  # PP_BIN
TILE = 2048                # TL_T
WARPS = 16                 # TL_THREADS / 32
STRIDE = 32 * WARPS        # slots between a warp's chunks
QCAP = 1024                # TL_QCAP: queued reads per tile
LONG_E = 512               # TL_LONG_E

# slots per tile (hi - lo), in contig order
SCHEDULE = [0, 1, 17, 31, 32, 33, 63, 64, 95, 96, 200, 511, 512, 513, 543, 544, 575, 700, 1023, 1024, 1025, 1055, 1056, 1087,
            1535, 1536, 1537, 1567, 0, 5, 31, 300, 1057, 545, 40, 2080, 97, 1600, 62, 0]

# offsets inside a tile (see _genome): homopolymer runs, repeat copies (reads inside a copy map to every copy of the tile)
RUN7, RUN8 = 480, 960
REP_AT, REP_LEN = (1100, 1350, 1600), 150
INNER_END = TILE - BIN     # inner reads start before the tile's last bin (and end inside the tile)


def warp_chunks(n):
    """Chunks of each warp for a tile of n slots."""
    return [max(0, -(-(n - 32 * w) // STRIDE)) for w in range(WARPS)]


def _mutate(rng, b):
    return rng.choice([x for x in "ACGT" if x != b])


def _genome(rng, n_tiles):
    truth = list(rand_seq(rng, n_tiles * TILE))
    for t in range(n_tiles):
        base = t * TILE
        for off, n, ch in ((RUN7, 7, "A"), (RUN8, 8, "C")):       # runs of exactly 7 A and 8 C
            truth[base + off - 1] = "G"
            truth[base + off:base + off + n] = ch * n
            truth[base + off + n] = "T"
        unit = truth[base + REP_AT[0]:base + REP_AT[0] + REP_LEN]
        for a in REP_AT[1:]:
            truth[base + a:base + a + REP_LEN] = unit
    truth = "".join(truth)
    draft = list(truth)                                           # draft errors away from the runs and the repeats
    protected = set()
    for t in range(n_tiles):
        base = t * TILE
        for off in (RUN7, RUN8):
            protected.update(range(base + off - 2, base + off + 10))
        for a in REP_AT:
            protected.update(range(base + a, base + a + REP_LEN))
    for p in range(20, len(draft) - 20, 173):
        q = p + rng.randint(0, 60)
        if q not in protected:
            draft[q] = _mutate(rng, draft[q])
    return truth, "".join(draft)


class _Builder:
    def __init__(self, rng, truth):
        self.rng, self.truth = rng, truth
        self.groups = []                  # [(kind, [(start, cigar, read)], extra tags)]

    def read(self, start, length, n_sub=None):
        """The truth at [start, start + length) with its own substitutions (none in the last 10 bases: the tails stay exact)."""
        rng = self.rng
        s = list(self.truth[start:start + length])
        if n_sub is None:
            n_sub = rng.randint(1, 2) if length >= 16 else (1 if length >= 10 else 0)
        for _ in range(n_sub):
            i = rng.randint(1, length - 11) if length >= 16 else rng.randint(0, max(0, length - 2))
            s[i] = _mutate(rng, s[i])
        return "".join(s), n_sub

    def single(self, kind, start, length, zp=False):
        seq, nm = self.read(start, length)
        self.groups.append((kind, [(start, "%dM" % length, seq, nm)], ["ZP:Z:fail"] if zp else []))

    def indel(self, start, a, b, c, is_del):
        t = self.truth
        if is_del:
            seq = t[start:start + a] + t[start + a + b:start + a + b + c]
        else:
            seq = t[start:start + a] + rand_seq(self.rng, b) + t[start + a:start + a + c]
        s = list(seq)
        i = self.rng.randint(1, max(1, a - 1)) if a > 2 else a + b + 1        # one substitution besides the indel
        s[i] = _mutate(self.rng, s[i])
        self.groups.append(("indel" if a + c + (b if is_del else 0) <= LONG_E else "long_indel",
                            [(start, "%dM%d%s%dM" % (a, b, "D" if is_del else "I", c), "".join(s), b + 1)], []))

    def multi(self, tile_base, r, length):
        """A read inside the tile's repeat unit, aligned to 2 or 3 of its copies; one in three is a one-indel read (queued with k)."""
        rng = self.rng
        k = rng.choice((2, 3))
        if rng.random() < 1 / 3:
            a = rng.randint(1, length - 20)
            ins = rand_seq(rng, rng.randint(1, 3))
            s0 = tile_base + REP_AT[0] + r
            seq = self.truth[s0:s0 + a] + ins + self.truth[s0 + a:s0 + length]
            cig, nm, kind = "%dM%dI%dM" % (a, len(ins), length - a), len(ins), "multi%d_indel" % k
        else:
            seq, nm = self.read(tile_base + REP_AT[0] + r, length)
            cig, kind = "%dM" % length, "multi%d" % k
        self.groups.append((kind, [(tile_base + a + r, cig, seq, nm) for a in REP_AT[:k]], []))


def _fill_inner(B, t, n):
    """n alignments that start in tile t's first 7 bins and end inside the tile: a mix of every kind."""
    rng = B.rng
    base = t * TILE
    while n > 0:
        x = rng.random()
        if n >= 3 and x < 0.06:
            length = rng.randint(30, 120)
            before = len(B.groups)
            B.multi(base, rng.randint(0, REP_LEN - length), length)
            n -= len(B.groups[before][1])
            continue
        n -= 1
        if x < 0.12:
            a, b, c = rng.randint(1, 60), rng.randint(1, 3), rng.randint(9, 80)
            B.indel(base + rng.randint(0, INNER_END - 200), a, b, c, rng.random() < 0.5)
        elif x < 0.16:
            B.single("short", base + rng.randint(0, INNER_END - 1), rng.randint(1, 7))
        elif x < 0.21:
            B.single("len8_15", base + rng.randint(0, INNER_END - 1), rng.randint(8, 15))
        elif x < 0.25:
            off, n_run = (RUN7, 7) if rng.random() < 0.5 else (RUN8, 8)
            length = rng.randint(20, 120)
            B.single("tail%d" % n_run, base + off + n_run - length, length)
        elif x < 0.30:
            B.single("zp", base + rng.randint(0, INNER_END - 1), rng.randint(40, 150), zp=True)
        elif x < 0.36:
            B.single("len192", base + rng.randint(0, INNER_END - 1), 192)
        else:
            B.single("plain", base + rng.randint(0, INNER_END - 1), rng.randint(40, 150))
    assert n == 0


def _fill_cross(B, t, n):
    """n alignments that start in tile t's last bin and cross its end (for tile t + 1 they start in the bin before it)."""
    rng = B.rng
    end = (t + 1) * TILE
    for i in range(n):
        length = 192 if i % 3 == 2 else rng.randint(40, 150)
        B.single("cross", end - rng.randint(10, min(BIN, length - 10)), length, zp=(i % 5 == 4))


def _lay_out(B, schedule, n_tiles):
    x = [0] * (len(schedule) + 1)                         # x[t]: alignments in the bin before tile t (tile t - 1's last bin)
    for t in range(1, len(schedule)):
        x[t] = min(3, schedule[t - 1] // 4, schedule[t] // 4)
    pieces = []
    for t, n in enumerate(schedule):
        inner = n - x[t] - x[t + 1]
        assert inner >= 0
        pieces.append((t, inner, x[t + 1]))
    for t, inner, cross in pieces:
        _fill_inner(B, t, inner)
        _fill_cross(B, t, cross)


def _slots(starts):
    """Slot order of the binned dataset (one contig at offset 0): by bin, then by alignment index."""
    return sorted(range(len(starts)), key=lambda i: (starts[i] // BIN, i))


def _tile_ranges(starts, n_tiles, lb=1):
    bins = [0] * (n_tiles * (TILE // BIN) + 1)
    for s in starts:
        bins[s // BIN + 1] += 1
    for i in range(1, len(bins)):
        bins[i] += bins[i - 1]
    return [(bins[max(0, 8 * t - lb)], bins[8 * t + 8]) for t in range(n_tiles)]


def _emit(B, rng, n_tiles, eight_bit, opts, facts):
    order = list(range(len(B.groups)))
    rng.shuffle(order)                                     # SAM order within a bin is the slot order: not position order
    lines, kinds, starts, lens = [], [], [], []
    for gi, g in enumerate(order):
        kind, recs, tags = B.groups[g]
        for j, (start, cig, seq, nm) in enumerate(recs):
            flag = (16 if (gi + j) % 2 else 0) | (256 if j else 0)
            lines.append(sam("r%d" % gi, flag, "ring", start, cig, seq, nm, tags))
            kinds.append(kind)
            starts.append(start)
            lens.append(len(seq))
    # the 192-base reads in lane 31 of a full chunk: turn a plain read there into one (it stays inside its tile)
    slots = _slots([s if k != "long_indel" else 1 << 40 for s, k in zip(starts, kinds)])
    lane31 = 0
    for t, (lo, hi) in enumerate(_tile_ranges([s for s, k in zip(starts, kinds) if k != "long_indel"], n_tiles)):
        for o in range(31, hi - lo, 32 * 7):
            a = slots[lo + o]
            if kinds[a] == "plain" and starts[a] % TILE < INNER_END:
                f = lines[a].split("\t")
                seq, nm = B.read(starts[a], 192)
                f[5], f[9], f[11] = "192M", seq, "NM:i:%d" % nm
                lines[a] = "\t".join(f)
                kinds[a] = "len192"
                lens[a] = 192
                lane31 += 1
    if eight_bit:                                          # a byte outside "=ACMGRSVTWYHKDBN": the batch goes to the 8-bit pool
        a = kinds.index("plain")
        f = lines[a].split("\t")
        f[9] = f[9][:5] + "." + f[9][6:]
        lines[a] = "\t".join(f)
    facts.update(kinds=kinds, starts=starts, lens=lens, seq_bits=8 if eight_bit else 4, lane31_192=lane31, n_tiles=n_tiles)
    case = Case(fasta([("ring", B.draft)]), ["\n".join(lines) + "\n"], opts)
    case.facts = facts
    return case


def chunk_shapes(seed, eight_bit=False, repeat=1):
    """A (4-bit) / B (eight_bit: the ring copies records only): one contig of len(SCHEDULE) * repeat tiles whose slot counts follow
    SCHEDULE.  repeat > 1 (D, for the GPU): the schedule again and again, so that a CTA that takes several tiles carries its parity."""
    rng = random.Random(seed)
    schedule = SCHEDULE * repeat
    n_tiles = len(schedule)
    truth, draft = _genome(rng, n_tiles)
    B = _Builder(rng, truth)
    B.draft = draft
    _lay_out(B, schedule, n_tiles)
    facts = dict(schedule=schedule)
    return _emit(B, rng, n_tiles, eight_bit, {}, facts)


def queue_overflow(seed, n_indel=1150):
    """C: three tiles; the middle one has n_indel one-indel reads (more than TL_QCAP: the rest are walked in place, from the live
    stage) among plain reads, and one-indel alignments of more than 512 entries (the long list, which takes the general walk)
    cross both tile borders."""
    rng = random.Random(seed)
    truth, draft = _genome(rng, 3)
    B = _Builder(rng, truth)
    B.draft = draft
    _fill_inner(B, 0, 150)
    _fill_cross(B, 0, 3)
    for _ in range(n_indel):
        a, b, c = rng.randint(1, 60), rng.randint(1, 3), rng.randint(9, 110)
        B.indel(TILE + rng.randint(0, INNER_END - 200), a, b, c, rng.random() < 0.5)
    _fill_inner(B, 1, 200)
    _fill_cross(B, 1, 3)
    _fill_inner(B, 2, 120)
    for start, a, b, c, d in ((TILE - 300, 300, 3, 300, False), (TILE - 250, 260, 2, 280, True), (2 * TILE - 320, 300, 4, 290, True),
                              (2 * TILE - 200, 240, 1, 300, False)):
        B.indel(start, a, b, c, d)
    facts = dict(n_indel=n_indel)
    return _emit(B, rng, 3, False, {}, facts)
