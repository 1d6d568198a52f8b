"""FASTA + SAM cases whose vote depends on the order the ordered depth walk merges its runs (seeded, deterministic, in the style of
tests/limitgen.py).

Where a position is covered by reads that map to several places (k != 1), the reference's depth is the sequential f64 sum of 1/k in
SAM order, and k_tile redoes that sum by merging the SAM-ordered runs of alignments that can reach the position's 128-position
sub-tile (polypolish_b200/csrc/polish_dev.cuh depth_walk): the bins b-1 and b (depth_walk_two), or b-2, b-1, b and the long list
of alignments with more than 512 entries (depth_walk_steps).  Each case puts a probe position P on a vote boundary: its covering
reads come in a SAM order whose sum is exactly the boundary ("on") or one ulp beside it ("off"), and in the "on" order the reads
are spread over the runs so that a merge which empties one run before the next (in run order or in reverse) gets a sum on the
other side of the boundary.  Decoy reads in the same bins that do not reach P's sub-tile are interleaved with the covering ones.

Each builder returns a fuzzgen.Case with a `facts` dict (what the case was built to reach) that a test asserts before it trusts a
pass: P's bin and sub-tile, the run of every covering read, the largest entry count of a binned alignment (max_ext) and so how many
bins a tile looks back (lb), the long-list count, and the sums of the order and of its run-by-run concatenations.
"""
import math
import random
import re

from tests.fuzzgen import Case
from tests.limitgen import fasta, rand_seq, sam, seq_sum

BIN = 256                  # PP_BIN: positions per bin of the alignment sort
SUB = 128                  # PP_SUB: positions per ordered-depth sub-tile
TILE = 2048                # TL_T
LONG_E = 512               # TL_LONG_E: alignments with more entries go to the long list


def concat_sums(order, n_runs):
    """The sums a merge gets if it empties one run before the next: runs in order and in reverse order."""
    by_run = [[k for k, r in order if r == i] for i in range(n_runs)]
    return [seq_sum([k for run in by_run for k in run]), seq_sum([k for run in reversed(by_run) for k in run])]


NONE32 = 0xFFFFFFFF


def merge_two(runs, mode="ok"):
    """The order in which depth_walk_two merges two runs of slots ((alignment, overlaps the sub-tile, payload) in slot order): windows
    of 32 slots, windows without an overlapping slot skipped, and per round the overlapping entries up to `limit` = the smaller of
    the two "complete up to" keys, merged by alignment index.  mode "max": `limit` the larger key; "batch": the round's entries of run
    0, then those of run 1 (no ranking).  Returns the payloads in merged order."""
    wb, loaded, mask, lastkey, out = [0, 0], [False, False], [[], []], [NONE32, NONE32], []
    while True:
        for r in (0, 1):
            S = runs[r]
            while not mask[r] and (not loaded[r] or wb[r] < len(S)):
                if loaded[r]:
                    wb[r] += 32
                loaded[r] = True
                if wb[r] >= len(S):
                    break
                mask[r] = [e for e in S[wb[r]:wb[r] + 32] if e[1]]
                lastkey[r] = S[wb[r] + 31][0] if wb[r] + 32 < len(S) else NONE32
        if not mask[0] and not mask[1]:
            return out
        lim = [lastkey[r] if (mask[r] or wb[r] < len(runs[r])) else NONE32 for r in (0, 1)]
        limit = max(lim) if mode == "max" else min(lim)
        e = [[x for x in mask[r] if x[0] <= limit] for r in (0, 1)]
        out += [x[2] for x in (e[0] + e[1] if mode == "batch" else sorted(e[0] + e[1]))]
        mask = [[x for x in mask[r] if x[0] > limit] for r in (0, 1)]


def run_orders(seed, ks, target, n_runs, side=-1, min_per_run=1, tries=50_000):
    """Two SAM orders of the multiset ks, every read assigned to one of n_runs runs: `on`, whose sequential f64 sum of 1/k is exactly
    `target` and whose run-by-run concatenations (in run order and in reverse) both sum to the `side` of it (-1 below, +1 above);
    `off`, whose sum is one ulp beside the target on that side.  Lists of (k, run) in SAM order.  (limitgen.boundary_orders with
    runs.)"""
    rng = random.Random(seed)
    off_target = math.nextafter(target, side * math.inf)
    ks = list(ks)
    on = off = None
    for _ in range(tries):
        rng.shuffle(ks)
        runs = [rng.randrange(n_runs) for _ in ks]
        if min(runs.count(r) for r in range(n_runs)) < min_per_run:
            continue
        order = list(zip(ks, runs))
        s = seq_sum(ks)
        if s == target and on is None and (n_runs == 1 or all((c - target) * side > 0 for c in concat_sums(order, n_runs))):
            on = order
        elif s == off_target and off is None:
            off = order
        if on and off:
            return on, off
    raise AssertionError("no such pair of orders for %r over %d runs" % (target, n_runs))


def seq_sum_inv(invs):
    s = 0.0
    for v in invs:
        if v:
            s += v
    return s


def entries(cigar):
    return sum(int(n) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", cigar) if op in "MD=X")


# Layouts: P, contig length, per run (first start, last start, read length) of the covering reads, decoy ranges (first start, last
# start, length) that stay off P's sub-tile, and extra reads (contig position, length, NM, carries the probe base, k).
def layout_two():
    """W1: P in bin 2 (sub-tile [512, 640)); runs bin 1 and bin 2, 60-base reads (lb = 1, depth_walk_two)."""
    return dict(P=522, length=1000, runs=[(468, 511, 60), (512, 517, 60)], labels=["b-1", "b"],
                decoys=[(256, 440, 60), (645, 700, 60)], extra=[])


def layout_three():
    """W2: P in bin 5 (sub-tile [1280, 1408)); 300-base reads from bins 3, 4 and 5 (lb = 2, depth_walk_steps)."""
    return dict(P=1300, length=2000, runs=[(1006, 1023, 300), (1024, 1279, 300), (1280, 1295, 300)], labels=["b-2", "b-1", "b"],
                decoys=[(768, 900, 300), (1024, 1200, 60), (1410, 1500, 60)], extra=[])


def layout_long():
    """W3: P in bin 5; 60-base reads from bins 4 and 5 (lb = 1) and 600-base reads of the long list, all over P.  Plus a long read
    over P with NM above max_errors (left out), and long reads on tile 1."""
    return dict(P=1300, length=6000, runs=[(1246, 1279, 60), (1280, 1295, 60), (706, 1295, 600)], labels=["b-1", "b", "long"],
                decoys=[(1024, 1200, 60), (1410, 1500, 60)],
                extra=[(1000, 600, 20, True, 1), (900, 700, 20, True, 3)] + [(2100 + 300 * i, 600, 0, False, 1 + i % 3) for i in range(8)])


def layout_border_at():
    """W4: P = 2048, the first position of tile 1 (sub-tile 0); 300-base reads from bins 6 and 7 of tile 0 (lb = 2: the lookback
    into the previous tile's bins)."""
    return dict(P=2048, length=3000, runs=[(1754, 1791, 300), (1792, 2043, 300)], labels=["b-2", "b-1"],
                decoys=[(1536, 1700, 300), (2180, 2250, 60)], extra=[])


def layout_border_before():
    """W4: P = 2047, the last position of tile 0; 300-base reads from bins 6 and 7 that run on into tile 1."""
    return dict(P=2047, length=3000, runs=[(1753, 1791, 300), (1792, 2042, 300)], labels=["b-1", "b"],
                decoys=[(1536, 1600, 300), (1280, 1500, 60)], extra=[])


def layout_contig_border():
    """W5: contig `head` (1000 bases) ends inside bin 3, where `probe` starts; P is the probe's position 10 (global 1010).  Reads of
    `head` that end in the same bin (and sub-tile) are interleaved with the covering reads."""
    return dict(P=10, length=1000, head=1000, runs=[(0, 5, 60)], labels=["b"], decoys=[], extra=[], head_reads=(900, 940, 60))


LAYOUTS = dict(two=layout_two, three=layout_three, long=layout_long, border_at=layout_border_at, border_before=layout_border_before,
               contig_border=layout_contig_border)


def walk_case(seed, order, layout, x_reads=0, opts=None, decoy_rate=0.6, eight_bit=False):
    """Contig `probe` with position P covered by the reads of `order` ((k, run) in SAM order): read i has k good alignments, the
    others SEQ="*" secondaries on contig `filler`; every read over P carries base Y != draft there, the first x_reads base X.
    Positions, runs and decoys are those of the probe contig; with layout["head"], contig `head` comes first and the bins are
    counted from its start.  eight_bit: one read on `filler` has a SEQ byte outside the 4-bit alphabet (the 8-bit pool, k_tile<8>)."""
    rng = random.Random(seed)
    lay = layout
    H = lay.get("head", 0)
    head = rand_seq(rng, H) if H else ""
    P = lay["P"]
    probe = rand_seq(rng, lay["length"])
    flen = 8_000
    filler = rand_seq(rng, flen)
    others = [b for b in "ACGT" if b != probe[P]]
    y, x = others[0], others[1]
    lines = []
    nsec = [0]

    def secondaries(q, k, L):
        for _ in range(k - 1):
            fpos = 10 + (37 * nsec[0]) % (flen - L - 20)
            nsec[0] += 1
            lines.append(sam(q, 256, "filler", fpos, "%dM" % L, "*", 0))

    def decoy(j):
        lo, hi, L = lay["decoys"][rng.randrange(len(lay["decoys"]))]
        s = rng.randint(lo, hi)
        lines.append(sam("d%d" % j, 16 if j % 2 else 0, "probe", s, "%dM" % L, probe[s:s + L], 0))

    starts = []
    nd = 0
    meta = []                                   # per covering read: (SAM index, 1/k)
    for i, (k, r) in enumerate(order):
        lo, hi, L = lay["runs"][r]
        s = rng.randint(lo, hi)
        assert s + 5 <= P < s + L - 5 and s + L <= len(probe)            # (P away from the read's ends, which may be trimmed)
        starts.append((s, L))
        q = "r%d" % i
        meta.append((len(lines), 1.0 / k))
        lines.append(sam(q, 16 if i % 2 else 0, "probe", s, "%dM" % L, probe[s:P] + (x if i < x_reads else y) + probe[P + 1:s + L], 1))
        secondaries(q, k, L)
        while lay["decoys"] and rng.random() < decoy_rate:
            decoy(nd)
            nd += 1
        if H and rng.random() < 0.7:                                   # a read of `head` ending in P's bin, k = 2
            lo, hi, L = lay["head_reads"]
            s = rng.randint(lo, hi)
            lines.append(sam("h%d" % i, 0, "head", s, "%dM" % L, head[s:s + L], 0))
            secondaries("h%d" % i, 2, L)
    if eight_bit:
        lines.append(sam("q8bit", 0, "filler", 20, "60M", filler[20:50] + "." + filler[51:80], 1))
    for j, (s, L, nm, over, k) in enumerate(lay["extra"]):
        q = "e%d" % j
        seq = probe[s:P] + y + probe[P + 1:s + L] if over else probe[s:s + L]
        assert (s <= P < s + L) == over and s + L <= len(probe)
        lines.append(sam(q, 0, "probe", s, "%dM" % L, seq, nm))
        secondaries(q, k, L)
    # facts (global positions: `head` first)
    P += H
    starts = [(s + H, L) for s, L in starts]
    sub_lo = P // SUB * SUB
    runs = []
    for s, L in starts:
        runs.append("long" if L > LONG_E else "b-%d" % (P // BIN - s // BIN) if s // BIN != P // BIN else "b")
    assert runs == [lay["labels"][r] for _, r in order], runs
    recs = [l.split("\t") for l in lines]
    ext = [entries(c[5]) for c in recs]
    max_ext = max(e for e in ext if e <= LONG_E)
    decoys = [(int(c[3]) - 1 + H, entries(c[5])) for c in recs if c[0].startswith("d")]
    assert all(s // BIN in {P // BIN - i for i in range(3)} and (s + L <= sub_lo or s >= sub_lo + SUB) for s, L in decoys)
    n_runs = len(lay["runs"])
    facts = dict(P=P, bin=P // BIN, sub=(P % TILE) // SUB, tile=P // TILE, runs=runs,
                 run_counts={lab: runs.count(lab) for lab in lay["labels"]}, max_ext=max_ext, lb=(max_ext + BIN - 1) // BIN,
                 n_long=sum(1 for e in ext if e > LONG_E), long_k=[k for k, r in order if lay["labels"][r] == "long"],
                 decoys=len(decoys), sum=seq_sum([k for k, _ in order]), concat=concat_sums(order, n_runs), n_records=len(lines),
                 seq_bits=8 if eight_bit else 4, probe_local=lay["P"], head=H,
                 head_in_bin=sum(1 for c in recs if c[2] == "head" and (int(c[3]) - 1) // BIN == P // BIN))
    if lay["labels"] == ["b-1", "b"] and max_ext <= BIN:
        # depth_walk_two's windows over the slots of bins b-1 and b (SAM order in a bin): the sums a correct merge, a merge whose
        # `limit` is the larger key, and one that concatenates each round's entries run by run get at P
        cover = dict(meta)
        slots = [[], []]
        for a, c in enumerate(recs):
            if c[2] != "probe":
                continue
            s, L = int(c[3]) - 1 + H, entries(c[5])
            b = P // BIN - s // BIN
            if L <= LONG_E and b in (0, 1):
                slots[1 - b].append((a, s < sub_lo + SUB and s + L > sub_lo, cover.get(a, 0.0)))
        facts["merge"] = {m: seq_sum_inv(merge_two(slots, m)) for m in ("ok", "max", "batch")}
        facts["windows"] = [(len(x) + 31) // 32 for x in slots]
    parts = ([("head", head)] if H else []) + [("probe", probe), ("filler", filler)]
    c = Case(fasta(parts), ["\n".join(lines) + "\n"], dict(opts or {}))
    c.facts = facts
    return c


# k multisets over P and the boundary they sum to.  min_depth boundaries: the depth equals min_depth ("on": changed to Y) or is one
# ulp below it (low depth: kept).  half: depth 7 with fraction_invalid 0.5 against an allele seen 3 times (changed, or too close).
# print: 3.25 or one ulp above, printed "3.2" or "3.3" by --debug / --changes (both changed).
WIDE18 = [3] * 30 + [6] * 30 + [10] * 30                 # 90 reads: at least 40 per run of depth_walk_two
MIX20 = [3] * 27 + [5] * 25 + [6] * 30 + [10] * 10       # 92 reads
K34_MIN = [1] * 4 + [34] * 34                            # k > 32: the walk divides instead of reading its 1/k table
K35_HALF = [1] * 6 + [35] * 35
PRINT = [12, 6, 3, 12, 6, 10, 6, 1, 10, 3, 6, 5, 10, 6, 12]
HALF_OPTS = dict(min_depth=1, fraction_valid=0.9, fraction_invalid=0.5)

# name: (layout, multiset, target, side, options, x_reads, min reads per run, what the oracle prints as P's depth)
CASES = {
    "W1-two": ("two", WIDE18, 18.0, -1, dict(min_depth=18), 0, 40, b"18.0"),
    "W2-three": ("three", MIX20, 20.0, -1, dict(min_depth=20), 0, 8, b"20.0"),
    "W3-long": ("long", MIX20, 20.0, -1, dict(min_depth=20), 0, 8, b"20.0"),
    "W6-three-k34": ("three", K34_MIN, 5.0, -1, dict(min_depth=5), 0, 6, b"5.0"),
    "W6-long-k35": ("long", K35_HALF, 7.0, -1, HALF_OPTS, 3, 6, b"7.0"),
    "W8-two-print": ("two", PRINT, 3.25, 1, dict(min_depth=1), 0, 4, b"3.2"),
    "W8-three-print": ("three", PRINT, 3.25, 1, dict(min_depth=1), 0, 3, b"3.2"),
    "W8-long-print": ("long", PRINT, 3.25, 1, dict(min_depth=1), 0, 3, b"3.2"),
    "W4-tile-start": ("border_at", MIX20, 20.0, -1, dict(min_depth=20), 0, 30, b"20.0"),
    "W4-tile-end": ("border_before", MIX20, 20.0, -1, dict(min_depth=20), 0, 30, b"20.0"),
    "W5-contig-border": ("contig_border", K34_MIN, 5.0, -1, dict(min_depth=5), 0, 1, b"5.0"),
    "W7-three-8bit": ("three", MIX20, 20.0, -1, dict(min_depth=20), 0, 8, b"20.0"),
    "W7-long-8bit": ("long", K35_HALF, 7.0, -1, HALF_OPTS, 3, 6, b"7.0"),
}
WINDOWED = {"W1-two"}          # the on order must also cross the boundary under the two mis-merges of depth_walk_two


def crosses(x, target, side):
    return (x - target) * side > 0


def case_pair(name, seed=7):
    """The on and off cases of CASES[name]: (on_case, off_case, spec).  For WINDOWED cases the search goes on (other orders, other
    decoy placements) until the merge model of the on case also crosses the boundary with `limit` = the larger key and with each
    round concatenated run by run."""
    lay, ks, target, side, opts, x_reads, per_run, printed = CASES[name]
    layout = LAYOUTS[lay]()
    eight = "8bit" in name
    for attempt in range(200):
        on, off = run_orders(seed + 1000 * attempt, ks, target, len(layout["runs"]), side=side, min_per_run=per_run)
        for ds in range(20 if name in WINDOWED else 1):
            c_on = walk_case(seed + 100 * ds, on, layout, x_reads=x_reads, opts=opts, eight_bit=eight)
            m = c_on.facts.get("merge")
            if name not in WINDOWED or (m["ok"] == target and crosses(m["max"], target, side) and crosses(m["batch"], target, side)):
                c_off = walk_case(seed + 100 * ds + 1, off, layout, x_reads=x_reads, opts=opts, eight_bit=eight)
                return c_on, c_off, dict(target=target, side=side, printed=printed, layout=lay, labels=layout["labels"], per_run=per_run,
                                         windowed=name in WINDOWED, eight_bit=eight)
    raise AssertionError("no case for %s" % name)


# ---- W9: high cover ----------------------------------------------------------------------------------------------------------
def bankers(x):
    """misc.rs:208-215 on a non-negative double."""
    rd = int(x)
    fr = x - math.trunc(x)
    return rd if fr < 0.5 else rd + 1 if fr > 0.5 else rd + (rd & 1)


def high_cover(seed=9, n1=100_000, n3=100_000, fv_near=0.85, fi=0.7):
    """W9: n1 reads with one alignment, then n3 reads with three (two secondaries on `filler`), all over P in that SAM order and split
    between bins b-1 and b.  Where the reference's sum d_ref sits below the fixed-point value d_fx by more than n 2^-41, only the n^2
    term of depth_bounds keeps d_ref inside the bound.  c of the covering reads carry Y, and fraction_valid puts the rounding tie
    B = (c + 1/2) / fv strictly between d_ref and d_fx - n 2^-41: the reference changes P (its valid threshold is c), while a bound
    without the n^2 term would lie wholly above B (threshold c + 1: P kept) and so would never walk."""
    from fractions import Fraction
    rng = random.Random(seed)
    lay = layout_two()
    P = lay["P"]
    probe = rand_seq(rng, lay["length"])
    flen = 8_000
    filler = rand_seq(rng, flen)
    y = [b for b in "ACGT" if b != probe[P]][0]
    n = n1 + n3
    d_ref = seq_sum([1] * n1 + [3] * n3)
    dd3 = (1 << 40) - round(Fraction(1 << 40, 3))
    x = n - Fraction(n3 * dd3, 1 << 40)                         # d_fx, exactly
    lo_nn = x - Fraction(n, 1 << 41)                            # the lower end of the bound without its n^2 term
    mid = (Fraction(d_ref) + lo_nn) / 2
    c = int(mid * Fraction(fv_near) - Fraction(1, 2))
    fv = float((c + Fraction(1, 2)) / mid)
    lines = []
    nsec = 0
    runs = [0, 0]
    for i in range(n):
        k = 1 if i < n1 else 3
        r = i % 2
        runs[r] += 1
        lo, hi, L = lay["runs"][r]
        s = lo + (i // 2) % (hi - lo + 1)
        base = y if (i + 1) * c // n > i * c // n else probe[P]
        q = "r%d" % i
        lines.append(sam(q, 16 if i % 4 >= 2 else 0, "probe", s, "%dM" % L, probe[s:P] + base + probe[P + 1:s + L], 1))
        for _ in range(k - 1):
            fpos = 10 + (37 * nsec) % (flen - 80)
            nsec += 1
            lines.append(sam(q, 256, "filler", fpos, "60M", "*", 0))
    facts = dict(P=P, n=n, c=c, fv=fv, fi=fi, d_ref=d_ref, d_fx=float(x), runs=dict(zip(lay["labels"], runs)),
                 ref_outside=abs(Fraction(d_ref) - x) > Fraction(n, 1 << 41),
                 ref_threshold=bankers(d_ref * fv), nn_threshold=bankers(float(lo_nn) * fv),
                 draft_below_invalid=n - c < bankers(d_ref * fi), n_records=len(lines))
    case = Case(fasta([("probe", probe), ("filler", filler)]), ["\n".join(lines) + "\n"], dict(fraction_valid=fv, fraction_invalid=fi))
    case.facts = facts
    return case
