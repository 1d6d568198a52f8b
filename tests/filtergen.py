"""Cases for the filter's insert-size select and pair verdicts, and an exact model of `polypolish filter` (filter.rs) to check them with.

The model restates filter.rs over mate arrays in plain Python integers: get_orientation (:189-209), get_insert_size (:212-218),
auto_determine_orientation (:238-246), get_percentile (:249-259, f64 `ceil`, `max(1)`, `unwrap_or(0)`) and alignment_pass_qc
(:352-377).  A record is (name id, contig id, ref_start, ref_end, reverse), ref_start 0-based; every case is also written as the two SAM
texts (QNAME `q<id>`, RNAME `ctg<id>`, POS = ref_start + 1, CIGAR `<ref_end - ref_start>M`).

The select on the device is a radix select of the two nearest ranks, one 8-bit digit per round, most significant first.  `radix_select`
restates it, and can run it with one of three mistakes (MUTATIONS): a dropped round, `rank < c` for `rank <= c` in the pick, or rank 1
counted under rank 0's prefix.  `sharp(case, mutation)` says whether that mistake changes a threshold *and* a verdict of the case, so a
case that is sharp for a mistake would catch it.  Every case carries probes: multi-mapped reads whose only same-contig mate gives an
insert of low - 1, low, high and high + 1, so any change of a threshold changes a verdict.
"""
import math
import random

import numpy as np

ORIENT = ["fr", "rf", "ff", "rr"]
MAX_COORD = 0xFFFFFFFE                                  # the filter's coordinate limit (ref_end <= 2^32 - 2)
MUTATIONS = ["drop0", "drop1", "drop2", "drop3", "lt", "prefix0"]


class ModelError(Exception):
    pass


# ---- the model (filter.rs) ------------------------------------------------------------------------------------------------------
def get_orientation(a, b):
    """filter.rs:189-209 on (start, end, reverse) triples."""
    strand_1, strand_2 = ("r" if a[2] else "f"), ("r" if b[2] else "f")
    a_1_pos = a[1] if a[2] else a[0]
    a_2_pos = b[1] if b[2] else b[0]
    if strand_1 != strand_2:
        return strand_1 + strand_2 if a_1_pos < a_2_pos else strand_2 + strand_1
    if strand_1 == "f":
        return "ff" if a_1_pos < a_2_pos else "rr"
    return "ff" if a_2_pos < a_1_pos else "rr"


def get_insert_size(a, b):
    positions = [a[0], a[1], b[0], b[1]]
    return (max(positions) - min(positions)) & 0xFFFFFFFF


def nearest_rank(percentile, n):
    """filter.rs:256-257: max(1, ceil(percentile / 100 * n)), in f64."""
    return max(1, math.ceil(percentile / 100.0 * float(n)))


def get_percentile(sorted_list, percentile):
    if not sorted_list:
        return 0
    rank = nearest_rank(percentile, len(sorted_list))
    return sorted_list[rank - 1] if rank - 1 < len(sorted_list) else 0


def auto_determine_orientation(counts):
    max_count = max(counts)
    orientations = [o for o, c in zip(ORIENT, counts) if c == max_count]
    if len(orientations) != 1:
        raise ModelError("could not automatically determine read pair orientation")
    return orientations[0]


def pick_digit(hist, rank, lt=False):
    d = 0
    while d < 256:
        c = int(hist[d])
        if (rank < c) if lt else (rank <= c):
            break
        rank -= c
        d += 1
    return min(d, 255), rank


def radix_select(values, ranks, mutation=None, trace=None):
    """The device's select of two 1-based ranks over `values`, optionally with one of MUTATIONS.  trace (a list) receives, per
    round and rank, (digit, rank inside its bucket, the bucket's count)."""
    v = np.asarray(values, dtype=np.uint64)
    shifts = [24, 16, 8, 0]
    if mutation and mutation.startswith("drop"):
        shifts.remove(8 * int(mutation[4:]))
    prefix, rank, done = [0, 0], list(ranks), 0
    for shift in shifts:
        digits = (v >> np.uint64(shift)) & np.uint64(255)
        row = []
        for r in range(2):
            p = prefix[0] if (r == 1 and mutation == "prefix0") else prefix[r]
            row.append(np.bincount(digits[(v & np.uint64(done)) == np.uint64(p)].astype(np.int64), minlength=256))
        picked = []
        for r in range(2):
            d, rank[r] = pick_digit(row[r], rank[r], lt=(mutation == "lt"))
            prefix[r] |= d << shift
            picked.append((d, rank[r], int(row[r][d])))
        if trace is not None:
            trace.append(picked)
        done |= 255 << shift
    return prefix


def thresholds(sizes, low_pct, high_pct, mutation="exact"):
    """(low, high) from the insert sizes of the chosen orientation: sort + get_percentile, or the radix select (mutation None for
    the correct one)."""
    sizes = sorted(sizes)
    if mutation == "exact":
        return get_percentile(sizes, low_pct), get_percentile(sizes, high_pct)
    n = len(sizes)
    ranks = [nearest_rank(low_pct, n), nearest_rank(high_pct, n)]
    got = radix_select(sizes, [r if r <= n else 1 for r in ranks], mutation)
    return tuple(got[i] if ranks[i] <= n else 0 for i in range(2))


def model(case, mutation="exact"):
    """`polypolish filter` on the case's arrays: dict(pairs, orientation, low, high, pass1, pass2, n_pass), or ModelError."""
    recs = case.recs
    by_name = [{}, {}]
    for k in range(2):
        for i, r in enumerate(recs[k]):
            by_name[k].setdefault(r[0], []).append(i)
    sizes = {o: [] for o in ORIENT}
    for nid, l1 in by_name[0].items():                   # filter.rs:155-167
        l2 = by_name[1].get(nid)
        if len(l1) != 1 or not l2 or len(l2) != 1:
            continue
        a, b = recs[0][l1[0]], recs[1][l2[0]]
        if a[1] == b[1]:
            sizes[get_orientation(a[2:], b[2:])].append(get_insert_size(a[2:], b[2:]))
    counts = [len(sizes[o]) for o in ORIENT]
    if sum(counts) == 0:
        raise ModelError("no one-alignment-per-read pairs available to determine orientation and insert size thresholds")
    chosen = auto_determine_orientation(counts) if case.orientation == "auto" else case.orientation
    if not sizes.get(chosen):
        raise ModelError("no read pairs available to determine insert size thresholds")
    low, high = thresholds(sizes[chosen], case.low, case.high, mutation)
    passes = []
    for k in range(2):                                   # alignment_pass_qc, filter.rs:352-377
        out = []
        for r in recs[k]:
            this, pair = by_name[k][r[0]], by_name[1 - k].get(r[0], [])
            ok = not pair or len(this) == 1
            for j in pair:
                if ok:
                    break
                m = recs[1 - k][j]
                ins = get_insert_size(r[2:], m[2:])
                ok = r[1] == m[1] and low <= ins <= high and get_orientation(r[2:], m[2:]) == chosen
            out.append(1 if ok else 0)
        passes.append(out)
    return dict(pairs=counts, orientation=chosen, low=low, high=high, pass1=passes[0], pass2=passes[1],
                n_pass=sum(passes[0]) + sum(passes[1]))


def sharp(case, mutation):
    """True when `mutation` of the select changes a threshold and at least one verdict of the case."""
    good, bad = model(case), model(case, mutation)
    return (good["low"], good["high"]) != (bad["low"], bad["high"]) and (good["pass1"], good["pass2"]) != (bad["pass1"], bad["pass2"])


def select_trace(case, m=None):
    """Per round and rank: (digit, rank inside its bucket, bucket count) of the correct radix select over the chosen sizes."""
    m = m or model(case)
    sizes = sorted(unique_sizes(case)[m["orientation"]])
    n = len(sizes)
    ranks = [nearest_rank(case.low, n), nearest_rank(case.high, n)]
    tr = []
    radix_select(sizes, [r if r <= n else 1 for r in ranks], None, tr)
    return tr


def unique_sizes(case):
    by_name = [{}, {}]
    for k in range(2):
        for r in case.recs[k]:
            by_name[k].setdefault(r[0], []).append(r)
    sizes = {o: [] for o in ORIENT}
    for nid, l1 in by_name[0].items():
        l2 = by_name[1].get(nid, [])
        if len(l1) == 1 and len(l2) == 1 and l1[0][1] == l2[0][1]:
            sizes[get_orientation(l1[0][2:], l2[0][2:])].append(get_insert_size(l1[0][2:], l2[0][2:]))
    return sizes


# ---- cases ----------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, seed, orientation="auto", low=0.1, high=99.9):
        self.name, self.orientation, self.low, self.high = name, orientation, low, high
        self.rng = random.Random(seed)
        self.recs = [[], []]
        self.n_names = 0
        self.sharp_for = []                             # mutations this case must be sharp for
        self.digit = None

    def new_name(self):
        self.n_names += 1
        return self.n_names - 1

    def rec(self, k, nid, contig, start, end, rev):
        assert 0 <= start <= end <= MAX_COORD
        self.recs[k].append((nid, contig, start, end, bool(rev)))

    def mates(self, ins, orient, start=None):
        """Two (start, end, reverse) triples with this orientation and insert size, or None when no such layout exists."""
        if orient == "fr":
            a = min(100, ins)
            shape = ((0, a, False), (ins - a, ins, True))
        elif orient == "rf":
            a = min(100, (ins - 1) // 2)
            shape = ((0, a, True), (ins - a, ins, False))
        elif orient == "ff":
            a = min(100, ins - 1)
            shape = ((0, a, False), (ins - a, ins, False))
        else:
            a = min(100, ins - 1)
            shape = ((ins - a, ins, False), (0, a, False))
        if ins < 1 or ins > MAX_COORD or a < 1:
            return None
        s = self.rng.randint(0, MAX_COORD - ins) if start is None else start
        m1, m2 = [(s + x, s + y, rv) for x, y, rv in shape]
        assert get_orientation(m1, m2) == orient and get_insert_size(m1, m2) == ins, (orient, ins)
        return m1, m2

    def pair(self, ins, orient="fr", contig=0):
        """A unique pair (one record per mate, same contig)."""
        m = self.mates(ins, orient)
        nid = self.new_name()
        self.rec(0, nid, contig, *m[0])
        self.rec(1, nid, contig, *m[1])

    def probe(self, ins, orient, second_first=False):
        """A multi-mapped read: mate 1 has the candidate alignment (insert `ins`, orientation `orient` to mate 2's only alignment)
        and a second one on another contig at the same coordinates; mate 2 has one alignment (which passes: cnt == 1)."""
        m = self.mates(ins, orient)
        if m is None:
            return False
        nid = self.new_name()
        recs = [(nid, 0) + m[0], (nid, 1) + m[0]]
        for r in (recs[::-1] if second_first else recs):
            self.rec(0, *r)
        self.rec(1, nid, 0, *m[1])
        return True

    def add_probes(self):
        m = model(self)
        for k, ins in enumerate((m["low"] - 1, m["low"], m["high"], m["high"] + 1)):
            self.probe(ins, m["orientation"], second_first=bool(k & 1))
        return self

    def shuffled(self):
        """Records in a random file order (names are not consecutive; the filter groups by name anyway)."""
        for k in range(2):
            self.rng.shuffle(self.recs[k])
        return self

    # ---- text form --------------------------------------------------------------------------------------------------------------
    def lines(self, k):
        seen, out = set(), []
        for nid, contig, s, e, rev in self.recs[k]:
            flag = (16 if rev else 0) | (256 if nid in seen else 0)
            seen.add(nid)
            out.append(f"q{nid}\t{flag}\tctg{contig}\t{s + 1}\t60\t{e - s}M\t*\t0\t0\tACGT\tIIII\tNM:i:0")
        return out

    def texts(self):
        return tuple(("@HD\tVN:1.6\n" + "".join(x + "\n" for x in self.lines(k))).encode() for k in range(2))

    def expected_texts(self, m=None):
        m = m or model(self)
        res = []
        for k, pas in enumerate((m["pass1"], m["pass2"])):
            res.append(("@HD\tVN:1.6\n" + "".join(x + ("\n" if p else "\tZP:Z:fail\n") for x, p in zip(self.lines(k), pas))).encode())
        return tuple(res)

    def arrays(self):
        """The pp_filter_mate arrays of both mates (numpy)."""
        out = []
        for k in range(2):
            r = self.recs[k]
            out.append(dict(name_id=np.array([x[0] for x in r], np.uint32), contig=np.array([x[1] for x in r], np.uint32),
                            ref_start=np.array([x[2] for x in r], np.uint32), ref_end=np.array([x[3] for x in r], np.uint32),
                            flags=np.array([1 if x[4] else 0 for x in r], np.uint8)))
        return out

    @property
    def orientation_code(self):
        return -1 if self.orientation == "auto" else (ORIENT.index(self.orientation) if self.orientation in ORIENT else 4)


def pct_for_rank(rank, n):
    """A percentile whose nearest rank over n values is `rank` (half a rank below it, far from any f64 edge)."""
    p = 100.0 * (rank - 0.5) / n
    assert nearest_rank(p, n) == rank
    return p


def digit_values(rng, d, top_lo, top_hi, mode):
    """A cluster around one rank value v: v's highest differing digit from every neighbour is d.  mode 'first': the other values of
    v's round-d bucket (same digits >= d) lie above v; 'last': below.  Returns (values, v)."""
    unit = 1 << (8 * d)
    digs = [rng.randint(1, 254) for _ in range(4)]
    digs[3] = rng.randint(top_lo, top_hi)
    v = sum(x << (8 * i) for i, x in enumerate(digs))
    low_mask = unit - 1
    vals = [v, v - unit, v + unit]                                   # differ only in digit d
    vals += [(v & ~low_mask) - 1, (v | low_mask) + 1]                # 0x..FF / 0x..100: the carries into and out of v's bucket
    hi_mask = ~((unit << 8) - 1) & 0xFFFFFFFF
    span = range(256) if d < 3 else range(top_lo - 1, top_hi + 2)   # (digit 3 stays inside the cluster's range)
    for _ in range(rng.randint(3, 7)):                               # decoys with v's higher digits, another digit d
        dd = rng.choice([x for x in span if abs(x - digs[d]) > 1])
        vals.append((v & hi_mask) | (dd << (8 * d)) | rng.randint(0, low_mask))
    for _ in range(rng.randint(2, 4)):                               # v's round-d bucket
        if d == 0:
            vals.append(v)                                           # (in round 0 the bucket holds copies of v)
        elif mode == "first":
            vals.append((v & ~low_mask) | rng.randint((v & low_mask) + 1, low_mask))
        else:
            vals.append((v & ~low_mask) | rng.randint(0, (v & low_mask) - 1))
    return vals, v


def digit_case(d, mode, seed):
    """Low and high ranks on values whose neighbours differ from them first in digit d; low's digit 3 is small and high's large, so
    the ranks part in round 24.  mode 'first': the low rank is first in its round-d bucket and the high rank last; 'last': the reverse."""
    c = Case(f"digit{d}_{mode}", seed)
    rng = c.rng
    hi_mode = "last" if mode == "first" else "first"
    lo_vals, lo_v = digit_values(rng, d, 1, 0x3C, mode)
    hi_vals, hi_v = digit_values(rng, d, 0x84, 0xFD, hi_mode)
    fill = [rng.randint(0x41000000, 0x7EFFFFFF) for _ in range(len(lo_vals) + len(hi_vals) + 6)]
    if d == 3:
        hi_vals.append(MAX_COORD)                                    # the largest insert the filter takes
    vals = sorted(lo_vals + fill + hi_vals)
    n = len(vals)
    at = lambda v, m: vals.index(v) + 1 if m == "first" else n - vals[::-1].index(v)
    rank_lo, rank_hi = at(lo_v, mode), at(hi_v, hi_mode)
    c.low, c.high = pct_for_rank(rank_lo, n), pct_for_rank(rank_hi, n)
    assert 0 < c.low < 50 < c.high < 100
    for v in rng.sample(vals, n):
        c.pair(v)
    c.digit = d
    c.sharp_for = [f"drop{d}", "lt", "prefix0"]
    return c.add_probes().shuffled()


def ties_all(seed):
    c = Case("ties_all", seed)
    for _ in range(40):
        c.pair(0x01020304)
    c.sharp_for = ["drop0", "drop1", "drop2", "drop3", "lt"]
    return c.add_probes().shuffled()


def ties_carry(seed, below, k=10):
    """A tied run of `below` and one of below + 1 (a carry across digits): the low rank is the last of the first run, the high rank
    the first of the second."""
    c = Case(f"ties_carry_{below:08x}", seed)
    for _ in range(k):
        c.pair(below)
        c.pair(below + 1)
    c.low, c.high = pct_for_rank(k, 2 * k), pct_for_rank(k + 1, 2 * k)
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def small_n(n, seed, low=0.1, high=99.9):
    c = Case(f"small_n{n}_{low}_{high}", seed, low=low, high=high)
    for _ in range(n):
        c.pair(c.rng.randint(0x100, 0xFFFFFF00))
    c.sharp_for = ["lt"]
    return c.add_probes()


def rank_edge_pairs(lo=20, hi=400):
    """(n, p) with p / 100 * n an exact integer in f64 (kind 'exact') or one ulp above an integer ('ulp'), for low and high
    percentiles in tenths."""
    found = {}
    for n in range(lo, hi):
        for t in range(1, 1000):
            if t == 500:
                continue
            p = t / 10.0
            x = p / 100.0 * float(n)
            k = math.floor(x)
            kind = "exact" if x == k else ("ulp" if x == math.nextafter(float(k), math.inf) else None)
            if kind:
                found.setdefault((kind, p < 50), []).append((n, p))
    return found


def rank_edge_case(seed, low_kind, high_kind):
    """n distinct values (all four digits vary) and percentiles where the f64 rank arithmetic lands on an integer or one ulp above."""
    edges = rank_edge_pairs()
    rng = random.Random(seed)
    for _ in range(10000):
        n, lp = rng.choice(edges[(low_kind, True)])
        hp = [p for m, p in edges[(high_kind, False)] if m == n]
        if hp:
            break
    c = Case(f"rank_edge_{low_kind}_{high_kind}_n{n}", seed, low=lp, high=rng.choice(hp))
    for v in rng.sample(range(1, MAX_COORD + 1), n):
        c.pair(v)
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def verdicts(seed):
    """Thresholds from ~N(5e6, 2e5) inserts; multi-mapped reads on both mates whose candidates give inserts of low - 1, low, high,
    high + 1 or another value, in all four orientations and on either contig."""
    c = Case("verdicts", seed)
    rng = c.rng
    for _ in range(300):
        c.pair(max(200, int(rng.gauss(5_000_000, 200_000))))
    m = model(c)
    lo, hi = m["low"], m["high"]
    for _ in range(120):
        nid = c.new_name()
        for k_mate in range(rng.choice([1, 2, 3])):
            ins = rng.choice([lo - 1, lo, hi, hi + 1, rng.randint(lo, hi), rng.randint(1, 10 * hi)])
            o = rng.choice(ORIENT + ["fr"] * 4)
            mm = c.mates(ins, o)
            if mm is None:
                continue
            c.rec(0, nid, rng.choice([0, 0, 0, 1]), *mm[0])
            c.rec(1, nid, rng.choice([0, 0, 0, 1]), *mm[1])
        if rng.random() < 0.5:
            c.rec(0, nid, 0, *c.mates(rng.randint(1, 1000), "fr")[0])
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def position_ties(strands, seed):
    """Unique pairs whose read starts are equal (p1 == p2), strands (mate 1, mate 2) = `strands`: filter.rs:199-206 name them
    fr -> 'rf', rf -> 'fr', ff -> 'rr', rr -> 'rr'.  They outnumber a set of 'fr' pairs (or 'ff' ones), so the tie decides the
    orientation; probes in each tie layout then pass only if their tie names the chosen orientation."""
    c = Case(f"position_ties_{strands}", seed)
    rng = c.rng

    def tie(a, b, s=None):
        s = rng.randint(1000, MAX_COORD - 1000) if s is None else s
        r1, r2 = strands[0] == "r", strands[1] == "r"
        m1 = (s - a, s, True) if r1 else (s, s + a, False)
        m2 = (s - b, s, True) if r2 else (s, s + b, False)
        return m1, m2
    for _ in range(30):
        m1, m2 = tie(rng.randint(1, 150), rng.randint(1, 150))
        nid = c.new_name()
        c.rec(0, nid, 0, *m1)
        c.rec(1, nid, 0, *m2)
    other = "ff" if strands == "rf" else "fr"
    for _ in range(12):
        c.pair(rng.randint(150, 300), other)
    m = model(c)
    assert m["orientation"] == {"fr": "rf", "rf": "fr", "ff": "rr", "rr": "rr"}[strands]
    for st in ("fr", "rf", "ff", "rr"):                  # tie probes of every layout, insert = high
        for _ in range(2):
            nid = c.new_name()
            r1, r2 = st[0] == "r", st[1] == "r"
            s = rng.randint(1000, MAX_COORD - 1000)
            a = m["high"] if r1 == r2 else m["high"] // 2       # same strand: the longer one spans the insert; else the two add up
            b = max(1, m["high"] // 2) if r1 == r2 else m["high"] - a
            m1 = (s - a, s, True) if r1 else (s, s + a, False)
            m2 = (s - b, s, True) if r2 else (s, s + b, False)
            assert get_insert_size(m1, m2) == m["high"]
            c.rec(0, nid, 0, *m1)
            c.rec(0, nid, 1, *m1)
            c.rec(1, nid, 0, *m2)
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def other_contigs(seed):
    """Mates on another contig at the same coordinates: not pairs (filter.rs:161), and no good candidate (:369)."""
    c = Case("other_contigs", seed)
    rng = c.rng
    for _ in range(60):
        c.pair(rng.randint(200, 400))
    for _ in range(40):                                  # one record per mate, other contig: not a pair
        m = c.mates(rng.randint(200, 400), "fr")
        nid = c.new_name()
        c.rec(0, nid, 0, *m[0])
        c.rec(1, nid, 1, *m[1])
    m = model(c)
    for _ in range(20):                                  # a perfect candidate on the other contig only
        mm = c.mates(rng.randint(m["low"], m["high"]), "fr", start=rng.randint(0, 1 << 31))
        nid = c.new_name()
        c.rec(0, nid, 1, *mm[0])
        c.rec(0, nid, 1, mm[0][0] + 5000, mm[0][1] + 5000, False)
        c.rec(1, nid, 0, *mm[1])
        c.rec(1, nid, 2, *mm[1])
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def one_mate(seed):
    """Reads with records in one file only (they pass: filter.rs:362-364), and reads with one record against several mate records
    that all miss (the one record passes, :365-367; the several fail)."""
    c = Case("one_mate", seed)
    rng = c.rng
    for _ in range(50):
        c.pair(rng.randint(250, 350))
    for k in range(2):
        for _ in range(10):
            nid = c.new_name()
            for _ in range(rng.randint(1, 3)):
                c.rec(k, nid, 0, *c.mates(rng.randint(250, 350), "fr")[k])
    for k in range(2):
        for _ in range(10):
            nid = c.new_name()
            s = rng.randint(0, 1 << 30)
            c.rec(k, nid, 0, s, s + 100, k == 1)
            for _ in range(rng.randint(2, 3)):
                t = s + rng.randint(100_000, 1 << 20)
                c.rec(1 - k, nid, 0, t, t + 100, k == 0)
    c.sharp_for = ["lt"]
    return c.add_probes().shuffled()


def cases():
    """Every case of the CPU and text GPU tests (the large one is separate: large_case)."""
    out = []
    for d in range(4):
        for i, mode in enumerate(("first", "last")):
            out.append(digit_case(d, mode, 100 + 10 * d + i))
    out += [ties_all(200), ties_carry(201, 0x00FFFFFF), ties_carry(202, 0x0A0B00FF), small_n(1, 210), small_n(2, 211),
            small_n(2, 212, 49.9, 50.1), rank_edge_case(220, "exact", "ulp"), rank_edge_case(221, "ulp", "exact"),
            rank_edge_case(222, "ulp", "ulp"), verdicts(230)]
    out += [position_ties(s, 240 + i) for i, s in enumerate(("fr", "rf", "ff", "rr"))]
    out += [other_contigs(250), one_mate(251)]
    return out


def large_case(n=4 << 20, seed=300):
    """4 M unique 'fr' pairs: half of the inserts 0x000180xx (round 8's bucket of both ranks holds ~2 M names, round 0's ~8 K), the
    rest 0x0001xxxx; ranks at 40 % and 60 %; probes.  Arrays only: rec() lists are built with numpy and turned into tuples once."""
    rng = np.random.default_rng(seed)
    c = Case("large_4M", seed, low=40.0, high=60.0)
    heavy = rng.random(n) < 0.5
    ins = np.where(heavy, 0x00018000 | rng.integers(0, 256, n), 0x00010000 | rng.integers(0, 0x10000, n)).astype(np.int64)
    start = rng.integers(0, 1 << 31, n).astype(np.int64)
    a = np.minimum(100, ins)
    ids = np.arange(n)
    c.recs[0] = list(zip(ids.tolist(), [0] * n, start.tolist(), (start + a).tolist(), [False] * n))
    c.recs[1] = list(zip(ids.tolist(), [0] * n, (start + ins - a).tolist(), (start + ins).tolist(), [True] * n))
    c.n_names = n
    c.sharp_for = ["lt", "drop0", "drop1", "drop2"]
    return c.add_probes()
