"""SAM texts whose read groups straddle the byte ranges of multi-GPU ingestion, and a plain model of how the reference groups records.

`polish --gpus N` cuts every SAM file into N byte ranges (pp_sam_split_ranges); each GPU tokenises its range and opens a new read group at
the range's first alignment.  A cut inside one of the reference's read groups therefore turns that group into two, each with its own k.
The reference (alignment.rs:238-264) groups by aligned records only: blank lines, '@' lines and unaligned records (FLAG & 4) are
skipped without closing the open group, and a record with an empty QNAME joins the group of the record after it.

- ref_groups: that grouping, restated.
- old_cuts: the earlier cut rule (before the first line whose QNAME differs from the previous line's, or before any '@' line), kept
  as the model of a rule that splits groups.
- group_case: FASTA + SAM cases in which a split group changes the vote at a probe position P (the facts say by how much).
- order_case: FASTA + SAM cases in which P's depth sits on a vote boundary only in (file, range, line) order of the pieces.
"""
import random
from fractions import Fraction

from tests import fuzzgen
from tests.fuzzgen import Case
from tests.limitgen import fasta, rand_seq, sam

NS = (1, 2, 3, 4, 8, 16, 32)             # range counts the CPU test cuts every text into
GPU_NS = (2, 3, 8)                       # context counts of the GPU tests


def lines_of(data):
    """(start, line without its newline and one trailing CR) of every line of a SAM text, as Rust's BufRead::lines() gives them."""
    out, pos = [], 0
    while pos < len(data):
        nl = data.find(b"\n", pos)
        end = len(data) if nl < 0 else nl
        line = data[pos:end]
        out.append((pos, line[:-1] if line.endswith(b"\r") else line))
        pos = end + 1
    return out


def ref_groups(data):
    """alignment.rs:238-264: [(line start, group index)] of every aligned record.  Empty and '@' lines are skipped, so are records
    with FLAG & 4; a record joins the open group iff the open name is empty or equals its QNAME; a file starts with no open group."""
    out, gid, cur = [], -1, None
    for start, line in lines_of(data):
        if not line or line.startswith(b"@"):
            continue
        f = line.split(b"\t")
        if int(f[1]) & 4:
            continue
        if cur is None or not (cur == b"" or cur == f[0]):
            gid += 1
        out.append((start, gid))
        cur = f[0]
    return out


def old_cuts(data, n):
    """The earlier split_ranges rule, restated: each cut moves from g * S / n to the first line start, then on to the first line whose
    QNAME (the text before its first tab) differs from the previous line's, or that starts with '@'."""
    S = len(data)
    cut = [S] * (n + 1)
    cut[0] = 0

    def line_at(pos):
        nl = data.find(b"\n", pos)
        ln = (nl if nl >= 0 else S) - pos
        t = data.find(b"\t", pos, pos + ln)
        return data[pos:(t if t >= 0 else pos + ln)], pos + ln + 1

    for g in range(1, n):
        pos = max(S // n * g, cut[g - 1])
        if pos >= S:
            continue
        if pos > 0:
            pos = min(line_at(pos - 1)[1], S)
        if pos >= S:
            continue
        qa, cand = line_at(pos)
        cand = min(cand, S)
        while cand < S:
            qb, nb = line_at(cand)
            if qb != qa or qb[:1] == b"@":
                break
            qa, cand = qb, min(nb, S)
        cut[g] = max(cand, cut[g - 1])
    return cut


def sam_cuts(path, n):
    """pp_sam_split_ranges: the n + 1 cuts of the file at `path`."""
    import ctypes as C
    from polypolish_b200 import api
    L = api.lib()
    L.pp_sam_split_ranges.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_uint64)]
    cuts = (C.c_uint64 * (n + 1))()
    rc = L.pp_sam_split_ranges(str(path).encode(), n, cuts)
    assert rc == 0, rc
    return list(cuts)


def range_of(cuts, pos):
    return max(i for i in range(len(cuts) - 1) if cuts[i] <= pos)


def split_groups(data, cuts):
    """The reference groups whose aligned records fall into more than one range of `cuts`."""
    where = {}
    for start, g in ref_groups(data):
        where.setdefault(g, set()).add(range_of(cuts, start))
    return sorted(g for g, r in where.items() if len(r) > 1)


def pieces(data, cuts):
    """The text of every range: what one file cut at `cuts` and read as separate files looks like to the reference."""
    return [data[cuts[i]:cuts[i + 1]] for i in range(len(cuts) - 1)]


# ---- texts -----------------------------------------------------------------------------------------------------------------------
UNALIGNED = "u%d\t4\t*\t0\t0\t*\t*\t0\t0\tACGT\tIIII"

# what goes inside (or in front of) each read group: "unaligned" an unaligned record of another name between its two records, "comment"
# an @CO line there, "blank" an empty line there, "empty" a record with an empty QNAME in front of it (that record joins it), "empty_run"
# two such records, "plain" nothing
KINDS = ("unaligned", "comment", "blank", "empty", "empty_run", "plain")


def group_lines(kind, i, recs):
    """The lines of read group i (records recs: the first covers the probe) with the insertion of `kind`; the records given an empty
    QNAME are the first ones."""
    r = list(recs)
    if kind in ("empty", "empty_run"):
        ne = 1 if kind == "empty" else 2
        r = ["\t".join([""] + x.split("\t")[1:]) if j < ne else x for j, x in enumerate(r)]
    if kind == "unaligned":
        r.insert(1, UNALIGNED % i)
    elif kind == "comment":
        r.insert(1, "@CO\tgroup %d" % i)
    elif kind == "blank":
        r.insert(1, "")
    return r


def toy_record(q, flag, pos):
    return sam(q, flag, "c1", pos, "50M", "A" * 50, 0)


def toy_text(kind, n_groups=300, eol="\n", terminated=True, seed=0):
    """n_groups two-record (three for empty_run) groups of `kind` on contig c1 (the CPU test: only the text matters)."""
    rng = random.Random(seed)
    lines = ["@HD\tVN:1.6", "@SQ\tSN:c1\tLN:5000"]
    for i in range(n_groups):
        recs = [toy_record("r%d" % i, 0, rng.randint(0, 4000))]
        recs += [toy_record("r%d" % i, 256, rng.randint(0, 4000)) for _ in range(2 if kind == "empty_run" else 1)]
        lines += group_lines(kind, i, recs)
    t = eol.join(lines) + (eol if terminated else "")
    return t.encode()


def fuzz_text(seed):
    """A fuzzgen SAM text with insertions of every kind put inside its read groups (between two records of one QNAME), and empty-QNAME
    records in front of some groups."""
    rng = random.Random(seed)
    case = fuzzgen.make_case(seed, n_files=1)
    t = case.sam_texts[0]
    eol = "\r\n" if "\r\n" in t else "\n"
    lines = t.split(eol)
    out = []
    for j, x in enumerate(lines):
        prev = out[-1].split("\t")[0] if out and out[-1] and not out[-1].startswith("@") else None
        q = x.split("\t")[0]
        if x and not x.startswith("@") and prev == q:
            r = rng.random()
            if r < 0.15:
                out.append(UNALIGNED % j)
            elif r < 0.25:
                out.append("@CO\tinside")
            elif r < 0.35:
                out.append("")
        elif x and not x.startswith("@") and rng.random() < 0.1:
            for _ in range(rng.choice([1, 1, 2, 3])):
                out.append("\t".join([""] + x.split("\t")[1:]))           # an empty-QNAME copy: joins the group after it
        out.append(x)
    return eol.join(out).encode()


def cpu_texts():
    """name -> SAM text (bytes) for the cut invariant."""
    t = {k: toy_text(k) for k in KINDS}
    t["empty_alone"] = toy_text("empty", n_groups=1)
    t["unaligned_crlf"] = toy_text("unaligned", eol="\r\n", seed=1)
    t["empty_crlf_unterminated"] = toy_text("empty_run", eol="\r\n", terminated=False, seed=2)
    t["blank_unterminated"] = toy_text("blank", terminated=False, seed=3)
    big = ["@HD\tVN:1.6"] + group_lines("unaligned", 0, [toy_record("big", 0, 10)] + [toy_record("big", 256, 20 + i) for i in range(3000)])
    big += [x for i in range(1, 40) for x in group_lines("comment", i, [toy_record("r%d" % i, 0, 5), toy_record("r%d" % i, 256, 9)])]
    t["group_larger_than_range"] = ("\n".join(big) + "\n").encode()
    t["two_lines"] = ("\n".join(group_lines("blank", 0, [toy_record("r", 0, 1), toy_record("r", 256, 2)])) + "\n").encode()
    t["one_unterminated_line"] = toy_record("r", 0, 1).encode()
    for s in range(6):
        t["fuzz%d" % s] = fuzz_text(100 + s)
    return t


# ---- GPU group cases -------------------------------------------------------------------------------------------------------------
N_FILLERS = 7            # eight contigs: `polish` over n contexts uses min(n, contigs) of them


def depth_at_p(data_list, over):
    """The reference's depth at P (exact): per file, per reference group, the group's records over P over its size (every record is a
    good alignment).  over: QNAME-free test of one line -> does the record cover P."""
    d = Fraction(0)
    for data in data_list:
        groups = {}
        lines = dict(lines_of(data))
        for start, g in ref_groups(data):
            groups.setdefault(g, []).append(over(lines[start]))
        d += sum((Fraction(sum(v), len(v)) for v in groups.values()), Fraction(0))
    return d


def careful_depth_at_p(data_list, over):
    d = 0
    for data in data_list:
        groups = {}
        lines = dict(lines_of(data))
        for start, g in ref_groups(data):
            groups.setdefault(g, []).append(over(lines[start]))
        d += sum(1 for v in groups.values() if len(v) == 1 and v[0])
    return d


def group_case(kind, careful=False, seed=1, eol="\n", n_fillers=N_FILLERS):
    """A probe contig with position P, covered by one record of each read group of `kind` (base Y != draft at P); the other records of
    the group sit on the filler contigs and carry their own SEQ (no SEQ="*": a split group would lose its source and go to the host
    packer).  Groups of four (one record over P) tune the depth; min_depth is the first integer above the reference's depth, so P keeps
    its draft base, and every group cut in two by old_cuts for n in GPU_NS adds at least the margin, so P would change.  With careful:
    five reads with one alignment over P (depth 5), min_depth 6, and a piece of a split group adds one.  Also a second SAM file of read pairs on the fillers (the mates for `filter`)."""
    for attempt in range(200):
        rng = random.Random(seed * 1000 + attempt)
        L, P = 1200, 600
        probe = rand_seq(rng, L)
        fill = [rand_seq(rng, 1500) for _ in range(n_fillers)]
        y = [b for b in "ACGT" if b != probe[P]][0]

        def over(q):
            a = rng.randint(P - 45, P - 5)
            return sam(q, 16 if rng.random() < 0.5 else 0, "probe", a, "60M", probe[a:P] + y + probe[P + 1:a + 60], 1)

        def filler(q):
            f = rng.randrange(n_fillers)
            a = rng.randint(0, 1500 - 60)
            return sam(q, 256 | rng.choice([0, 16]), "f%d" % (f + 1), a, "60M", fill[f][a:a + 60], 0)

        n_groups = rng.randint(61, 90)
        n_tune = attempt % 4
        lines = ["@HD\tVN:1.6", "@SQ\tSN:probe\tLN:%d" % L] + ["@SQ\tSN:f%d\tLN:1500" % (f + 1) for f in range(n_fillers)]
        pairs1, pairs2 = [], []
        for j in range(40):                              # read pairs on the fillers, one alignment per read (`filter`'s insert sizes)
            f = j % n_fillers
            a = rng.randint(0, 1500 - 400)
            pairs1.append(sam("p%d" % j, 0, "f%d" % (f + 1), a, "60M", fill[f][a:a + 60], 0))
            b = a + rng.randint(250, 300)
            pairs2.append(sam("p%d" % j, 16, "f%d" % (f + 1), b, "60M", fill[f][b:b + 60], 0))
        body = []
        for t in range(5 if careful else n_tune):                     # (with careful: reads with one alignment, over P)
            body += [over("t%d" % t)] + ([] if careful else [filler("t%d" % t) for _ in range(3)])
        for i in range(n_groups):
            q = "r%d" % i
            recs = [over(q)] + [filler(q) for _ in range(2 if kind == "empty_run" else 1)]
            body += group_lines(kind, i, recs)
            if pairs1 and rng.random() < 0.3:
                body.append(pairs1.pop())
        body += pairs1
        text = (eol.join(lines + body) + eol).encode()
        mates = ("\n".join(lines + pairs2) + "\n").encode()

        def covers(line):
            f = line.split(b"\t")
            return f[2] == b"probe"
        facts = dict(P=P, kind=kind, careful=careful, n_groups=n_groups, split={}, old_depth={})
        if careful:
            d = careful_depth_at_p([text], covers)
            facts["depth"], facts["min_depth"] = d, d + 1
            ok = d == 5
        else:
            d = depth_at_p([text], covers)
            facts["depth"], facts["min_depth"] = d, int(d) + 1
            ok = d != int(d)
        for n in GPU_NS:
            c = old_cuts(text, n)
            facts["split"][n] = split_groups(text, c)
            facts["old_depth"][n] = (careful_depth_at_p if careful else depth_at_p)(pieces(text, c), covers)
            ok = ok and facts["split"][n] and facts["old_depth"][n] - facts["min_depth"] >= (0 if careful else Fraction(1, 100))
        if not ok:
            continue
        opts = dict(min_depth=facts["min_depth"], careful=careful)
        case = Case(fasta([("probe", probe)] + [("f%d" % (f + 1), s) for f, s in enumerate(fill)]),
                    [text.decode(), mates.decode()], opts)
        case.facts = facts
        return case
    raise AssertionError("no group case for %s" % kind)


# ---- GPU order cases -------------------------------------------------------------------------------------------------------------
# Every destination context holds its records in global SAM order, (file, range, line): the pieces of every source range are placed at
# [file][range].  The reference's depth at a position is the sequential f64 sum of 1/k in that order, so a probe position P whose sum
# sits exactly on a vote boundary changes its vote if the pieces arrive in another order.  The wrong orders modelled (keys of a piece
# (f, r); o is the context that owns the probe contig, n the number of ranges):
def wrong_orders(n_files, n, o):
    return {"range_major": lambda f, r: (r, f), "ranges_reversed": lambda f, r: (f, -r),
            "files_swapped": lambda f, r: (n_files - 1 - f, r), "rotated": lambda f, r: (f, (o - r) % n)}


def owners(lengths, n):
    """plan_device_shards (host_api.cpp): min(n, contigs) shards; contigs longest first (a stable sort), each onto the lightest shard
    (the first of equally light ones)."""
    n = min(n, len(lengths))
    load, own = [0] * n, [0] * len(lengths)
    for c in sorted(range(len(lengths)), key=lambda c: -lengths[c]):
        b = load.index(min(load))
        own[c] = b
        load[b] += lengths[c]
    return own


def seq_sum(ks):
    s = 0.0
    for k in ks:
        s += 1.0 / k
    return s


def ordered(reads, key):
    """The k of reads [(k, (f, r))] (in SAM order within each piece) with the pieces in the order of `key`."""
    return [k for k, p in sorted(reads, key=lambda x: key(*x[1]))]


def piece_orders(seed, ks, target, side, n_files, n, o, tries=200_000):
    """Two SAM orders of the multiset ks over the pieces (file, range), every piece holding at least one read: `on`, whose sum of 1/k
    in (file, range, line) order is exactly `target` while every wrong order of wrong_orders gives a sum on the `side` of it; `off`,
    whose sum is one ulp beside the target on that side.  Lists of (k, (f, r)) in SAM order."""
    rng = random.Random(seed)
    import math
    off_target = math.nextafter(target, side * math.inf)
    pcs = [(f, r) for f in range(n_files) for r in range(n)]
    models = wrong_orders(n_files, n, o)
    ks = list(ks)
    on = off = None
    for _ in range(tries):
        rng.shuffle(ks)
        where = [pcs[i % len(pcs)] for i in range(len(pcs))] + [rng.choice(pcs) for _ in range(len(ks) - len(pcs))]
        rng.shuffle(where)
        reads = sorted(zip(ks, where), key=lambda x: x[1])               # (a stable sort: SAM order inside each piece kept)
        s = seq_sum([k for k, _ in reads])
        if s == target and on is None and all((seq_sum(ordered(reads, m)) - target) * side > 0 for m in models.values()):
            on = reads
        elif s == off_target and off is None:
            off = reads
        if on and off:
            return on, off
    raise AssertionError("no orders of %r over %d x %d pieces" % (target, n_files, n))


# name: (walkgen multiset, target, side, min_depth or other options, SAM files, ranges, 8-bit pool)
ORDER_CASES = {
    "W1-8ranges-2files": ("WIDE18", 18.0, -1, dict(min_depth=18), 2, 8, False),
    "W2-3ranges-3files": ("MIX20", 20.0, -1, dict(min_depth=20), 3, 3, False),
    "W8-print-2ranges-3files": ("PRINT", 3.25, 1, dict(min_depth=1), 3, 2, False),
    "W6-k34-3ranges-2files": ("K34_MIN", 5.0, -1, dict(min_depth=5), 2, 3, False),
    "W2-8bit-3ranges-2files": ("MIX20", 20.0, -1, dict(min_depth=20), 2, 3, True),
}

PAD_LEN = 6000


def order_case(name, on=True, seed=11):
    """ORDER_CASES[name] as a Case (on or off order).  Contigs: `pad` (the longest: context 0) carries padding reads, `probe` (context 1)
    the reads over P = 522, fillers the other records of their groups.  A covering read with k alignments is either its record over P
    (with SEQ) and k - 1 SEQ="*" records on fillers, or a record with SEQ on a filler first and the record over P as SEQ="*" (its base at P
    comes from that source, reverse-complemented when the strands differ), then k - 2 SEQ="*" records on fillers.  Every file has n
    blocks of equal size; block r holds the reads of piece (f, r) between padding reads, so that cut r of pp_sam_split_ranges falls
    between blocks (the facts hold the range of every covering record as the library cuts the files)."""
    import math
    import os
    import tempfile
    from tests import walkgen
    ms, target, side, opts, n_files, n, eight = ORDER_CASES[name]
    ks = getattr(walkgen, ms)
    rng = random.Random(seed)
    P = 522
    names = ["pad", "probe"] + ["f%d" % i for i in range(max(n, 4) - 2)]
    lengths = [PAD_LEN, 5000] + [1500 - 10 * i for i in range(len(names) - 2)]
    own = owners(lengths, n)
    o = own[1]
    on_o, off_o = piece_orders(seed, ks, target, side, n_files, n, o)
    reads = on_o if on else off_o
    seqs = {c: rand_seq(rng, L) for c, L in zip(names, lengths)}
    probe = seqs["probe"]
    y = [b for b in "ACGT" if b != probe[P]][0]
    fillers = names[2:]
    comp = {"A": "T", "C": "G", "G": "C", "T": "A"}

    def rc(s):
        return "".join(comp[c] for c in reversed(s))

    def filler_rec(q, flag, seq):
        c = rng.choice(fillers)
        a = rng.randint(0, len(seqs[c]) - 61)
        return sam(q, flag, c, a, "60M", seq if seq != "." else seqs[c][a:a + 60], 0), c

    def group(i, k):
        """The lines of covering read i, the (contig, SEQ="*") of its records and the index of its record over P."""
        q = "r%d" % i
        a = rng.randint(470, 517)
        cover = probe[a:P] + y + probe[P + 1:a + 60]
        fc = rng.choice([0, 16])
        out, recs = [], []
        if k >= 2 and rng.random() < 0.5:
            fs = rng.choice([0, 16])
            line, c = filler_rec(q, fs | 256, cover if fs == fc else rc(cover))
            out.append(line)
            recs.append((c, False))
            out.append(sam(q, fc, "probe", a, "60M", "*", 1))
            recs.append(("probe", True))
            nsec = k - 2
        else:
            out.append(sam(q, fc, "probe", a, "60M", cover, 1))
            recs.append(("probe", False))
            nsec = k - 1
        for _ in range(nsec):
            line, c = filler_rec(q, 256 | rng.choice([0, 16]), "*")
            out.append(line)
            recs.append((c, True))
        return out, recs

    pad_no = [0]

    def pad_line():
        pad_no[0] += 1
        a = rng.randint(1000, 4000)
        return sam("pad%07d" % pad_no[0], 0, "pad", a, "60M", seqs["pad"][a:a + 60], 0)

    head = ["@HD\tVN:1.6"] + ["@SQ\tSN:%s\tLN:%d" % (c, L) for c, L in zip(names, lengths)]
    plen = len(pad_line()) + 1
    texts, plan = [], []                          # plan: per covering read (file, range, line index in the file, source contig info)
    i = 0
    for f in range(n_files):
        blocks = []
        for r in range(n):
            body, meta = [], []
            for k, p in reads:
                if p != (f, r):
                    continue
                g, recs = group(i, k)
                meta.append((len(body), g, recs, k, i))
                body += g + [pad_line() for _ in range(rng.randint(0, 2))]
                i += 1
            blocks.append((body, meta))
        size = max(sum(len(x) + 1 for x in b) for b, _ in blocks) + 20 * plen + sum(len(x) + 1 for x in head)
        lines = []
        for r, (body, meta) in enumerate(blocks):
            pre = head if r == 0 else []
            fill = (size - sum(len(x) + 1 for x in pre + body)) // plen
            h = fill // 2
            base = len(lines) + len(pre) + h
            lines += pre + [pad_line() for _ in range(h)] + body + [pad_line() for _ in range(fill - h)]
            for at, g, recs, k, ri in meta:
                plan.append(dict(file=f, range=r, line=base + at, n_lines=len(g), recs=recs, k=k, read=ri))
        if eight and f == n_files - 1:                                   # the last range of the last file: an 8-bit SEQ byte
            j = len(lines) - 3
            fl = lines[j].split("\t")
            fl[9] = fl[9][:30] + "Z" + fl[9][31:]
            lines[j] = "\t".join(fl)
        texts.append("\n".join(lines) + "\n")
    # the ranges as the library cuts the files
    d = tempfile.mkdtemp(prefix="pp_rangegen_")
    try:
        ranges = []
        for f, t in enumerate(texts):
            path = os.path.join(d, "t%d.sam" % f)
            open(path, "wb").write(t.encode())
            cuts = sam_cuts(path, min(n, len(names)))
            starts = [s for s, _ in lines_of(t.encode())]
            ranges.append([range_of(cuts, s) for s in starts])
    finally:
        import shutil
        shutil.rmtree(d, ignore_errors=True)
    got = [(x["file"], ranges[x["file"]][x["line"] + j]) for x in plan for j in range(x["n_lines"])]
    cover = {x["read"]: x for x in plan}
    order = [(cover[ri]["k"], (cover[ri]["file"], ranges[cover[ri]["file"]][cover[ri]["line"]])) for ri in range(len(plan))]
    models = wrong_orders(n_files, n, o)
    star_src = []                                  # SEQ="*" records: (their contig's owner, the owner of their group's source, range)
    for x in plan:
        src = next(c for c, star in x["recs"] if not star)
        for c, star in x["recs"]:
            if star:
                star_src.append((own[names.index(c)], own[names.index(src)], ranges[x["file"]][x["line"]], c == "probe"))
    facts = dict(P=P, row=1 + PAD_LEN + P, n=n, n_files=n_files, owner=dict(zip(names, own)), probe_owner=o, target=target, side=side,
                 planned=[p for _, p in reads], pieces=[p for _, p in order], groups_whole=len(set(got)) == len(set((x["file"], x["range"]) for x in plan)),
                 group_ranges=[sorted({ranges[x["file"]][x["line"] + j] for j in range(x["n_lines"])}) for x in plan],
                 sum=seq_sum([k for k, _ in order]), models={m: seq_sum(ordered(order, key)) for m, key in models.items()},
                 star_src=star_src, seq_bits=8 if eight else 4, off_target=math.nextafter(target, side * math.inf))
    case = Case(fasta([(c, seqs[c]) for c in names]), texts, dict(opts))
    case.facts = facts
    case.blocks = ranges
    return case


def reorder(case, model):
    """The case's SAM text with its pieces in the order of wrong_orders()[model], as one file: each piece is a whole range of lines (every
    group lies inside one), so the reference's sum at P over this file is that model's sum."""
    f = case.facts
    key = wrong_orders(f["n_files"], f["n"], f["probe_owner"])[model]
    parts = {}
    head = None
    for fi, t in enumerate(case.sam_texts):
        for (s, line), r in zip(lines_of(t.encode()), case.blocks[fi]):
            if line.startswith(b"@"):
                head = (head or []) + ([line] if fi == 0 else [])
                continue
            parts.setdefault((fi, r), []).append(line)
    out = list(head or [])
    for p in sorted(parts, key=lambda p: key(*p)):
        out += parts[p]
    return b"\n".join(out) + b"\n"
