"""Status-boundary cases for `polish --status-bed` (seeded, deterministic), and the run-length encoding that defines the BED.

Where a position is covered by reads that map to several places (k != 1), the reference's depth is the sequential f64 sum of 1/k in
SAM order, and k_tile only knows a bound [lo, hi] around it unless it runs the ordered depth walk (polypolish_b200/csrc/polish_dev.cuh,
depth_bounds).  Each case here puts a probe position P on a status boundary: its covering reads come in a SAM order whose sum is
exactly the boundary ("on") or one ulp below it ("off") (walkgen.run_orders, over the runs of walkgen's layouts).  The boundaries:

  too_close  round(depth * fraction_invalid) against the count of a non-draft allele far below the valid threshold: at depth 7,
             fraction_invalid 0.5, three reads carry Y: the invalid threshold is 4 on the boundary (Y invalid: kept) and 3 below it
             (Y intermediate: too_close);
  min_depth  depth == min_depth with every read carrying the draft base: kept on it, low_depth below it;
  multiple   the valid threshold with two alleles in reach: at depth 7, fraction_valid 0.5, three reads carry Y: the valid threshold
             is 4 on the boundary (Y intermediate: too_close) and 3 below it (Y valid next to the draft base: multiple).

P keeps its draft base in both orders of every case.  In the too_close and min_depth cases the vote's shortcuts decide that base
without depth (no allele other than the draft's comes near the valid threshold), so a kernel that walks only where the base is in
doubt never walks there; and the bound's lower end, which the vote then reads, gives the "off" thresholds (facts th_lo == th_off !=
th_on).  Only the status mode's walk rule - walk where the thresholds at lo and hi differ - gets the "on" status right.  In the
multiple cases a non-draft allele is within rounding of the valid threshold, so the walk opens under the older rule as well.
"""
import math
from fractions import Fraction

from tests import walkgen
from tests.walkgen import bankers, crosses, run_orders

STATUS = [b"low_depth", b"none", b"multiple", b"too_close", b"kept", b"changed"]


def bed_from_debug_tsv(tsv):
    """The run-length encoding, per contig, of the status column of a --debug TSV: what --status-bed writes."""
    out = []
    run = None                                            # [name, start, end, status]
    for line in tsv.split(b"\n")[1:]:
        if not line:
            continue
        c = line.split(b"\t")
        name, pos, st = c[0], int(c[1]), c[7]
        if run and run[0] == name and run[3] == st and run[2] == pos:
            run[2] = pos + 1
            continue
        if run:
            out.append(run)
        run = [name, pos, pos + 1, st]
    if run:
        out.append(run)
    return b"".join(b"%s\t%d\t%d\t%s\n" % (n, s, e, st) for n, s, e, st in out)


def status_at(debug_tsv, contig, pos):
    for line in debug_tsv.split(b"\n")[1:]:
        c = line.split(b"\t")
        if c[0] == contig.encode() and int(c[1]) == pos:
            return c[7]
    raise KeyError((contig, pos))


def thresholds(depth, opts):
    """vote_thresholds: (valid threshold, invalid threshold, low depth) at this depth."""
    md = opts.get("min_depth", 5)
    return (max(md, bankers(depth * opts.get("fraction_valid", 0.5))), bankers(depth * opts.get("fraction_invalid", 0.2)), depth < md)


def lower_bound(ks):
    """The lower end of depth_bounds for alignments with these k over one position (exact arithmetic, then rounded down)."""
    n = len(ks)
    M = sum((1 << 40) - ((1 << 40) + k // 2) // k for k in ks if k != 1)
    lo = n - Fraction(M, 1 << 40) - Fraction(n, 1 << 41) - Fraction(n * n, 1 << 52)
    x = float(lo)
    return x if Fraction(x) <= lo else math.nextafter(x, -math.inf)


K35_HALF = [1] * 6 + [35] * 35             # 7.0
K34_MIN = [1] * 4 + [34] * 34              # 5.0
WIDE18 = walkgen.WIDE18                    # 18.0
MIX20 = walkgen.MIX20                      # 20.0
TOO_CLOSE = dict(min_depth=1, fraction_valid=0.9, fraction_invalid=0.5)
MULTIPLE = dict(min_depth=1, fraction_valid=0.5, fraction_invalid=0.2)

# name: (layout, multiset, target, options, reads carrying Y, min reads per run, status on, status off, the shortcut decides P)
CASES = {
    "close-two": ("two", K35_HALF, 7.0, TOO_CLOSE, 3, 6, b"kept", b"too_close", True),
    "close-three": ("three", K35_HALF, 7.0, TOO_CLOSE, 3, 6, b"kept", b"too_close", True),
    "close-long": ("long", K35_HALF, 7.0, TOO_CLOSE, 3, 6, b"kept", b"too_close", True),
    "close-three-8bit": ("three", K35_HALF, 7.0, TOO_CLOSE, 3, 6, b"kept", b"too_close", True),
    "depth-two": ("two", WIDE18, 18.0, dict(min_depth=18), 0, 40, b"kept", b"low_depth", True),
    "depth-three": ("three", K34_MIN, 5.0, dict(min_depth=5), 0, 6, b"kept", b"low_depth", True),
    "depth-long": ("long", MIX20, 20.0, dict(min_depth=20), 0, 8, b"kept", b"low_depth", True),
    "depth-long-8bit": ("long", MIX20, 20.0, dict(min_depth=20), 0, 8, b"kept", b"low_depth", True),
    "multiple-two": ("two", K35_HALF, 7.0, MULTIPLE, 3, 6, b"too_close", b"multiple", False),
    "multiple-three": ("three", K35_HALF, 7.0, MULTIPLE, 3, 6, b"too_close", b"multiple", False),
}


def _with_alleles(case, n_y):
    """The covering reads of a walkgen case carry Y at P; all but the first n_y are given the draft base there instead."""
    fa = case.fasta_text.split("\n")
    probe = fa[fa.index(">probe") + 1]
    P = case.facts["probe_local"]
    lines = case.sam_texts[0].split("\n")
    for j, line in enumerate(lines):
        c = line.split("\t")
        if len(c) < 10 or c[2] != "probe" or not c[0].startswith("r") or int(c[1]) & 256:
            continue
        if int(c[0][1:]) >= n_y:
            s = int(c[3]) - 1
            c[9] = c[9][:P - s] + probe[P] + c[9][P - s + 1:]
            lines[j] = "\t".join(c)
    case.sam_texts = ["\n".join(lines)]
    return case


def case_pair(name, seed=5):
    """The on and off cases of CASES[name] (fuzzgen.Case objects with .facts) and the spec."""
    lay, ks, target, opts, n_y, per_run, st_on, st_off, shortcut = CASES[name]
    layout = walkgen.LAYOUTS[lay]()
    on, off = run_orders(seed, ks, target, len(layout["runs"]), side=-1, min_per_run=per_run)
    eight = "8bit" in name
    pair = []
    for order in (on, off):                               # (the same seed: the same assembly)
        c = _with_alleles(walkgen.walk_case(seed, order, layout, opts=opts, eight_bit=eight), n_y)
        kk = [k for k, _ in order]
        c.facts.update(ks=kk, th_lo=thresholds(lower_bound(kk), opts), n_y=n_y)
        pair.append(c)
    off_sum = math.nextafter(target, -math.inf)
    spec = dict(target=target, P=pair[0].facts["probe_local"], st_on=st_on, st_off=st_off, shortcut=shortcut, eight_bit=eight,
                th_on=thresholds(target, opts), th_off=thresholds(off_sum, opts), labels=layout["labels"])
    assert pair[0].facts["sum"] == target and crosses(target, pair[1].facts["sum"], 1)
    return pair[0], pair[1], spec
