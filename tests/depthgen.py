"""Printed-depth cases for `polish --depth-bedgraph` (seeded, deterministic), and the run-length encoding that defines the bedGraph.

The --debug depth column is "%.1f" of the reference's sequential f64 sum of 1/k in SAM order, and k_tile only knows a bound [lo, hi]
around that sum unless it runs the ordered depth walk (polypolish_b200/csrc/polish_dev.cuh, depth_bounds).  Each case puts a probe
position P next to a print boundary (a decimal tie x.x5): its covering reads come in one SAM order whose f64 sum prints one tenth
("on") and in another whose sum prints the tenth below it ("off"), for the same multiset of k (walkgen.run_orders over the runs of
walkgen's layouts, the "on" order spread over the runs so that a merge which empties one run before the next prints "off" too).

Every covering read carries the draft base at P, so P keeps its base in both orders and the vote's shortcuts decide it without
depth: only the depth mode's walk rule (walk where lo and hi print differently) opens the walk there.  The lower end of the bound
prints the "off" tenth (facts tenths_lo), so a kernel that keyed P on lo would write the wrong line for the "on" order.

  m235  {5 x6, 10 x7, 20 x11}, 2.45: f64 2.45 prints 2.5, one ulp below prints 2.4;
  m100  {1 x100, 5 x2, 10 x3, 20 x5}, 100.95: integer depth from k = 1 reads under the fraction (101.0 against 100.9).

The dyadic cases have exact ties that no order changes: depth x.75 (k = 4 reads and k = 1 reads) prints x.8 by round-half-even while
lo prints x.7 ("on"); x.25 prints x.2 ("off", the even tenth, which is also what lo prints).
"""
import math
from fractions import Fraction

from tests import statusgen, walkgen
from tests.walkgen import run_orders

M235 = [5] * 6 + [10] * 7 + [20] * 11
M100 = [1] * 100 + [5] * 2 + [10] * 3 + [20] * 5
OPTS = dict(min_depth=1)


def bedgraph_from_debug_tsv(tsv):
    """The run-length encoding, per contig, of the depth column of a --debug TSV: what --depth-bedgraph writes."""
    out = []
    run = None                                            # [name, start, end, depth text]
    for line in tsv.split(b"\n")[1:]:
        if not line:
            continue
        c = line.split(b"\t")
        name, pos, dp = c[0], int(c[1]), c[3]
        if run and run[0] == name and run[3] == dp and run[2] == pos:
            run[2] = pos + 1
            continue
        if run:
            out.append(run)
        run = [name, pos, pos + 1, dp]
    if run:
        out.append(run)
    return b"".join(b"%s\t%d\t%d\t%s\n" % (n, s, e, d) for n, s, e, d in out)


def bedgraph_from_runs(names, off, runs):
    """The bedGraph of Context.depth_runs() (global positions) over contigs `names` with offsets `off`."""
    out = []
    for s, e, t in zip(runs["start"].tolist(), runs["end"].tolist(), runs["tenths"].tolist()):
        c = max(i for i in range(len(names)) if off[i] <= s)
        out.append(b"%s\t%d\t%d\t%d.%d\n" % (names[c].encode(), s - off[c], e - off[c], t // 10, t % 10))
    return b"".join(out)


def depth_at(debug_tsv, contig, pos):
    for line in debug_tsv.split(b"\n")[1:]:
        c = line.split(b"\t")
        if c[0] == contig.encode() and int(c[1]) == pos:
            return c[3]
    raise KeyError((contig, pos))


def tenths(x):
    """What "%.1f" prints for x, times ten (the exact binary value, ties to even): depth_tenths' model."""
    q = Fraction(x) * 10
    f = math.floor(q)
    r = q - f
    return f + 1 if r > Fraction(1, 2) or (r == Fraction(1, 2) and f % 2) else f


# name: (layout, multiset, target, min reads per run); "-8bit": the 8-bit pool twin
CASES = {
    "m235-two": ("two", M235, 2.45, 3),
    "m235-three": ("three", M235, 2.45, 3),
    "m235-long": ("long", M235, 2.45, 3),
    "m235-tile-start": ("border_at", M235, 2.45, 3),
    "m235-tile-end": ("border_before", M235, 2.45, 3),
    "m235-contig-border": ("contig_border", M235, 2.45, 1),
    "m235-three-8bit": ("three", M235, 2.45, 3),
    "m100-two": ("two", M100, 100.95, 3),
    "m100-three": ("three", M100, 100.95, 3),
    "m100-long": ("long", M100, 100.95, 3),
    "m100-two-8bit": ("two", M100, 100.95, 3),
}
# name: (layout, k multiset of "on", of "off")
DYADIC = {
    "tie-two": ("two", [4] * 3 + [1] * 5, [4] + [1] * 5),
    "tie-three": ("three", [4] * 7 + [1] * 2, [4] * 5 + [1] * 2),
}


def _case(seed, order, lay, eight):
    c = statusgen._with_alleles(walkgen.walk_case(seed, order, walkgen.LAYOUTS[lay](), opts=OPTS, eight_bit=eight), 0)
    ks = [k for k, _ in order]
    c.facts.update(ks=ks, tenths_lo=tenths(statusgen.lower_bound(ks)), tenths_ref=tenths(c.facts["sum"]))
    return c


def case_pair(name, seed=5):
    """The on and off cases of CASES[name] or DYADIC[name] (fuzzgen.Case objects with .facts) and the spec: P (in the probe contig)
    and the depth text each order prints there."""
    eight = "8bit" in name
    if name in DYADIC:
        lay, ks_on, ks_off = DYADIC[name]
        n_runs = len(walkgen.LAYOUTS[lay]()["runs"])
        on, off = ([(k, i % n_runs) for i, k in enumerate(ks)] for ks in (ks_on, ks_off))
    else:
        lay, ks, target, per_run = CASES[name]
        on, off = run_orders(seed, ks, target, len(walkgen.LAYOUTS[lay]()["runs"]), side=-1, min_per_run=per_run)
    pair = [_case(seed, order, lay, eight) for order in (on, off)]
    text = [b"%d.%d" % divmod(c.facts["tenths_ref"], 10) for c in pair]
    spec = dict(P=pair[0].facts["probe_local"], on=text[0], off=text[1], eight_bit=eight)
    assert text[0] != text[1] and pair[0].facts["tenths_lo"] != pair[0].facts["tenths_ref"]
    assert name in DYADIC or pair[0].facts["tenths_lo"] == pair[1].facts["tenths_ref"]
    return pair[0], pair[1], spec
