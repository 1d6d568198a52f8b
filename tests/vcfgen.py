"""The VCF of `polish --vcf`: a model of the file built from the oracle's --debug TSV, a strict applier, and cases (seeded, deterministic)
that make each kind of record.

The model follows the record rules of polypolish_b200/csrc/vcf_records.h, written out again here from the rules rather than from that
code.  out(p) is what position p puts into the FASTA: the new_base allele when its status is changed, else the draft character, with
every '-' dropped.  E = the changed positions and the draft's '-'; every maximal run [a, b] of E is one record with REF = draft[a..=b]
and ALT = out(a..=b), none when ALT == REF; an empty ALT is padded with draft[a - 1] (POS = a), at a contig start with draft[b + 1]
(POS = 1), and a run over the whole contig becomes <DEL>.  A padded run at the contig start and a next run at b + 2 with an empty
ALT become one record.

Every case is a fuzzgen.Case with `facts`: "expect", the (contig, position, status, new_base) the oracle's --debug TSV must show, and
"records" / "no_record", the (contig, POS, REF, ALT) lines the model's VCF must and must not hold.
"""
import random

from tests.fuzzgen import Case, cigar_str, merge_ops

HEADER_TAIL = (
    '##ALT=<ID=DEL,Description="Whole contig removed by polishing">\n'
    '##INFO=<ID=CHANGED,Number=1,Type=Integer,Description="Positions in the record whose polish status is changed">\n'
    '##INFO=<ID=DEPTH,Number=.,Type=Float,Description="Read depth of each changed position, as in the --debug depth column">\n'
    '##INFO=<ID=SUPPORT,Number=.,Type=Integer,Description="Pileup count of the allele each changed position took">\n'
    "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")


def read_fasta(path_or_bytes):
    """[(name, sequence)]: the first word of each header, the sequence ASCII-upper-cased (as the polish loads a draft)."""
    data = path_or_bytes if isinstance(path_or_bytes, bytes) else open(path_or_bytes, "rb").read()
    out = []
    for line in data.split(b"\n"):
        line = line.rstrip(b"\r")
        if line.startswith(b">"):
            w = line[1:].split()
            out.append([w[0].decode("latin-1") if w else "", []])
        elif out:
            out[-1][1].append(line.decode("latin-1"))
    return [(n, "".join(s).translate(_UPPER)) for n, s in out]


_UPPER = {c: c - 32 for c in range(ord("a"), ord("z") + 1)}


def changed_rows(debug_tsv):
    """{contig: {pos: (allele, depth text, support)}} of the TSV's changed rows; support = the allele's <allele>x<count> entry."""
    out = {}
    for line in debug_tsv.decode("latin-1").split("\n")[1:]:
        if not line:
            continue
        c = line.split("\t")
        if c[7] != "changed":
            continue
        counts = {}
        for e in c[6].split(",") if c[6] else []:
            a, n = e.rsplit("x", 1)
            counts[a] = int(n)
        out.setdefault(c[0], {})[int(c[1])] = (c[8], c[3], counts[c[8]])
    return out


def contig_records(name, d, ch):
    """The record lines of one contig: draft d, ch = {pos: (allele, depth text, support)} of its changed positions."""
    L = len(d)

    def alt_of(a, b):
        return "".join((ch[p][0] if p in ch else d[p]).replace("-", "") for p in range(a, b + 1))

    edited = sorted(set(ch) | {p for p, x in enumerate(d) if x == "-"})
    runs = []
    for p in edited:
        if runs and runs[-1][1] == p - 1:
            runs[-1][1] = p
        else:
            runs.append([p, p])
    lines = []
    i = 0
    while i < len(runs):
        a, b = runs[i]
        i += 1
        alt = alt_of(a, b)
        if a == 0 and alt == "" and i < len(runs) and runs[i][0] == b + 2 and alt_of(*runs[i]) == "":
            b = runs[i][1]                                  # rule 4: both runs would take draft[b + 1] as their padding
            i += 1
            alt = alt_of(a, b)
        ref = d[a:b + 1]
        if alt == ref:
            continue
        pos = a + 1
        if alt == "":
            if a > 0:
                ref, alt, pos = d[a - 1] + ref, d[a - 1], a
            elif b + 1 < L:
                ref, alt, pos = ref + d[b + 1], d[b + 1], 1
            else:
                alt, pos = "<DEL>", 1
        cp = [p for p in range(a, b + 1) if p in ch]
        info = "CHANGED=%d" % len(cp)
        if cp:
            info += ";DEPTH=" + ",".join(ch[p][1] for p in cp) + ";SUPPORT=" + ",".join(str(ch[p][2]) for p in cp)
        lines.append("%s\t%d\t.\t%s\t%s\t.\tPASS\t%s\n" % (name, pos, ref, alt, info))
    return lines


def header(contigs):
    return ("##fileformat=VCFv4.2\n##source=polypolish-b200\n" +
            "".join("##contig=<ID=%s,length=%d>\n" % (n, len(s)) for n, s in contigs) + HEADER_TAIL)


def vcf_from_debug(draft_fasta, debug_tsv):
    """The bytes `--vcf` writes for this draft, from the --debug TSV of the same polish."""
    contigs = read_fasta(draft_fasta)
    bases = {}
    for line in debug_tsv.decode("latin-1").split("\n")[1:]:
        if line:
            c = line.split("\t")
            bases.setdefault(c[0], []).append(c[2])
    for n, s in contigs:                                  # the draft as read here is the draft the polish saw
        assert "".join(bases[n]) == s, n
    ch = changed_rows(debug_tsv)
    body = "".join("".join(contig_records(n, s, ch.get(n, {}))) for n, s in contigs)
    return (header(contigs) + body).encode("latin-1")


def apply_vcf(draft_fasta, vcf):
    """[(name, edited sequence)]: the draft with the VCF's records applied.  Refuses records out of order or overlapping, a REF
    that is not the draft's, and ALT == REF."""
    contigs = read_fasta(draft_fasta)
    order = {n: i for i, (n, _) in enumerate(contigs)}
    recs = {n: [] for n, _ in contigs}
    last = (-1, 0)
    for line in vcf.decode("latin-1").split("\n"):
        if not line or line.startswith("#"):
            continue
        c = line.split("\t")
        assert len(c) == 8 and c[2] == "." and c[5] == "." and c[6] == "PASS", line
        name, pos, ref, alt = c[0], int(c[1]), c[3], c[4]
        key = (order[name], pos)
        assert key > last, "records out of order: " + line
        last = key
        assert alt != ref, "ALT == REF: " + line
        recs[name].append((pos - 1, ref, alt))
    out = []
    for n, s in contigs:
        parts, at = [], 0
        for p, ref, alt in recs[n]:
            assert p >= at, "overlapping records at %s:%d" % (n, p + 1)
            assert s[p:p + len(ref)] == ref, "REF is not the draft at %s:%d" % (n, p + 1)
            assert alt != "<DEL>" or (p == 0 and ref == s), "<DEL> is not a whole contig at %s" % n
            parts += [s[at:p], "" if alt == "<DEL>" else alt]
            at = p + len(ref)
        parts.append(s[at:])
        out.append((n, "".join(parts)))
    return out


def records_of(vcf):
    """(contig, POS, REF, ALT) of every record."""
    return [tuple(x.split("\t")[:2] + x.split("\t")[3:5]) for x in vcf.decode("latin-1").split("\n") if x and not x.startswith("#")]


def check_claims(case, debug_tsv, vcf):
    """What the case was built to make: the oracle's statuses and alleles, and the records the model writes or leaves out."""
    rows = {}
    for line in debug_tsv.decode("latin-1").split("\n")[1:]:
        if line:
            c = line.split("\t")
            rows[(c[0], int(c[1]))] = (c[7], c[8])
    for contig, pos, status, new in case.facts["expect"]:
        assert rows[(contig, pos)] == (status, new), (contig, pos, rows[(contig, pos)])
    recs = records_of(vcf)
    for r in case.facts.get("records", []):
        assert (r[0], str(r[1]), r[2], r[3]) in recs, (r, recs)
    for contig, pos in case.facts.get("no_record", []):
        assert all(not (x[0] == contig and int(x[1]) <= pos + 1 < int(x[1]) + len(x[2])) for x in recs), (contig, pos, recs)


# ---- cases -----------------------------------------------------------------------------------------------------------------
W = 40                 # draft positions per read
PAST = "AC"            # bases past a contig's end (the reference ignores them; the read's last counted entry is then the last base)


def _reads(name, d, out, rng, qn, dot=None):
    """SAM lines tiling contig `name` (draft d) with reads that carry out[p] at every position: "" a D, a longer string a match
    then inserted bases.  Ten reads start at the contig start, ten reach past its end, and one starts every 4 positions between,
    so every position is covered about ten times.  dot = a position whose base one extra read carries as '.'."""
    L = len(d)
    lines = []
    starts = [0] * 10 + list(range(4, L, 4)) + [max(0, L - W)] * 10
    for s in starts:
        if out[s] == "":
            continue
        e = min(L, s + W)
        while e < L and len(out[e - 1]) != 1:
            e -= 1
        ops, seq, nm = [], "", 0
        for p in range(s, e):
            if out[p] == "":
                ops.append(("D", 1))
                nm += 1
            else:
                ops += [("M", 1), ("I", len(out[p]) - 1)]
                seq += out[p]
                nm += (out[p][0] != d[p]) + len(out[p]) - 1
        if e == L:
            ops.append(("M", len(PAST)))
            seq += PAST
        qn[0] += 1
        lines.append("\t".join(["v%d" % qn[0], str(rng.choice([0, 16])), name, str(s + 1), "60", cigar_str(merge_ops(ops)), "*", "0", "0",
                                seq, "*", "NM:i:%d" % nm]))
    if dot is not None:                                    # a plain read with one '.' in it: the 8-bit pool
        s = dot - 5
        seq = d[s:dot] + "." + d[dot + 1:s + W]
        qn[0] += 1
        lines.append("\t".join(["v%d" % qn[0], "0", name, str(s + 1), "60", "%dM" % W, "*", "0", "0", seq, "*", "NM:i:1"]))
    return lines


def _case(seed, contigs, expect, records=(), no_record=(), eight_bit=False, opts=None):
    """contigs: [(name, draft, {pos: what the reads carry there})]; every other position carries the draft base (a draft '-' a D)."""
    rng = random.Random(seed)
    qn = [0]
    fa, sam = [], ["@HD\tVN:1.6\tSO:unsorted"]
    for name, d, edits in contigs:
        fa.append(">%s\n%s\n" % (name, d))
        sam.append("@SQ\tSN:%s\tLN:%d" % (name, len(d)))
    body = []
    for i, (name, d, edits) in enumerate(contigs):
        out = [edits.get(p, "" if x == "-" else x) for p, x in enumerate(d)]
        dot = None
        if eight_bit and i == 0:
            dot = next(p for p in range(20, len(d) - W) if all(q not in edits and d[q] != "-" for q in range(p - 8, p + W)))
        body += _reads(name, d, out, rng, qn, dot)
    rng.shuffle(body)
    c = Case("".join(fa), ["\n".join(sam + body) + "\n"], dict(opts or {}))
    c.facts = dict(expect=list(expect), records=list(records), no_record=list(no_record), eight_bit=eight_bit)
    return c


def _draft(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def _other(rng, b):
    return rng.choice([x for x in "ACGT" if x != b])


def substitutions(seed=1, eight_bit=False):
    """Three adjacent substitutions (one record of three bases) and a lone one."""
    rng = random.Random(seed)
    d = _draft(rng, 240)
    new = {p: _other(rng, d[p]) for p in (60, 61, 62, 150)}
    return _case(seed, [("subs", d, new)], [("subs", p, "changed", b) for p, b in new.items()],
                 records=[("subs", 61, d[60:63], new[60] + new[61] + new[62]), ("subs", 151, d[150], new[150])], eight_bit=eight_bit)


def insertion(seed=2, eight_bit=False):
    """A -> AT (one base after the draft base) and a three-base insertion."""
    rng = random.Random(seed)
    d = _draft(rng, 240)
    new = {70: d[70] + "T", 160: d[160] + "GCA"}
    return _case(seed, [("ins", d, new)], [("ins", p, "changed", a) for p, a in new.items()],
                 records=[("ins", 71, d[70], d[70] + "T"), ("ins", 161, d[160], d[160] + "GCA")], eight_bit=eight_bit)


def deletions(seed=3):
    """Deletions at position 0 and at the last position (reads carry '-' there, so the pool is 8-bit), one in the middle (a D) and
    a two-base one."""
    rng = random.Random(seed)
    d = _draft(rng, 240)
    L = len(d)
    new = {0: "-", 100: "", 170: "", 171: "", L - 1: "-"}
    return _case(seed, [("del", d, new)], [("del", p, "changed", "-") for p in new],
                 records=[("del", 1, d[0:2], d[1]), ("del", 100, d[99:101], d[99]), ("del", 170, d[169:172], d[169]),
                          ("del", L - 1, d[L - 2:], d[L - 2])], eight_bit=True)


def start_merge(seed=4):
    """Rule 4: deletions at 0 and 2 would both take draft[1] as padding, so they are one record (POS 1, REF draft[0..=2])."""
    rng = random.Random(seed)
    d = _draft(rng, 200)
    new = {0: "-", 2: "-"}
    return _case(seed, [("merge", d, new)], [("merge", 0, "changed", "-"), ("merge", 1, "kept", d[1]), ("merge", 2, "changed", "-")],
                 records=[("merge", 1, d[0:3], d[1])], eight_bit=True)


def no_op(seed=5, eight_bit=False):
    """Rule 2: A -> AC followed by C -> - gives the draft back: both positions are changed and there is no record."""
    rng = random.Random(seed)
    d = list(_draft(rng, 220))
    d[90], d[91], d[92] = "A", "C", "G"
    d = "".join(d)
    new = {90: "AC", 91: ""}
    return _case(seed, [("noop", d, new)], [("noop", 90, "changed", "AC"), ("noop", 91, "changed", "-")],
                 no_record=[("noop", 90), ("noop", 91)], eight_bit=eight_bit)


def dashes(seed=6):
    """Draft '-' characters: kept (one alone, two in a row), changed to a base, kept next to a substitution."""
    rng = random.Random(seed)
    d = list(_draft(rng, 260))
    for p in (40, 120, 121, 170, 200):
        d[p] = "-"
    d = "".join(d)
    sub = _other(rng, d[201])
    new = {170: "G", 201: sub}
    return _case(seed, [("dash", d, new)],
                 [("dash", 40, "kept", "-"), ("dash", 120, "kept", "-"), ("dash", 121, "kept", "-"), ("dash", 170, "changed", "G"),
                  ("dash", 200, "kept", "-"), ("dash", 201, "changed", sub)],
                 records=[("dash", 40, d[39:41], d[39]), ("dash", 120, d[119:122], d[119]), ("dash", 171, "-", "G"),
                          ("dash", 201, "-" + d[201], sub)])


def whole_contig(seed=7):
    """Rule 3: a contig made entirely of '-' (no reads), and a three-base contig every position of which becomes '-': both <DEL>."""
    rng = random.Random(seed)
    d = _draft(rng, 200)
    gone = _draft(rng, 3)
    sub = _other(rng, d[100])
    return _case(seed, [("keep", d, {100: sub}), ("dashes", "-----", {}), ("gone", gone, {0: "-", 1: "-", 2: "-"})],
                 [("keep", 100, "changed", sub), ("dashes", 0, "low_depth", "-"), ("gone", 0, "changed", "-"), ("gone", 2, "changed", "-")],
                 records=[("dashes", 1, "-----", "<DEL>"), ("gone", 1, gone, "<DEL>")], eight_bit=True)


def iupac(seed=8, eight_bit=False):
    """An IUPAC draft: N and R changed to bases, Y kept (the reads carry Y), and A changed to N (an allele of the pool)."""
    rng = random.Random(seed)
    d = list(_draft(rng, 240))
    d[50], d[120], d[121], d[180] = "N", "R", "Y", "A"
    d = "".join(d)
    new = {50: "A", 120: "G", 121: "Y", 180: "N"}
    return _case(seed, [("iupac", d, new)],
                 [("iupac", 50, "changed", "A"), ("iupac", 120, "changed", "G"), ("iupac", 121, "kept", "Y"), ("iupac", 180, "changed", "N")],
                 records=[("iupac", 51, "N", "A"), ("iupac", 121, "R", "G"), ("iupac", 181, "A", "N")], eight_bit=eight_bit)


CASES = {
    "substitutions": substitutions,
    "insertion": insertion,
    "deletions": deletions,
    "start-merge": start_merge,
    "no-op": no_op,
    "dashes": dashes,
    "whole-contig": whole_contig,
    "iupac": iupac,
    "substitutions-8bit": lambda: substitutions(eight_bit=True),
    "insertion-8bit": lambda: insertion(eight_bit=True),
    "no-op-8bit": lambda: no_op(eight_bit=True),
    "iupac-8bit": lambda: iupac(eight_bit=True),
}
