"""pyport.py — a second, independent CPU restatement of the reference's hot path, in plain Python.

TEST INFRASTRUCTURE ONLY (imported by tests/test_golden.py and tests/test_pyport.py): it exists so that the golden
fixtures and the C++ oracle are pinned by TWO separate readings of the Rust source instead of one.  It was written from
reference src/*.rs directly (not from oracle/polypolish_oracle.cpp) and follows the reference's own structure:
strings, a dict per position, sequential float depth.  Pure-Python loops: small inputs only.

  alignment.rs:49-98    Alignment.new            alignment.rs:102-128  Alignment.new_quick
  alignment.rs:138-149  get_ref_end              alignment.rs:175-201  get_read_bases_for_each_target_base
  alignment.rs:225-272  add_to_pileup            alignment.rs:275-305  process_one_read
  alignment.rs:325-346  get_expanded_cigar       alignment.rs:364-378  trim_bases_for_homopolymers
  pileup.rs:56-134      add_seq, get_polished_seq   pileup.rs:137-166  debug line
  polish.rs:157-203     polish_one_sequence, print_seq_to_stdout
  filter.rs:110-259, 296-377   filter
  misc.rs:102-133 load_fasta, :170-191 reverse_complement, :208-215 bankers_rounding
"""
import gzip
import math
import re

CIGAR_RE = re.compile(r"\d+[MIDNSHP=X]")            # alignment.rs:27-29


class RefError(Exception):
    """quit_with_error (misc.rs:29-33)"""


def lines_of(path):
    """BufReader::lines(): split on \\n, drop one trailing \\r; a final empty piece is not a line."""
    data = open(path, "rb").read().decode("latin-1")
    parts = data.split("\n")
    if parts and parts[-1] == "":
        parts.pop()
    return [p[:-1] if p.endswith("\r") else p for p in parts]


def parse_uint(s, bits):
    """Rust str::parse::<u32 / usize>(): optional '+', ASCII digits, overflow is an error (the reference unwraps -> panic)."""
    if not re.fullmatch(r"\+?[0-9]+", s) or int(s) >= (1 << bits):
        raise RefError("panic: invalid integer %r" % s)
    return int(s)


def bankers_rounding(x):                              # misc.rs:208-215
    rounded_down = min(int(x), 0xFFFFFFFF) if x > 0 else 0
    f = x - math.trunc(x)
    if f < 0.5:
        return rounded_down
    if f > 0.5:
        return rounded_down + 1
    return rounded_down + (rounded_down & 1)


COMP = {"A": "T", "T": "A", "G": "C", "C": "G", "a": "t", "t": "a", "g": "c", "c": "g", "N": "N", "n": "n", "R": "Y", "Y": "R", "S": "S",
        "W": "W", "K": "M", "M": "K", "B": "V", "V": "B", "D": "H", "H": "D", "r": "y", "y": "r", "s": "s", "w": "w", "k": "m", "m": "k",
        "b": "v", "v": "b", "d": "h", "h": "d", ".": ".", "-": "-", "?": "?"}


def reverse_complement(seq):                          # misc.rs:170-191
    return "".join(COMP.get(c, "N") for c in reversed(seq))


def load_fasta(path):                                 # misc.rs:38-133 (+ gzip by magic bytes :81-99)
    raw = open(path, "rb").read()
    if raw[:2] == b"\x1f\x8b":
        raw = gzip.decompress(raw)
    parts = raw.decode("latin-1").split("\n")
    if parts and parts[-1] == "":
        parts.pop()
    seqs, name, desc, seq = [], "", "", []
    for text in parts:
        if text.endswith("\r"):
            text = text[:-1]
        if len(text) == 0:
            continue
        if text.startswith(">"):
            if name:
                seqs.append((name, desc, "".join(seq).upper()))
                seq = []
            m = re.match(r"(\S*)(?:\s(.*))?$", text[1:], re.S)      # splitn(2, char::is_whitespace)
            name, desc = m.group(1), m.group(2) or ""
        else:
            if not name:
                raise RefError("%r is not correctly formatted" % path)
            seq.append(text)
    if name:
        seqs.append((name, desc, "".join(seq).upper()))
    return seqs


def get_expanded_cigar(cigar):                        # alignment.rs:325-346
    if cigar == "*":
        return ""
    out, total = [], 0
    for m in CIGAR_RE.finditer(cigar):
        out.append(m.group()[-1] * parse_uint(m.group()[:-1], 32))
        total += len(m.group())
    if total != len(cigar):
        raise ValueError("invalid CIGAR")
    return "".join(out)


class Alignment:
    def __init__(self, line, quick=False):            # alignment.rs:49-128
        parts = line.split("\t")
        if len(parts) < 11:
            raise ValueError("too few columns")
        self.read_name = parts[0]
        self.sam_flags = parse_uint(parts[1], 32)
        self.ref_name = parts[2]
        pos = parse_uint(parts[3], 64)
        self.ref_start = pos - 1 if pos > 0 else 0
        self.cigar = parts[5]
        self.mismatches, self.pass_qc, self.expanded_cigar, self.read_seq = 0, True, "", ""
        if quick:
            return
        mismatches = None
        for p in parts[11:]:
            if p.startswith("NM:i:"):
                mismatches = parse_uint(p[5:], 32)
            if p.lower() == "zp:z:fail":
                self.pass_qc = False
        if mismatches is None and self.sam_flags & 4 == 0:
            raise ValueError("missing NM tag")
        self.mismatches = mismatches
        try:
            self.expanded_cigar = get_expanded_cigar(self.cigar)
        except ValueError:
            raise RefError('encountered an invalid CIGAR string for read %s: "%s"' % (self.read_name, self.cigar))
        self.read_seq = "".join(c.upper() if "a" <= c <= "z" else c for c in parts[9])

    def is_aligned(self):
        return self.sam_flags & 4 == 0

    def forward(self):
        return self.sam_flags & 16 == 0

    def get_ref_end(self):                            # alignment.rs:138-149
        end = self.ref_start
        for m in CIGAR_RE.finditer(self.cigar):
            if m.group()[-1] in "MDN=X":
                end += int(m.group()[:-1])
        return end

    def read_bases_for_each_target_base(self):        # alignment.rs:175-201
        i, rb = 0, []
        for c in self.expanded_cigar:
            if c in "M=X":
                rb.append([i, i + 1])
                i += 1
            elif c == "I":
                rb[-1][1] = i + 1
                i += 1
            elif c == "D":
                rb.append([i, i])
            else:
                raise RefError('unexpected character (other than M, =, X, I or D) in CIGAR string for read %s: "%s" - did you use BWA MEM '
                               'to generate your alignments?' % (self.read_name, self.cigar))
        if i != len(self.read_seq):
            raise RefError("CIGAR string for read %s does not match read sequence" % self.read_name)
        # trim_bases_for_homopolymers, alignment.rs:364-378
        last = self.read_seq[rb[-1][0]:rb[-1][1]]
        while rb and self.read_seq[rb[-1][0]:rb[-1][1]] == last:
            rb.pop()
        if rb:
            rb.pop()
        return rb


class PileupBase:
    def __init__(self, original):
        self.original, self.depth, self.counts = original, 0.0, {}

    def add_seq(self, seq, contribution):             # pileup.rs:56-65 (A/C/G/T integer counters folded into the dict)
        self.counts[seq] = self.counts.get(seq, 0) + 1
        self.depth += contribution

    def polished(self, min_depth, fv, fi):            # pileup.rs:67-134
        valid_threshold = max(min_depth, bankers_rounding(self.depth * fv))
        invalid_threshold = bankers_rounding(self.depth * fi)
        valid, inter = [], []
        present = dict(self.counts)
        for b in "ACGT":                               # the four dedicated counters take part even at zero
            present.setdefault(b, 0)
        for seq, count in present.items():
            if count >= valid_threshold:
                valid.append(seq)
            elif count >= invalid_threshold:
                inter.append(seq)
        new_base, status = self.original, "kept"
        if self.depth < float(min_depth):
            status = "low_depth"
        elif len(valid) == 1:
            if inter:
                status = "too_close"
            else:
                new_base = valid[0]
                if new_base != self.original:
                    status = "changed"
        elif len(valid) == 0:
            status = "none"
        else:
            status = "multiple"
        return new_base, status, valid_threshold, invalid_threshold

    def debug_line(self, min_depth, fv, fi):          # pileup.rs:137-166
        new_base, status, vt, it = self.polished(min_depth, fv, fi)
        counts = sorted("%sx%d" % (s, c) for s, c in self.counts.items() if c > 0)
        return "%s\t%.1f\t%d\t%d\t%s\t%s\t%s" % (self.original, self.depth, it, vt, ",".join(counts), status, new_base)


def process_one_read(alignments, pileups, max_errors, careful):   # alignment.rs:275-305
    if careful and len(alignments) > 1:
        return 0
    src = next((a for a in alignments if a.read_seq != "*"), None)
    if src is None:
        raise RefError("no alignments for read %s contain sequence" % alignments[0].read_name)
    read_seq, strand = src.read_seq, src.forward()
    good = [a for a in alignments
            if a.expanded_cigar[0] in "M=" and a.expanded_cigar[-1] in "M=" and a.mismatches <= max_errors and a.pass_qc]
    for a in good:
        if a.read_seq == "*":
            a.read_seq = read_seq if a.forward() == strand else reverse_complement(read_seq)
    for a in good:
        contribution = 1.0 / float(len(good))
        if a.ref_name not in pileups:
            raise RefError("query name %s in SAM but not in assembly" % a.ref_name)
        bases = pileups[a.ref_name]
        i = a.ref_start
        for start, end in a.read_bases_for_each_target_base():   # pileup.rs:189-200
            if i >= len(bases):
                raise RefError("panic: index out of bounds")
            bases[i].add_seq("-" if start == end else a.read_seq[start:end], contribution)
            i += 1
    return len(good)


def polish(assembly, sams, fraction_invalid=0.2, fraction_valid=0.5, max_errors=10, min_depth=5, careful=False, debug=False):
    """polish::polish (polish.rs:26-38): returns dict(fasta=bytes, debug_tsv=bytes|None, changed=[..], zero_depth=[..], used_total=int)."""
    seqs = load_fasta(assembly)
    pileups = {name: [PileupBase(b) for b in seq] for name, _, seq in seqs}
    used_total = 0
    for sam in sams:                                   # alignment.rs:225-272
        current_name, current, count = "", [], 0
        for n, line in enumerate(lines_of(sam), 1):
            if len(line) == 0 or line.startswith("@"):
                continue
            try:
                a = Alignment(line)
            except ValueError as e:
                raise RefError('%s in "%s" (line %d)' % (e, sam, n))
            if not a.is_aligned():
                continue
            count += 1
            if current_name == "" or current_name == a.read_name:
                current.append(a)
            else:
                used_total += process_one_read(current, pileups, max_errors, careful)
                current = [a]
            current_name = a.read_name
        if count == 0:
            raise RefError('no alignments in "%s"' % sam)     # (the reference panics one line earlier; same exit path)
        used_total += process_one_read(current, pileups, max_errors, careful)
    out, dbg, changed, zero = [], ["name\tpos\tbase\tdepth\tinvalid\tvalid\tpileup\tstatus\tnew_base"], [], []
    for name, desc, _ in seqs:                         # polish.rs:157-203
        bases = pileups[name]
        pieces, n_changed, n_zero = [], 0, 0
        for pos, b in enumerate(bases):
            new_base, status, _, _ = b.polished(min_depth, fraction_valid, fraction_invalid)
            n_changed += status == "changed"
            n_zero += b.depth == 0.0
            if debug:
                dbg.append("%s\t%d\t%s" % (name, pos, b.debug_line(min_depth, fraction_valid, fraction_invalid)))
            pieces.append(new_base)
        seq = "".join(pieces).replace("-", "")
        out.append(">%s%s polypolish\n%s\n" % (name, (" " + desc) if desc else "", seq))
        changed.append(n_changed)
        zero.append(n_zero)
    return dict(fasta="".join(out).encode("latin-1"), debug_tsv=("\n".join(dbg) + "\n").encode("latin-1") if debug else None,
                changed=changed, zero_depth=zero, used_total=used_total)


# ---- filter (filter.rs) ---------------------------------------------------------------------------------------------
def get_orientation(a1, a2):                           # filter.rs:189-209
    s1, s2 = ("f" if a1.forward() else "r"), ("f" if a2.forward() else "r")
    p1 = a1.ref_start if a1.forward() else a1.get_ref_end()
    p2 = a2.ref_start if a2.forward() else a2.get_ref_end()
    if s1 != s2:
        return s1 + s2 if p1 < p2 else s2 + s1
    if s1 == "f":
        return "ff" if p1 < p2 else "rr"
    return "ff" if p2 < p1 else "rr"


def get_insert_size(a1, a2):                           # filter.rs:212-218
    pos = [a1.ref_start, a1.get_ref_end(), a2.ref_start, a2.get_ref_end()]
    return max(pos) - min(pos)


def get_percentile(sorted_list, percentile):           # filter.rs:249-259
    if not sorted_list:
        return 0
    rank = max(int(math.ceil(percentile / 100.0 * float(len(sorted_list)))), 1)
    return sorted_list[rank - 1] if rank - 1 < len(sorted_list) else 0


def filter_sams(in1, in2, orientation="auto", low=0.1, high=99.9):
    """filter::filter (filter.rs:26-37): returns dict(out1=bytes, out2=bytes, low, high, orientation)."""
    alignments = {}
    for path, suffix in ((in1, "_1"), (in2, "_2")):    # filter.rs:110-145
        for n, line in enumerate(lines_of(path), 1):
            if line.startswith("@"):
                continue
            try:
                a = Alignment(line, quick=True)
            except ValueError as e:
                raise RefError('%s in "%s" (line %d)' % (e, path, n))
            if a.is_aligned():
                alignments.setdefault(a.read_name + suffix, []).append(a)
        if not alignments:
            raise RefError('no alignments found in "%s"' % path)
    sizes = {}                                         # filter.rs:148-186
    for name1, al1 in alignments.items():
        if not name1.endswith("_1") or len(al1) != 1:
            continue
        al2 = alignments.get(name1[:-2] + "_2")
        if al2 is not None and len(al2) == 1 and al1[0].ref_name == al2[0].ref_name:
            sizes.setdefault(get_orientation(al1[0], al2[0]), []).append(get_insert_size(al1[0], al2[0]))
    if not sizes:
        raise RefError("no one-alignment-per-read pairs available to determine orientation and insert size thresholds")
    if orientation == "auto":                          # filter.rs:238-246
        mx = max(len(v) for v in sizes.values())
        best = [o for o in ("fr", "rf", "ff", "rr") if len(sizes.get(o, [])) == mx]
        if len(best) != 1:
            raise RefError("could not automatically determine read pair orientation")
        orientation = best[0]
    chosen = sorted(sizes.get(orientation, []))
    if not chosen:
        raise RefError("no read pairs available to determine insert size thresholds")
    lo, hi = get_percentile(chosen, low), get_percentile(chosen, high)
    outs = []
    for path, num in ((in1, 1), (in2, 2)):             # filter.rs:296-349
        out = []
        for line in lines_of(path):
            if line.startswith("@"):
                out.append(line)
                continue
            a = Alignment(line, quick=True)
            if not a.is_aligned():
                out.append(line)
                continue
            this = alignments[a.read_name + ("_1" if num == 1 else "_2")]
            pair = alignments.get(a.read_name + ("_2" if num == 1 else "_1"), [])
            ok = not pair or len(this) == 1 or any(                    # alignment_pass_qc, filter.rs:352-377
                a.ref_name == p.ref_name and lo <= get_insert_size(a, p) <= hi and get_orientation(a, p) == orientation for p in pair)
            out.append(line if ok else line + "\tZP:Z:fail")
        outs.append(("\n".join(out) + "\n").encode("latin-1") if out else b"")
    return dict(out1=outs[0], out2=outs[1], low=lo, high=hi, orientation=orientation)
