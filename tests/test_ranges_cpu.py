"""The byte ranges of multi-GPU ingestion (pp_sam_split_ranges) against the reference's read groups, without a GPU.

Every GPU tokenises one range of every SAM file and opens a read group at the range's first alignment, so a cut must never fall between
two aligned records of one group as the reference forms them (tests/rangegen.py ref_groups): unaligned records, '@' lines and blank
lines inside a group, empty-QNAME records (which join the group after them), CRLF, an unterminated last line, a group larger than a
range, files with fewer lines than ranges, and fuzzgen texts with those insertions."""
import pytest

from tests import rangegen as rg

TEXTS = rg.cpu_texts()


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


@pytest.mark.parametrize("name", sorted(TEXTS))
def test_cuts_keep_reference_groups(tmp_path, name):
    """For every range count: the cuts start at 0, end at the file size, never decrease, fall on line starts, and no reference group
    has aligned records in two ranges."""
    data = TEXTS[name]
    p = tmp_path / "x.sam"
    p.write_bytes(data)
    starts = {s for s, _ in rg.lines_of(data)} | {len(data)}
    for n in rg.NS:
        cuts = rg.sam_cuts(p, n)
        assert len(cuts) == n + 1 and cuts[0] == 0 and cuts[-1] == len(data), (n, cuts)
        assert cuts == sorted(cuts), (n, cuts)
        assert set(cuts) <= starts, (n, cuts)
        assert rg.split_groups(data, cuts) == [], (n, cuts)


def test_cuts_spread_plain_groups():
    """Where nothing holds a cut back (one-record and two-record groups of plain names), n ranges are all non-empty and none holds
    more than twice its share."""
    import tempfile
    import os
    data = TEXTS["plain"]
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "x.sam")
        open(p, "wb").write(data)
        for n in (2, 3, 4, 8, 16, 32):
            cuts = rg.sam_cuts(p, n)
            sizes = [b - a for a, b in zip(cuts, cuts[1:])]
            assert min(sizes) > 0 and max(sizes) < 2 * len(data) / n, (n, sizes)


def test_old_rule_splits_groups():
    """The model of the earlier rule (cut before the first line whose QNAME differs from the previous line's) splits groups of every
    kind of text but the plain one: the invariant above is not empty."""
    for name, data in TEXTS.items():
        split = {n: len(rg.split_groups(data, rg.old_cuts(data, n))) for n in rg.NS}
        if name in ("plain", "one_unterminated_line"):
            assert not any(split.values()), (name, split)
        else:
            assert any(split.values()), (name, split)


def test_broken_line_takes_a_cut(tmp_path):
    """A line whose FLAG does not parse may take a cut (the tokeniser hands such a file to the host packer); the cuts still fall on line
    starts, and a line longer than the window makes the call fail (one GPU reads the whole file)."""
    lines = [rg.toy_record("r%d" % (i // 3), 0, 5) for i in range(60)]
    lines[31] = "broken\tx\tc1"
    data = ("\n".join(lines) + "\n").encode()
    p = tmp_path / "b.sam"
    p.write_bytes(data)
    cuts = rg.sam_cuts(p, 2)
    assert cuts[1] == data.index(b"broken")
    long = tmp_path / "long.sam"
    long.write_bytes(data + b"x" * (3 << 20) + b"\n" + data)
    import ctypes as C
    from polypolish_b200 import api
    assert api.lib().pp_sam_split_ranges(str(long).encode(), 2, (C.c_uint64 * 3)()) != 0


@pytest.mark.parametrize("kind,careful", [(k, False) for k in rg.KINDS if k != "plain"] + [("unaligned", True), ("comment", True)])
def test_group_cases_are_sharp(oracle, tmp_path, kind, careful):
    """The GPU group cases (tests/test_gpu_ranges.py): for every context count the earlier rule splits at least one group over P, and
    the oracle reading the file cut at those places as separate files (what the GPUs do with a split group: a file's pieces open their
    own groups) changes P, while the whole file keeps it."""
    case = rg.group_case(kind, careful=careful)
    f = case.facts
    fa, sams = case.write(tmp_path)
    whole = oracle.polish(fa, sams, debug=True, **case.opts)
    row = whole["debug_tsv"].split(b"\n")[1 + f["P"]].split(b"\t")
    assert row[7] == b"low_depth", row
    data = sams[0].read_bytes()
    for n in rg.GPU_NS:
        assert f["split"][n] and f["old_depth"][n] >= f["min_depth"] > f["depth"], (n, f)
        parts = []
        for i, piece in enumerate(rg.pieces(data, rg.old_cuts(data, n))):
            if rg.ref_groups(piece):
                q = tmp_path / ("p%d_%d.sam" % (n, i))
                q.write_bytes(piece)
                parts.append(q)
        cut = oracle.polish(fa, parts + sams[1:], debug=True, **case.opts)
        assert cut["fasta"] != whole["fasta"], n
        assert cut["debug_tsv"].split(b"\n")[1 + f["P"]].split(b"\t")[7] == b"changed", n


@pytest.mark.parametrize("name", sorted(rg.ORDER_CASES))
def test_order_cases(oracle, tmp_path, name):
    """The order cases of tests/test_gpu_ranges.py: the covering reads lie in every range of every file as the library cuts them, no
    group crosses a range, the probe contig's owner is not context 0 and SEQ="*" records have their source on another context's contig.
    The "on" order sums exactly to the boundary and every wrong piece order (range-major, ranges reversed, files swapped, rotated by
    destination) crosses it; the oracle on the text reordered by each wrong model gives P another row than on the "on" text, and so does
    the "off" twin."""
    on, off = rg.order_case(name, on=True), rg.order_case(name, on=False)
    f = on.facts
    assert f["pieces"] == f["planned"] and off.facts["pieces"] == off.facts["planned"]
    assert set(f["pieces"]) == {(i, r) for i in range(f["n_files"]) for r in range(f["n"])}
    assert all(len(g) == 1 for g in f["group_ranges"] + off.facts["group_ranges"])
    assert f["probe_owner"] != 0 and f["sum"] == f["target"] and off.facts["sum"] == f["off_target"]
    for m, s in f["models"].items():
        assert (s - f["target"]) * f["side"] > 0, (m, s)
    assert any(a != b for a, b, _, _ in f["star_src"])
    assert any(over and a != b for a, b, _, over in f["star_src"])                 # a record over P whose source is on a filler
    if f["n"] >= 3:
        assert any(len({a, b, r}) == 3 for a, b, r, _ in f["star_src"])             # destination, source's owner, range: three contexts
    d = tmp_path / "on"
    d.mkdir()
    fa, sams = on.write(d)
    exp = oracle.polish(fa, sams, debug=True, **on.opts)
    row = exp["debug_tsv"].split(b"\n")[f["row"]]
    assert row.split(b"\t")[:2] == [b"probe", b"522"] and row.split(b"\t")[7] == b"changed"
    for m in f["models"]:
        q = tmp_path / ("%s.sam" % m)
        q.write_bytes(rg.reorder(on, m))
        got = oracle.polish(fa, [q], debug=True, **on.opts)["debug_tsv"].split(b"\n")[f["row"]]
        assert got != row, m
    d = tmp_path / "off"
    d.mkdir()
    fa2, sams2 = off.write(d)
    assert oracle.polish(fa2, sams2, debug=True, **off.opts)["debug_tsv"].split(b"\n")[f["row"]] != row
