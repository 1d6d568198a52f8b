"""`polish` and `filter-polish` over several contexts read every SAM file in byte ranges (pp_sam_split_ranges), one range per context, and
exchange read groups between the contexts.  These cases (tests/rangegen.py group_case) put read groups where a cut before the first line
of another QNAME would split them: unaligned records of another name, @CO lines and blank lines inside a group, empty-QNAME records in
front of it.  A split group would change the vote at the probe position (its halves count 1/1 instead of 1/k, or pass --careful), so
each case is compared with the oracle: the FASTA and the change report, with 2, 3 and 8 contexts on one device, and every run must have
gone through the exchange (not through a fallback to one context or the host packer).  The order cases (tests/rangegen.py order_case)
check that every destination holds the pieces of the ranges in global SAM order."""
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import rangegen as rg
from tests.test_gpu_filter_multi import changed_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctxs():
    import __graft_entry__ as g
    g.build()
    cs = [pp.Context(0) for _ in range(max(rg.GPU_NS))]
    yield cs
    for c in cs:
        c.close()


def with_8bit_pair_read(path):
    """A read pair record on a filler contig gets a SEQ byte outside the 4-bit alphabet (every context tokenises again with 8 bits)."""
    lines = path.read_bytes().split(b"\n")
    for i, x in enumerate(lines):
        f = x.split(b"\t")
        if f[0].startswith(b"p") and len(f) > 10:
            f[9] = f[9][:20] + b"Z" + f[9][21:]
            lines[i] = b"\t".join(f)
            break
    path.write_bytes(b"\n".join(lines))


def seq_bits(cs):
    """The base width of the datasets the contexts hold after a call."""
    return {c.dataset_arrays()["seq_bits"] for c in cs}


CASES = [(k, False, False) for k in rg.KINDS if k != "plain"] + [("unaligned", True, False), ("comment", False, True)]


@pytest.mark.parametrize("kind,careful,eight_bit", CASES)
def test_groups_across_ranges(ctxs, oracle, tmp_path, capfd, kind, careful, eight_bit):
    case = rg.group_case(kind, careful=careful)
    f = case.facts
    fa, sams = case.write(tmp_path)
    if eight_bit:
        with_8bit_pair_read(sams[0])
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    assert exp["debug_tsv"].split(b"\n")[1 + f["P"]].split(b"\t")[7] == b"low_depth"
    for n in rg.GPU_NS:
        assert f["split"][n], n                                       # the earlier cut rule splits a group over P
        chg = tmp_path / f"chg_{n}.tsv"
        got = api.polish_files_multi(fa, sams, contexts=ctxs[:n], verbose=True, changes=chg, **case.opts)
        err = capfd.readouterr().err
        assert f"read groups exchanged between {n} GPUs" in err, (n, err)
        assert got == exp["fasta"], n
        assert chg.read_bytes() == changed_rows(exp["debug_tsv"]), n
        assert seq_bits(ctxs[:n]) == {8 if eight_bit else 4}, n        # the 8-bit case went through the PP_TOK_NEED8 retry
    ctxs[0].set_parser(1)
    try:                                                              # the control: host packer and host sharder
        assert api.polish_files_multi(fa, sams, contexts=ctxs[:3], parser=1, **case.opts) == exp["fasta"]
    finally:
        ctxs[0].set_parser(0)


@pytest.mark.parametrize("kind,careful", [("unaligned", False), ("empty_run", False), ("comment", True)])
def test_filter_polish_groups_across_ranges(ctxs, oracle, tmp_path, capfd, kind, careful):
    """The same files through the fused `filter-polish` over n contexts: the oracle's `filter` keeps every record over P (the group
    reads have no mates), then its `polish` of the filtered files."""
    case = rg.group_case(kind, careful=careful)
    fa, sams = case.write(tmp_path)
    fo = oracle.filter(sams[0], sams[1])
    assert not [x for x in fo["out1"].split(b"\n") if b"\tprobe\t" in x and b"ZP:Z:fail" in x]
    o1, o2 = tmp_path / "of1.sam", tmp_path / "of2.sam"
    o1.write_bytes(fo["out1"])
    o2.write_bytes(fo["out2"])
    exp = oracle.polish(fa, [o1, o2], debug=True, **case.opts)
    assert exp["debug_tsv"].split(b"\n")[1 + case.facts["P"]].split(b"\t")[7] == b"low_depth"
    for n in rg.GPU_NS:
        chg = tmp_path / f"chg_{n}.tsv"
        got = api.filter_polish_files_multi(fa, sams[0], sams[1], contexts=ctxs[:n], changes=chg, verbose=True, **case.opts)
        err = capfd.readouterr().err
        assert f"filter over {n} GPUs" in err and f"read groups exchanged between {n} GPUs" in err, (n, err)
        assert got == exp["fasta"], n
        assert chg.read_bytes() == changed_rows(exp["debug_tsv"]), n


def test_more_contexts_than_contigs(ctxs, oracle, tmp_path, capfd):
    """Eight contexts on three contigs: `polish` uses one context per contig (no context would own nothing), so the files are cut into
    three ranges, and the group case still gives the oracle's FASTA."""
    case = rg.group_case("unaligned", n_fillers=2)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, **case.opts)
    assert api.polish_files_multi(fa, sams, contexts=ctxs[:8], verbose=True, **case.opts) == exp["fasta"]
    assert "read groups exchanged between 3 GPUs" in capfd.readouterr().err


@pytest.mark.parametrize("name", sorted(rg.ORDER_CASES))
def test_sam_order_across_ranges(ctxs, oracle, tmp_path, capfd, name):
    """The order cases (tests/rangegen.py order_case): a probe position on a vote boundary whose covering reads lie in every range of 2
    or 3 SAM files, the probe contig owned by a context other than 0, SEQ="*" records whose source sits on another context's contig.
    Only (file, range, line) order at the probe's owner gives the reference's sum (tests/test_ranges_cpu.py test_order_cases); the
    "on" and "off" orders vote differently.  With --changes (every k != 1 sub-tile walks) and without (the depth bound must send P to
    the walk), and through the host sharder as the control."""
    rows = []
    for on in (True, False):
        case = rg.order_case(name, on=on)
        f = case.facts
        d = tmp_path / ("on" if on else "off")
        d.mkdir()
        fa, sams = case.write(d)
        exp = oracle.polish(fa, sams, debug=True, **case.opts)
        rows.append(exp["debug_tsv"].split(b"\n")[f["row"]])
        n = f["n"]
        chg = d / "chg.tsv"
        got = api.polish_files_multi(fa, sams, contexts=ctxs[:n], verbose=True, changes=chg, **case.opts)
        err = capfd.readouterr().err
        assert f"read groups exchanged between {n} GPUs" in err, err
        assert got == exp["fasta"], on
        assert chg.read_bytes() == changed_rows(exp["debug_tsv"]), on
        assert seq_bits(ctxs[:n]) == {f["seq_bits"]}
        assert api.polish_files_multi(fa, sams, contexts=ctxs[:n], **case.opts) == exp["fasta"], on
        assert api.polish_files_multi(fa, sams, contexts=ctxs[:n], parser=1, **case.opts) == exp["fasta"], on
        ctxs[0].set_parser(0)
    assert rows[0] != rows[1]
