"""Strings with one 64-bit key (tests/collidegen.py) on the device: the contig lookup of the polish tokeniser, `filter` and
`filter-polish` on one context and over several (where only the context that owns a read name can see both strings), and the
other-allele chain of k_tile.  Every case is compared with the oracle, and every case differs from its twin (the colliding strings
made one string) in the oracle's answer, so each would fail if the byte check it targets were skipped.  The contexts share one device
(`devices=[0] * n`), as in test_gpu_filter_multi.py."""
import subprocess

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import collidegen as cg
from tests.rangegen import range_of, sam_cuts
from tests.test_collide_cpu import ALLELES, check_sharp, allele_case
from tests.test_emu_changes import changed_rows
from tests.test_gpu_filter_multi import ROOT, log_numbers

pytestmark = pytest.mark.gpu

NS = (2, 3, 8)


@pytest.fixture(scope="module")
def ctxs():
    import __graft_entry__ as g
    g.build()
    cs = [pp.Context(0) for _ in range(max(NS))]
    yield cs
    for c in cs:
        c.close()


def oracle_or_error(fn, *a, **kw):
    try:
        return "ok", fn(*a, **kw)
    except Exception as e:
        return "err", e.msg


# ---- A. contig names -------------------------------------------------------------------------------------------------------------
def contig_twin_differs(oracle, tmp_path, exp, **kw):
    d = tmp_path / "twin"
    d.mkdir()
    fa, sams = cg.contig_case(twin=True, **kw).write(d)
    assert oracle_or_error(oracle.polish, fa, sams) != exp


@pytest.mark.parametrize("order", ["ab", "ba"])
def test_colliding_contig_names(ctxs, oracle, tmp_path, capfd, order):
    """Both names in the assembly: the device tokeniser settles the lookup itself (PP_OK, the host packer's arrays), the FASTA and the
    statistics are the oracle's through both parsers, and over 2 and 3 contexts (one contig per owner) through the read group exchange."""
    case = cg.contig_case(order)
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams)
    contig_twin_differs(oracle, tmp_path, ("ok", exp), order=order)
    f = pp.load_fasta(fa)
    ctx = ctxs[0]
    rc, _ = ctx.tokenise(f, [sams[0].read_bytes()])
    assert rc == 0
    packed = pp.pack_sams(f, sams)                                    # (its arrays are views of its buffers)
    dev, host = ctx.dataset_arrays(), packed.arrays()
    for k, v in host.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(dev[k], v), k
    assert len(set(dev["contig"].tolist())) == 2
    for parser in (0, 1):
        ctx.set_parser(parser)
        try:
            got = ctx.polish_files(fa, sams)
        finally:
            ctx.set_parser(0)
        assert got == exp["fasta"], parser
        capfd.readouterr()
    for n in (2, 3):
        assert api.polish_files_multi(fa, sams, contexts=ctxs[:n], verbose=True) == exp["fasta"], n
        err = capfd.readouterr().err
        assert "read groups exchanged between 2 GPUs" in err, (n, err)


def test_colliding_contig_missing(ctxs, oracle, tmp_path, capfd):
    """The assembly holds NAME_A only and reads name NAME_B: the reference's error, through both parsers and over 2 contexts."""
    case = cg.contig_case("ab", only="a")
    fa, sams = case.write(tmp_path)
    exp = oracle_or_error(oracle.polish, fa, sams)
    assert exp[0] == "err" and cg.NAME_B in exp[1]
    contig_twin_differs(oracle, tmp_path, exp, only="a")
    ctx = ctxs[0]
    for parser in (0, 1):
        ctx.set_parser(parser)
        try:
            with pytest.raises(pp.PolypolishError) as e:
                ctx.polish_files(fa, sams)
        finally:
            ctx.set_parser(0)
        assert e.value.msg == exp[1], parser
    with pytest.raises(pp.PolypolishError) as e:
        api.polish_files_multi(fa, sams, contexts=ctxs[:2])
    assert e.value.msg == exp[1]
    capfd.readouterr()


# ---- B - D. filter -------------------------------------------------------------------------------------------------------------
def filter_exp(oracle, tmp_path, kind):
    """The oracle's filter of the case, after checking that the twin's verdicts differ (the claw has no merged twin: a QNAME and an
    RNAME sharing a slot change no verdict, so for it the check is that the host text path ran)."""
    out = {}
    for twin in (False, True):
        d = tmp_path / ("twin" if twin else "case")
        d.mkdir()
        fa, sams = cg.filter_case(kind, twin=twin).write(d)
        out[twin] = (fa, sams, oracle.filter(sams[0], sams[1]))
    if kind != "claw":
        v = lambda r: (cg.verdicts(r["out1"]), cg.verdicts(r["out2"]))
        assert v(out[False][2]) != v(out[True][2]), kind
    return out[False]


def host_path_ran(err):
    assert "device text path" not in err and "\ndevice path:" in "\n" + err, err


@pytest.mark.parametrize("kind", cg.FILTER_KINDS)
def test_filter_one_context(ctxs, oracle, tmp_path, capfd, kind):
    """k_ftok_verify flags the collision, the host text path filters: the oracle's bytes in both outputs."""
    fa, sams, exp = filter_exp(oracle, tmp_path, kind)
    o1, o2 = tmp_path / "o1.sam", tmp_path / "o2.sam"
    capfd.readouterr()
    api.filter_files_multi(sams[0], sams[1], o1, o2, contexts=ctxs[:1], verbose=True)
    host_path_ran(capfd.readouterr().err)
    assert o1.read_bytes() == exp["out1"] and o2.read_bytes() == exp["out2"]


@pytest.mark.parametrize("kind", ["one_file", "two_files", "joux"])
def test_filter_names_in_different_ranges(ctxs, oracle, tmp_path, capfd, kind):
    """The two colliding QNAMEs lie in different byte ranges, so every context's own k_ftok_verify passes and only the owner of the
    key (k_fx_verify) sees two strings: the n-context path gives up, the host text path gives the oracle's bytes."""
    fa, sams, exp = filter_exp(oracle, tmp_path, kind)
    names = cg.JOUX if kind == "joux" else [cg.NAME_A, cg.NAME_B]
    for n in NS:
        cuts = [sam_cuts(s, n) for s in sams]
        where = set()
        for k, s in enumerate(sams):
            text = s.read_bytes()
            for nm in names:
                at = text.find(b"\n" + nm.encode() + b"\t")
                if at >= 0:
                    where.add((nm, k, range_of(cuts[k], at + 1)))
        assert {nm for nm, _, _ in where} == set(names)
        assert len({g for _, _, g in where}) >= 2 and (0 in {g for _, _, g in where}) and (n - 1 in {g for _, _, g in where}), (n, where)
        o1, o2 = tmp_path / f"o1_{n}.sam", tmp_path / f"o2_{n}.sam"
        capfd.readouterr()
        api.filter_files_multi(sams[0], sams[1], o1, o2, contexts=ctxs[:n], verbose=True)
        err = capfd.readouterr().err
        assert f"device text path over {n} GPUs" not in err, err
        host_path_ran(err)
        assert o1.read_bytes() == exp["out1"] and o2.read_bytes() == exp["out2"], n


@pytest.mark.parametrize("kind", cg.FILTER_KINDS)
def test_filter_polish(ctxs, oracle, tmp_path, capfd, kind):
    """The fused call on 1 - 3 contexts: the FASTA and both filtered files are the oracle's `filter` then `polish`."""
    fa, sams, exp = filter_exp(oracle, tmp_path, kind)
    f1, f2 = tmp_path / "of1.sam", tmp_path / "of2.sam"
    f1.write_bytes(exp["out1"])
    f2.write_bytes(exp["out2"])
    want = oracle.polish(fa, [f1, f2])["fasta"]
    for n in (1, 2, 3):
        o1, o2 = tmp_path / f"g1_{n}.sam", tmp_path / f"g2_{n}.sam"
        assert api.filter_polish_files_multi(fa, sams[0], sams[1], o1, o2, contexts=ctxs[:n]) == want, n
        assert o1.read_bytes() == exp["out1"] and o2.read_bytes() == exp["out2"], n
    capfd.readouterr()


# ---- E. other alleles ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,vote,bits", ALLELES)
def test_colliding_alleles(ctxs, oracle, tmp_path, key, vote, bits):
    """Reads of every walk (fast one-indel, staged general, queued, escape), both strands, interleaved, some with k = 2, carry one of
    two alleles with one make_sig at one position: FASTA, --debug and --changes are the oracle's."""
    exp = check_sharp(oracle, tmp_path, key, vote, bits)
    d = tmp_path / "dev"
    d.mkdir()
    fa, sams = allele_case(key, vote, bits).write(d)
    dbg, chg = d / "debug.tsv", d / "changes.tsv"
    assert ctxs[0].polish_files(fa, sams, debug=dbg, changes=chg) == exp["fasta"]
    assert ctxs[0].dataset_arrays()["seq_bits"] == bits
    assert dbg.read_bytes() == exp["debug_tsv"]
    assert chg.read_bytes() == changed_rows(exp["debug_tsv"])


# ---- F. the command line -------------------------------------------------------------------------------------------------------
def test_cli_filter_and_polish_debug(oracle, tmp_path):
    """`polypolish filter` on colliding QNAMEs in two files and `polypolish polish --debug` on colliding alleles: the oracle's files."""
    exe = f"{ROOT}/build/polypolish"
    fa, sams, exp = filter_exp(oracle, tmp_path, "two_files")
    o1, o2 = tmp_path / "c1.sam", tmp_path / "c2.sam"
    r = subprocess.run([exe, "filter", "--in1", sams[0], "--in2", sams[1], "--out1", o1, "--out2", o2], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert o1.read_bytes() == exp["out1"] and o2.read_bytes() == exp["out2"]
    assert log_numbers(r.stderr.decode())
    d = tmp_path / "alleles"
    d.mkdir()
    exp = check_sharp(oracle, d, "sig4", "too_close", 4)
    fa, sams = allele_case("sig4", "too_close", 4).write(d)
    dbg = d / "cli_debug.tsv"
    r = subprocess.run([exe, "polish", "--debug", dbg, fa] + sams, capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"] and dbg.read_bytes() == exp["debug_tsv"]
