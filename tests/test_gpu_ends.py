"""Contig ends on the GPU against the oracle: the cases of tests/test_emu_ends.py through polish_files with both parsers (plain,
--debug, --changes), polish_packed's statistics, polish_files_multi with 2 and 3 contexts on one device (a P record's k crosses to
its partner's context as a ghost), and the CLI's per-contig log once.  Error cases: the reference's message, or for an overrun the
library's message naming the read the reference's panic names."""
import os
import re

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests.test_emu_ends import ERRORS, LEGAL, expected_error, first_oob
from tests.test_gpu_limits import check_files, fasta_of, same_stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("name", list(LEGAL))
def test_ends(ctx, oracle, tmp_path, name):
    case = LEGAL[name]()
    fa, sams = case.write(tmp_path)
    exp = check_files(ctx, oracle, tmp_path, fa, sams)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == case.facts["seq_bits"]
    r = ctx.polish_packed(f.view, p.view)
    assert fasta_of(f, r["sequences"]) == exp["fasta"]
    same_stats(r, exp)
    p.close()
    for parser in (0, 1):
        for n in (2, 3):
            assert api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser) == exp["fasta"], (parser, n)


def test_ends_cli_log(oracle, tmp_path):
    """The CLI's per-contig log lines on P: mean depth, zero-depth bp and changed positions are the oracle's statistics."""
    import subprocess
    case = LEGAL["P"]()
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams)
    r = subprocess.run([os.path.join(ROOT, "build", "polypolish"), "polish", str(fa)] + [str(s) for s in sams], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == exp["fasta"]
    log = r.stderr.decode()
    lens = case.facts["lens"]
    depths = re.findall(r"mean read depth: ([0-9.]+)x", log)
    assert depths == ["%.1f" % (exp["total_depth"][i] / lens[i]) for i in range(len(lens))]
    assert [int(x.replace(",", "")) for x in re.findall(r"([0-9,]+) positions? changed", log)] == exp["changed"]
    assert [int(x.replace(",", "")) for x in re.findall(r"([0-9,]+) bp ha(?:s|ve) a depth of zero", log)] == exp["zero_depth"]


def check_message(got, msg, m):
    if m:
        assert got.startswith("alignment extends past the end of its reference sequence") and got.endswith("(read %s)" % m.group(1)), got
    else:
        assert got == msg


@pytest.mark.parametrize("name", list(ERRORS))
def test_end_errors(ctx, oracle, tmp_path, name):
    case = ERRORS[name]
    msg, m = expected_error(case, oracle, tmp_path)
    fa, sams = case.write(tmp_path)
    for parser in (0, 1):
        ctx.set_parser(parser)
        try:
            with pytest.raises(pp.PolypolishError) as e:
                ctx.polish_files(fa, sams)
        finally:
            ctx.set_parser(0)
        check_message(e.value.msg, msg, m)
    for n in (2, 3):
        with pytest.raises(pp.PolypolishError) as e:
            api.polish_files_multi(fa, sams, devices=[0] * n)
        check_message(e.value.msg, msg, m)
    if m:
        f = pp.load_fasta(fa)
        p = pp.pack_sams(f, sams)
        with pytest.raises(pp.PolypolishError) as e:
            ctx.polish_packed(f.view, p.view)
        assert e.value.error_aln == first_oob(case, m.group(1))
        p.close()
