"""The ordered depth walk's merge on the GPU against the oracle (the cases of tests/test_emu_depth_walk.py, and the high-cover case W9):
probe positions on a vote boundary whose covering reads are spread over the runs depth_walk_two and depth_walk_steps merge.  With
--debug / --changes every k != 1 sub-tile walks; without them the fixed-point bound has to see that the position straddles the
boundary and walk.  Either way the on and off orders vote differently, and the printed depth is the reference's."""
import pytest

import polypolish_b200 as pp
from tests import walkgen as wg
from tests.test_emu_depth_walk import check_facts, expected
from tests.test_gpu_limits import check_files, check_packed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def check_plain(ctx, oracle, fa, sams, ci, **opts):
    """test_gpu_limits.check_plain for the probe on contig `ci`: without --debug / --changes, through polish_files with both parsers,
    polish_packed and the resident dataset.  Returns the GPU's `changed` of contig ci from the last two."""
    exp = oracle.polish(fa, sams, **opts)
    for parser in (0, 1):
        ctx.set_parser(parser)
        try:
            assert ctx.polish_files(fa, sams, **opts) == exp["fasta"], parser
        finally:
            ctx.set_parser(0)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)                       # (kept alive while the device reads its arrays)
    rs = check_packed(ctx, oracle, fa, sams, f, p, [opts])
    p.close()
    return [r["changed"][ci] for r in rs]


@pytest.mark.parametrize("name", list(wg.CASES))
def test_depth_walk(ctx, oracle, tmp_path, name):
    on_case, off_case, spec = wg.case_pair(name)
    got, plain = [], []
    for on, case in ((True, on_case), (False, off_case)):
        check_facts(case, spec, on)
        d = tmp_path / ("on" if on else "off")
        d.mkdir()
        fa, sams = case.write(d)
        f = pp.load_fasta(fa)
        p = pp.pack_sams(f, sams)
        assert p.view.seq_bits == (8 if spec["eight_bit"] else 4)
        p.close()
        want, printed = expected(spec, on)
        ci = 1 if case.facts["head"] else 0
        exp = check_files(ctx, oracle, d, fa, sams, **case.opts)                # --debug and --changes, both parsers
        row = exp["debug_tsv"].split(b"\n")[1 + case.facts["P"]].split(b"\t")
        assert row[:2] == [b"probe", str(case.facts["probe_local"]).encode()] and row[3] == printed
        assert exp["changed"][ci] == want
        got.append(want)
        plain.append(check_plain(ctx, oracle, fa, sams, ci, **case.opts))        # without them: polish_files, packed, resident
        assert plain[-1] == [want, want]
    if spec["side"] < 0:
        assert got == [1, 0] and plain == [[1, 1], [0, 0]]


def test_high_cover_needs_the_n2_term(ctx, oracle, tmp_path):
    """W9: 200,000 alignments over P, the ones first.  The reference's sum lies below the fixed-point depth by more than n 2^-41, and
    the valid threshold's rounding tie lies in between: P changes only if the bound keeps its n^2 term (and the walk over thousands of
    windows gets the reference's sum)."""
    case = wg.high_cover()
    f = case.facts
    assert f["ref_outside"] and f["d_ref"] < f["d_fx"] - f["n"] * 2.0 ** -41
    assert f["ref_threshold"] == f["c"] and f["nn_threshold"] == f["c"] + 1 and f["draft_below_invalid"]
    assert f["runs"] == {"b-1": 100_000, "b": 100_000} and f["n"] == 200_000
    fa, sams = case.write(tmp_path)
    exp = check_files(ctx, oracle, tmp_path, fa, sams, **case.opts)
    assert exp["changed"][0] == 1
    row = exp["debug_tsv"].split(b"\n")[1 + f["P"]].split(b"\t")
    assert row[:2] == [b"probe", str(f["P"]).encode()] and row[7] == b"changed"
    assert check_plain(ctx, oracle, fa, sams, 0, **case.opts) == [1, 1]
