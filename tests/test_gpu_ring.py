"""k_tile's chunk ring on the GPU against the oracle: the cases of tests/test_emu_ring.py, and D, a contig of at least four tiles per
SM that repeats A's schedule, so that every CTA takes several tiles and carries its stages' parity from one to the next.  Each case
runs through polish_files plain, with --debug and with --changes (4-bit and 8-bit, with and without the change list: all four k_tile
instances), byte for byte; D also runs twice on one resident upload."""
import pytest

import polypolish_b200 as pp
from tests import ringgen as rg
from tests.test_emu_ring import CASES
from tests.test_gpu_changes import changed_rows
from tests.test_gpu_limits import fasta_of, same_stats

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def case_d():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    repeat = -(-4 * sms // len(rg.SCHEDULE))
    case = rg.chunk_shapes(14, repeat=repeat)
    sched = case.facts["schedule"]
    assert len(sched) >= 4 * sms
    # tiles whose warps end on odd and even chunk counts, next to each other: with four or more tiles per CTA, which of them a CTA
    # runs one after another is up to the ticket, and the mix is what makes its stages' parity carry both ways
    pairs = {(a % 2, b % 2) for x, y in zip(sched, sched[1:]) for a, b in zip(rg.warp_chunks(x), rg.warp_chunks(y)) if a and b}
    assert {(0, 1), (1, 0)} <= pairs
    return case


def check_files(ctx, oracle, d, case):
    fa, sams = case.write(d)
    exp = oracle.polish(fa, sams, debug=True)
    assert sum(exp["changed"]) > 0
    assert ctx.polish_files(fa, sams) == exp["fasta"]
    dbg, chg = d / "debug.tsv", d / "changes.tsv"
    assert ctx.polish_files(fa, sams, debug=dbg) == exp["fasta"]
    assert dbg.read_bytes() == exp["debug_tsv"]
    assert ctx.polish_files(fa, sams, changes=chg) == exp["fasta"]
    assert chg.read_bytes() == changed_rows(exp["debug_tsv"])
    return fa, sams


@pytest.mark.parametrize("name", list(CASES) + ["D"])
def test_ring(ctx, oracle, tmp_path, name):
    case = case_d() if name == "D" else CASES[name]()
    fa, sams = check_files(ctx, oracle, tmp_path, case)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == case.facts["seq_bits"]
    if name == "D":
        exp = oracle.polish(fa, sams)
        ctx.upload(f.view, p.view)
        r1, r2 = ctx.polish_resident(), ctx.polish_resident()
        assert fasta_of(f, r1["sequences"]) == exp["fasta"] and r1["sequences"] == r2["sequences"]
        same_stats(r1, exp)
        same_stats(r2, exp)
        assert r1["total_depth"] == pytest.approx(r2["total_depth"], rel=1e-12)
    p.close()
