"""The staged general walk of k_tile on the GPU against the oracle: the cases of tests/test_emu_staged.py through polish_files plain,
with --debug and with --changes, byte for byte, and once through the packed-array path's statistics."""
import pytest

import polypolish_b200 as pp
from tests.test_emu_staged import CASES
from tests.test_gpu_limits import fasta_of, same_stats
from tests.test_gpu_ring import check_files, ctx  # noqa: F401  (the module's context fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CASES))
def test_staged(ctx, oracle, tmp_path, name):  # noqa: F811
    case = CASES[name]()
    fa, sams = check_files(ctx, oracle, tmp_path, case)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == case.facts["seq_bits"]
    exp = oracle.polish(fa, sams)
    ctx.upload(f.view, p.view)
    r = ctx.polish_resident()
    assert fasta_of(f, r["sequences"]) == exp["fasta"]
    same_stats(r, exp)
    p.close()
