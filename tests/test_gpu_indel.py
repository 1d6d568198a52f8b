"""The one-indel fast walk of k_tile on the GPU against the oracle: the cases of tests/test_emu_indel.py through polish_files plain,
with --debug and with --changes, byte for byte, and once through the packed-array path's statistics."""
import pytest

import polypolish_b200 as pp
from tests.test_emu_indel import CASES
from tests.test_gpu_limits import fasta_of, same_stats
from tests.test_gpu_ring import check_files, ctx  # noqa: F401  (the module's context fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CASES))
def test_indel(ctx, oracle, tmp_path, name):  # noqa: F811
    fa, sams = check_files(ctx, oracle, tmp_path, CASES[name]())
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    exp = oracle.polish(fa, sams)
    ctx.upload(f.view, p.view)
    r = ctx.polish_resident()
    assert fasta_of(f, r["sequences"]) == exp["fasta"]
    same_stats(r, exp)
    p.close()
