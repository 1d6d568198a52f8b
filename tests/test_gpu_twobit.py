"""The 2-bit staged reads of k_tile on the GPU against the oracle: the case of tests/test_emu_twobit.py through polish_files plain, with
--debug and with --changes, byte for byte, and once through the packed-array path's statistics."""
import pytest

import polypolish_b200 as pp
from tests import twobitgen as tg
from tests.test_gpu_limits import fasta_of, same_stats
from tests.test_gpu_ring import check_files, ctx  # noqa: F401  (the module's context fixture)

pytestmark = pytest.mark.gpu


def test_twobit(ctx, oracle, tmp_path):  # noqa: F811
    case = tg.twobit(41)
    fa, sams = check_files(ctx, oracle, tmp_path, case)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    assert p.view.seq_bits == 4
    exp = oracle.polish(fa, sams)
    ctx.upload(f.view, p.view)
    r = ctx.polish_resident()
    assert fasta_of(f, r["sequences"]) == exp["fasta"]
    same_stats(r, exp)
    p.close()
