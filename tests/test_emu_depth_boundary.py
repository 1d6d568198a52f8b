"""Positions whose depth sits exactly on a vote boundary: the reference's sequential f64 sum of 1/k lands on the boundary or one
ulp below it depending on the SAM order of the covering alignments.  k_tile's fixed-point depth bound straddles the boundary
there, so only the ordered depth walk gives the reference's vote (polypolish_b200/csrc/polish_dev.cuh, depth_bounds)."""
import random

import pytest

from tests.test_emu_polish import check

# k of the alignments covering the probed position, in SAM order, and the reference's depth there (sequential sum of 1/k)
MIN_DEPTH_ON = [3, 6, 2, 3, 3, 6, 3, 1, 3, 1, 2]            # 5.0
MIN_DEPTH_BELOW = [2, 6, 3, 6, 3, 3, 1, 3, 1, 2, 3]         # 4.999999999999999
HALF_ON = [1, 10, 1, 10, 10, 10, 10, 10, 10, 10, 10, 1, 1, 10, 1, 1]      # 7.0
HALF_BELOW = [10, 10, 1, 1, 1, 10, 10, 10, 10, 1, 1, 10, 10, 10, 10, 1]   # 6.999999999999999


def _seq_sum(ks):
    s = 0.0
    for k in ks:
        s += 1.0 / k
    return s


def write_case(tmp_path, ks, x_reads=0):
    """Contig `probe` with one position P covered by len(ks) alignments (read i has ks[i] good alignments; the others sit on
    contig `filler`).  Every alignment over P carries base Y != draft, the first `x_reads` base X instead."""
    rng = random.Random(11)
    probe = "".join(rng.choice("ACGT") for _ in range(400))
    filler = "".join(rng.choice("ACGT") for _ in range(6000))
    P = 200
    others = [b for b in "ACGT" if b != probe[P]]
    y, x = others[0], others[1]
    fa = tmp_path / "a.fasta"
    fa.write_text(">probe\n" + probe + "\n>filler\n" + filler + "\n")
    lines = []
    fpos = 10
    for i, k in enumerate(ks):
        s = P - 30 + (i % 7)
        seq = probe[s:P] + (x if i < x_reads else y) + probe[P + 1:s + 60]
        lines.append(f"r{i}\t0\tprobe\t{s + 1}\t60\t60M\t*\t0\t0\t{seq}\t*\tNM:i:1")
        for _ in range(k - 1):
            lines.append(f"r{i}\t256\tfiller\t{fpos + 1}\t0\t60M\t*\t0\t0\t{filler[fpos:fpos + 60]}\t*\tNM:i:0")
            fpos += 37
    sam = tmp_path / "a.sam"
    sam.write_text("\n".join(lines) + "\n")
    return fa, sam, P


@pytest.mark.parametrize("ks", [MIN_DEPTH_ON, MIN_DEPTH_BELOW], ids=["on", "below"])
def test_emu_depth_on_min_depth(oracle, tmp_path, ks):
    """Depth 5 against min_depth 5: low_depth (keep the draft base) or changed to the base every read carries."""
    assert _seq_sum(ks) == (5.0 if ks is MIN_DEPTH_ON else 4.999999999999999)
    fa, sam, P = write_case(tmp_path, ks)
    r = check(oracle, fa, [sam], grid_tiles=1, min_depth=5)
    assert r["changed"][0] == (1 if ks is MIN_DEPTH_ON else 0)


@pytest.mark.parametrize("ks", [HALF_ON, HALF_BELOW], ids=["on", "below"])
def test_emu_depth_on_half(oracle, tmp_path, ks):
    """depth * fraction_invalid = 3.5 or one ulp below: invalid threshold 4 or 3 against an allele seen 3 times, next to one
    above the valid threshold (changed, or too_close)."""
    assert _seq_sum(ks) == (7.0 if ks is HALF_ON else 6.999999999999999)
    fa, sam, P = write_case(tmp_path, ks, x_reads=3)
    r = check(oracle, fa, [sam], grid_tiles=1, min_depth=1, fraction_valid=0.9, fraction_invalid=0.5)
    assert r["changed"][0] == (1 if ks is HALF_ON else 0)
