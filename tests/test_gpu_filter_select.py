"""The filter's insert-size thresholds and pair verdicts on the GPU against the exact model of tests/filtergen.py: pp_filter on the
mate arrays, `filter` through the device text path and the host parser, `filter` over 2, 3 and 8 contexts (thresholds reduced across
contexts), one `filter-polish` case whose FASTA hangs on a record at insert == high, and 4 M names through pp_filter."""
import random

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import filtergen as fg

pytestmark = pytest.mark.gpu

NS = (2, 3, 8)
CASES = fg.cases()
IDS = [c.name for c in CASES]


@pytest.fixture(scope="module")
def ctxs():
    import __graft_entry__ as g
    g.build()
    cs = [pp.Context(0) for _ in range(max(NS))]
    yield cs
    for c in cs:
        c.close()


def check_packed(ctx, case, m):
    a = case.arrays()
    got = ctx.filter_packed(a[0], a[1], case.n_names, case.orientation_code, case.low, case.high)
    assert (got["low"], got["high"]) == (m["low"], m["high"])
    assert (fg.ORIENT[got["orientation"]], got["pairs"], got["n_pass"]) == (m["orientation"], m["pairs"], m["n_pass"])
    assert np.array_equal(got["pass1"], np.array(m["pass1"], np.uint8))
    assert np.array_equal(got["pass2"], np.array(m["pass2"], np.uint8))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_packed_matches_model(ctxs, case):
    """pp_filter on the arrays: thresholds, orientation, pair counts, pass counts and every verdict."""
    check_packed(ctxs[0], case, fg.model(case))


def write_case(d, case):
    t1, t2 = case.texts()
    i1, i2 = d / "i1.sam", d / "i2.sam"
    i1.write_bytes(t1)
    i2.write_bytes(t2)
    return i1, i2


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_text_paths_match_oracle(ctxs, oracle, tmp_path, case):
    """`filter` on the SAM texts through the device text path and the host parser: both files are the oracle's, byte for byte."""
    ctx = ctxs[0]
    i1, i2 = write_case(tmp_path, case)
    kw = dict(orientation=case.orientation, low=case.low, high=case.high)
    exp = oracle.filter(i1, i2, **kw)
    assert (exp["out1"], exp["out2"]) == case.expected_texts()
    for mode in (0, 1):
        o1, o2 = tmp_path / f"o1_{mode}.sam", tmp_path / f"o2_{mode}.sam"
        ctx.set_parser(mode)
        try:
            ctx.filter_files(i1, i2, o1, o2, **kw)
        finally:
            ctx.set_parser(0)
        assert o1.read_bytes() == exp["out1"] and o2.read_bytes() == exp["out2"], mode


def threshold_lines(err):
    return [x for x in err.splitlines() if x.startswith(("Low threshold:", "High threshold:"))]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_multi_context_matches_oracle(ctxs, oracle, tmp_path, capfd, case):
    """`filter` over 2, 3 and 8 contexts: the histograms of every round are summed over the owners of the read names.  Same files
    and the same threshold lines as one context and the model, through the multi-context path."""
    i1, i2 = write_case(tmp_path, case)
    kw = dict(orientation=case.orientation, low=case.low, high=case.high)
    m = fg.model(case)
    e1, e2 = case.expected_texts(m)
    want = [f"Low threshold:  {m['low']}", f"High threshold: {m['high']}"]
    capfd.readouterr()
    for n in (1,) + NS:
        o1, o2 = tmp_path / f"o1_{n}.sam", tmp_path / f"o2_{n}.sam"
        api.filter_files_multi(i1, i2, o1, o2, contexts=ctxs[:n], verbose=True, **kw)
        err = capfd.readouterr().err
        assert n == 1 or f"device text path over {n} GPUs" in err, err
        assert threshold_lines(err) == want, n
        assert o1.read_bytes() == e1 and o2.read_bytes() == e2, n


def test_large_packed(ctxs):
    """4 M names: k_f_hist runs its full grid and the ranks' buckets hold ~2 M names in rounds 24, 16 and 8."""
    case = fg.large_case()
    m = fg.model(case)
    tr = fg.select_trace(case, m)
    assert all(c > (1 << 16) for rnd in tr[:3] for _, _, c in rnd), tr
    check_packed(ctxs[0], case, m)


# ---- filter-polish: a FASTA that depends on records at insert == high ---------------------------------------------------------
ALT = {"A": "C", "C": "G", "G": "T", "T": "A"}


def polish_case(d, variant_insert, seed=5):
    """Two contigs; 40 unique 'fr' pairs (inserts 300..400, one at 400 = the high threshold with the default percentiles) away from
    position P of ctg0; 6 reads with two alignments each: one on ctg0 over P with another base there, `variant_insert` from its
    mate, and one on ctg1.  With variant_insert == high the first passes and P changes; one past high, both fail and P keeps its base."""
    rng = random.Random(seed)
    asm = ["".join(rng.choice("ACGT") for _ in range(4000)) for _ in range(2)]
    fa = d / "asm.fasta"
    fa.write_text("".join(f">ctg{i}\n{s}\n" for i, s in enumerate(asm)))
    rows = [[], []]

    def rec(k, name, flag, c, start, seq=None, nm=0):
        s = seq or asm[c][start:start + 50]
        rows[k].append(f"{name}\t{flag}\tctg{c}\t{start + 1}\t60\t50M\t*\t0\t0\t{s}\t{'I' * 50}\tNM:i:{nm}")
    inserts = rng.sample(range(300, 400), 39) + [400]
    for i, ins in enumerate(inserts):
        s = rng.randint(0, 2000)
        rec(0, f"u{i}", 0, 0, s)
        rec(1, f"u{i}", 16, 0, s + ins - 50)
    P = 3000
    for j in range(6):
        x = P - 10 - 5 * j
        seq = asm[0][x:P] + ALT[asm[0][P]] + asm[0][P + 1:x + 50]
        rec(0, f"v{j}", 0, 0, x, seq, 1)
        rec(0, f"v{j}", 256, 1, 500 + 7 * j)
        rec(1, f"v{j}", 16, 0, x + variant_insert - 50)
    i1, i2 = d / "r1.sam", d / "r2.sam"
    i1.write_text("".join(r + "\n" for r in rows[0]))
    i2.write_text("".join(r + "\n" for r in rows[1]))
    return fa, i1, i2, asm[0][P], P


@pytest.mark.parametrize("delta", [0, 1])
def test_filter_polish_hangs_on_high(ctxs, oracle, tmp_path, delta):
    ctx = ctxs[0]
    fa, i1, i2, orig, P = polish_case(tmp_path, 400 + delta)
    fo = oracle.filter(i1, i2)
    assert fo["high"] == 400
    o1, o2 = tmp_path / "o1.sam", tmp_path / "o2.sam"
    o1.write_bytes(fo["out1"])
    o2.write_bytes(fo["out2"])
    exp = oracle.polish(fa, [o1, o2])["fasta"]
    ctg0 = exp.split(b"\n")[1].decode()
    assert ctg0[P] == (ALT[orig] if delta == 0 else orig)
    for mode in (0, 1):
        ctx.set_parser(mode)
        try:
            assert ctx.filter_polish_files(fa, i1, i2) == exp, mode
        finally:
            ctx.set_parser(0)
    assert api.filter_polish_files_multi(fa, i1, i2, contexts=ctxs[:2]) == exp
