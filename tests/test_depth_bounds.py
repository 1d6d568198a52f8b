"""The helpers the vote reads depth through (polypolish_b200/csrc/polish_dev.cuh), against exact arithmetic: depth_deficit(k) against
round(2^40 / k), depth_bounds(n, M) against n - M 2^-40 +- (n 2^-41 + n^2 2^-52) in fractions.Fraction and against the reference's
sequential f64 sums, and vote_thresholds / bankers_rounding against a restatement of pileup.rs:70-72 and misc.rs:208-215.  The helpers
run through tests/probe/depth_probe.cu twice: on the CPU with the emulated directed rounding, and on the GPU (-m gpu) with the
hardware's."""
import math
import random
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

from tests import probe_lib

TL_DEF_COVER = 1 << 23             # positions with this many covering alignments always walk: depth_bounds is not used there
K_MAX = (1 << 32) - 1


@pytest.fixture(scope="module", params=["cpu", pytest.param("gpu", marks=pytest.mark.gpu)])
def backend(request):
    probe_lib.build(request.param)
    return request.param


def dd(k):
    """2^40 - round(2^40 / k): what depth_deficit(k) must return (2^40 / k is never a tie for k < 2^41)."""
    return (1 << 40) - round(Fraction(1 << 40, k))


def seq_sum(ks):
    """The reference's depth: the sequential f64 sum of 1.0 / k (pileup.rs:64)."""
    inv = {k: 1.0 / k for k in set(ks)}
    s = 0.0
    for k in ks:
        s += inv[k]
    return s


# ---- depth_deficit -------------------------------------------------------------------------------------------------------------
def test_depth_deficit(backend):
    rng = random.Random(1)
    ks = list(range(2, 4097)) + [K_MAX, K_MAX - 1, 1 << 31, (1 << 31) - 1, (1 << 31) + 1, 1 << 20, 3 << 20, 65535, 65536, 65537]
    ks += [rng.randint(4097, K_MAX) for _ in range(20000)]
    out = probe_lib.run(backend, k=ks)
    for k, got in zip(ks, out["dd"].tolist()):
        assert got == dd(k), k
        assert abs(Fraction((1 << 40) - got, 1 << 40) - Fraction(1, k)) <= Fraction(1, 1 << 41), k


# ---- depth_bounds --------------------------------------------------------------------------------------------------------------
def bound_error(n):
    return Fraction(n, 1 << 41) + Fraction(n * n, 1 << 52)


def check_bounds(out, ns, ms):
    for i, (n, m) in enumerate(zip(ns, ms)):
        lo, hi, fx = float(out["lo"][i]), float(out["hi"][i]), float(out["fx"][i])
        x = n - Fraction(m, 1 << 40)
        e = bound_error(n)
        assert Fraction(lo) <= x - e and Fraction(hi) >= x + e, (n, m)                       # outward rounding
        assert Fraction(hi) - Fraction(lo) <= 2 * e + 8 * Fraction(math.ulp(float(n))), (n, m)   # and not needlessly wide
        assert fx == float(n) - float(m) * 2.0 ** -40, (n, m)                                 # round to nearest (float(int) is)


def test_depth_bounds_exact(backend):
    """Outward rounding against Fraction, for deficits M up to (2^23 - 1) dd(2^32 - 1), including M above 2^53 that no double
    represents (the _ru / _rd conversions matter there)."""
    rng = random.Random(2)
    ns = list(range(1, 300)) + [(1 << j) + d for j in range(9, 23) for d in (-1, 0, 1)] + [TL_DEF_COVER - 1]
    ns += [rng.randint(300, TL_DEF_COVER - 1) for _ in range(3000)]
    cases = []
    top = dd(K_MAX)
    for n in ns:
        mx = n * top
        cases += [(n, 0), (n, mx), (n, dd(2)), (n, n * dd(3)), (n, rng.randint(0, mx))]
        if mx > 1 << 53:
            m = rng.randint(1 << 53, mx) | 1                    # odd above 2^53: not a double
            cases += [(n, m), (n, (1 << 53) + 1), (n, mx - 1 if mx % 2 == 0 else mx)]
    big = [(n, m) for n, m in cases if m > 1 << 53 and float(m) != m]
    assert len(big) > 1000
    ns_, ms_ = zip(*cases)
    check_bounds(probe_lib.run(backend, cover=ns_, deficit=ms_), ns_, ms_)


def orders(rng, ks, only_ones_first=False):
    """SAM orders of the multiset: random, ascending 1/k, descending 1/k, and the ones first (the rest at random)."""
    ones = [k for k in ks if k == 1]
    rest = [k for k in ks if k != 1]
    rng.shuffle(rest)
    if only_ones_first:
        return dict(ones_first=ones + rest)
    r = list(ks)
    rng.shuffle(r)
    return dict(random=r, ascending=sorted(ks, reverse=True), descending=sorted(ks), ones_first=ones + rest)


def test_depth_bounds_contain_the_reference(backend):
    """The sequential f64 sum of 1/k in every order lies in [lo, hi] with n = count and M = sum of dd(k); for the ones-first orders
    of the big sets it lies outside d_fx +- n 2^-41, so the n^2 term of the bound is needed."""
    rng = random.Random(3)
    pool = [1, 2, 3, 5, 6, 7, 10, 12, 33, 35, 1000, 99991, K_MAX]
    sets = [[1] * 100_000 + [3] * 100_000, [1] * (1 << 20) + [3] * (1 << 20), [1] * (1 << 22) + [3] * ((1 << 22) - 1)]
    sets += [[rng.choice(pool) for _ in range(n)] for n in (2, 40, 1000, 30_000, 300_000)]
    sets += [[rng.choice([1, 3, 7]) for _ in range(200_000)]]
    ns, ms, sums, names = [], [], [], []
    for ks in sets:
        m = sum(c * dd(k) for k, c in Counter(ks).items() if k != 1)
        for name, o in orders(rng, ks, only_ones_first=len(ks) > 1 << 21).items():     # (the 8M set: only its worst order)
            ns.append(len(ks)); ms.append(m); sums.append(seq_sum(o)); names.append((len(ks), name))
    out = probe_lib.run(backend, cover=ns, deficit=ms)
    check_bounds(out, ns, ms)
    wide = 0
    for i, s in enumerate(sums):
        assert out["lo"][i] <= s <= out["hi"][i], names[i]
        if abs(Fraction(s) - (ns[i] - Fraction(ms[i], 1 << 40))) > Fraction(ns[i], 1 << 41):
            wide += 1
    assert wide >= 3                                             # at least the 200k, 2M and 8M ones-first sums need the n^2 term
    i = names.index((200_000, "ones_first"))
    assert abs(sums[i] - float(out["fx"][i])) > 3.5e-7 > 200_000 * 2.0 ** -41


# ---- vote_thresholds -----------------------------------------------------------------------------------------------------------
def bankers(x):
    """misc.rs:208-215 on a double, with Rust's saturating `as u32` and fract = x - trunc(x) (numpy, element-wise, IEEE)."""
    x = np.asarray(x, np.float64)
    rd = np.where(np.isnan(x) | (x <= 0), 0, np.where(x >= 4294967295.0, 4294967295.0, np.trunc(x))).astype(np.uint64)
    fr = x - np.trunc(x)
    up = np.where(fr < 0.5, 0, np.where(fr > 0.5, 1, rd & 1))
    return rd + up.astype(np.uint64)


def thresholds(x, fv, fi, min_depth):
    """pileup.rs:70-72 and the low-depth test: valid threshold, invalid threshold, depth < min_depth."""
    x = np.asarray(x, np.float64)
    return (np.maximum(np.uint64(min_depth), bankers(x * fv)), bankers(x * fi), x < float(min_depth))


def around(centres, ulps=3):
    """Every double within +-ulps ulps of each centre."""
    c = np.asarray(centres, np.float64)
    out = [c]
    up, down = c, c
    for _ in range(ulps):
        up, down = np.nextafter(up, np.inf), np.nextafter(down, -np.inf)
        out += [up, down]
    return np.concatenate(out)


FRACTIONS = [0.0, 0.1, 0.2, 1 / 3, 0.5, 0.7, 0.9, 1.0]
TOP = 1e6          # depths up to 1e6: x * f stays far below 2^31 (saturation at 2^32 - 1 is out of reach of real coverage)


def grid(rng, f):
    """Depths where x * f crosses j + 1/2: all j below 1000, a seeded sample of j up to TOP * f."""
    if f == 0.0:
        return np.zeros(0)
    js = list(range(1000)) + rng.sample(range(1000, int(TOP * f)), 1000)
    return np.array([(j + 0.5) / f for j in js])


def test_vote_thresholds(backend):
    """Equal to the restatement at every double within 3 ulps of a sample of the rounding ties of x * fv and x * fi (all ties below
    1000, 1000 seeded ones up to 1e6 * f) and of the integers (all below 1000, 1000 seeded ones up to 1e6) as min_depth, and monotone along each sorted grid: vt and it never decrease, `low` never turns back on (the vote's shortcut rests on it)."""
    rng = random.Random(4)
    ints = np.array(list(range(0, 1000)) + rng.sample(range(1000, int(TOP)), 1000), np.float64)
    ties = 0
    for a, fv in enumerate(FRACTIONS):
        for b, fi in enumerate(FRACTIONS):
            md = [0, 1, 2, 5, 10, 17, 1000, 999_999][(a + 3 * b) % 8]
            x = np.unique(around(np.concatenate([grid(rng, fv), grid(rng, fi), ints])))
            x = x[x >= 0]
            out = probe_lib.run(backend, x=x, fv=np.full(len(x), fv), fi=np.full(len(x), fi), min_depth=np.full(len(x), md))
            vt, it, low = thresholds(x, fv, fi, md)
            assert np.array_equal(out["vt"], vt), (fv, fi, md)
            assert np.array_equal(out["it"], it), (fv, fi, md)
            assert np.array_equal(out["low"] != 0, low), (fv, fi, md)
            assert np.array_equal(out["br"], bankers(x)), (fv, fi)
            assert (np.diff(out["vt"].astype(np.int64)) >= 0).all() and (np.diff(out["it"].astype(np.int64)) >= 0).all(), (fv, fi)
            assert (np.diff(out["low"].astype(np.int64)) <= 0).all(), (fv, fi, md)
            for f in (fv, fi):
                p = x * f
                ties += int(np.count_nonzero((p - np.trunc(p) == 0.5) & (np.trunc(p) % 2 == 0)))
    assert ties > 1000                                           # exact .5 ties with an even integer part: the rounding that differs
    # the low-depth test at every integer min_depth: x within 3 ulps of m, min_depth = m
    x = around(ints)
    md = np.concatenate([ints] * 7).astype(np.uint32)
    x, md = x[x >= 0], md[x >= 0]
    out = probe_lib.run(backend, x=x, fv=np.full(len(x), 0.5), fi=np.full(len(x), 0.2), min_depth=md)
    assert np.array_equal(out["low"] != 0, x < md.astype(np.float64))
    assert np.array_equal(out["vt"], np.maximum(md.astype(np.uint64), bankers(x * 0.5)))
