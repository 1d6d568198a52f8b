"""The filter's insert-size select on the CPU: filter_dev.h's rounds (tests/filter_select_harness.cpp) against sorting, and the exact
model of tests/filtergen.py against the oracle on the text form of every case."""
import collections
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from tests import filtergen as fg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "filter_select_harness.cpp")
DEPS = [SRC, os.path.join(ROOT, "polypolish_b200", "csrc", "filter_dev.h"), os.path.join(ROOT, "include", "pp_abi.h")]
CASES = fg.cases()
IDS = [c.name for c in CASES]


@pytest.fixture(scope="module")
def H():
    out = os.path.join(ROOT, "build", "filter_select_harness.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS):
        tmp = "%s.%d.tmp" % (out, os.getpid())
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-Wall", "-o", tmp, SRC])
        os.replace(tmp, out)
    L = C.CDLL(out)
    L.h_nearest_rank.restype = C.c_ulonglong
    L.h_nearest_rank.argtypes = [C.c_double, C.c_ulonglong]
    L.h_select.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint32, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    return L


def select(H, values, low, high, owners=1):
    """(low, high, trace) of the harness: trace[round][rank] = (digit, rank inside the bucket, bucket count)."""
    v = np.ascontiguousarray(values, dtype=np.uint32)
    out, tr = np.zeros(2, np.uint32), np.zeros(24, np.uint32)
    H.h_select(v.ctypes.data, len(v), owners, low, high, out.ctypes.data, tr.ctypes.data)
    return int(out[0]), int(out[1]), [[tuple(int(x) for x in tr[(rd * 2 + r) * 3:(rd * 2 + r) * 3 + 3]) for r in range(2)] for rd in range(4)]


def chosen_sizes(case):
    return sorted(fg.unique_sizes(case)[fg.model(case)["orientation"]])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_harness_select_matches_sorting(H, case):
    """filter_dev.h's rounds give sorted(v)[rank - 1] for both ranks, over one owner's histograms and summed over several."""
    v = chosen_sizes(case)
    exp = fg.thresholds(v, case.low, case.high)
    for owners in (1, 3, 8):
        lo, hi, _ = select(H, random.Random(owners).sample(v, len(v)), case.low, case.high, owners)
        assert (lo, hi) == exp, owners


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_harness_walks_the_model_rounds(H, case):
    """The harness picks the digits and bucket positions of the model's radix select, round by round."""
    _, _, tr = select(H, chosen_sizes(case), case.low, case.high)
    assert tr == [[tuple(x) for x in rnd] for rnd in fg.select_trace(case)]


@pytest.mark.parametrize("case", [c for c in CASES if c.digit is not None], ids=[c.name for c in CASES if c.digit is not None])
def test_digit_case_shape(H, case):
    """In round d the two ranks part from their neighbours: one is the first value of its bucket and the other the last, with other
    values in the bucket; the digit of each rank value is not 0 (so a dropped round shows)."""
    _, _, tr = select(H, chosen_sizes(case), case.low, case.high)
    rd = 3 - case.digit
    pos = sorted("first" if r == 1 else "last" if r == c else "inside" for _, r, c in tr[rd])
    assert pos == ["first", "last"] and all(c > 1 for _, _, c in tr[rd]), tr
    assert all(d != 0 for d, _, _ in tr[rd]), tr


def test_harness_select_random_multisets(H):
    rng = random.Random(7)
    for it in range(300):
        n = rng.choice([1, 2, 3, 5, 17, 256, 257, 1000, 5000])
        kind = it % 4
        if kind == 0:
            v = [rng.randint(0, fg.MAX_COORD) for _ in range(n)]
        elif kind == 1:                                  # few distinct values: long tied runs
            pool = [rng.randint(0, fg.MAX_COORD) for _ in range(3)]
            v = [rng.choice(pool) for _ in range(n)]
        elif kind == 2:                                  # values around one digit boundary
            b = 1 << (8 * rng.randint(1, 3))
            v = [b + rng.randint(-3, 2) for _ in range(n)]
        else:
            v = [rng.randint(0, 600) for _ in range(n)]
        low, high = rng.uniform(0.01, 49.99), rng.uniform(50.01, 99.99)
        lo, hi, _ = select(H, v, low, high, rng.choice([1, 2, 5]))
        assert (lo, hi) == fg.thresholds(v, low, high), (n, kind, low, high)


def test_nearest_rank_f64(H):
    """The rank arithmetic in f64, on (p, n) where p / 100 * n is an exact integer and where it is one ulp above one."""
    edges = fg.rank_edge_pairs(1, 2000)
    for key in (("exact", True), ("exact", False), ("ulp", True), ("ulp", False)):
        assert len(edges[key]) > 20, key
        for n, p in edges[key][:400]:
            r = H.h_nearest_rank(p, n)
            assert r == fg.nearest_rank(p, n), (n, p)
            x = p / 100.0 * n
            assert r == (int(x) if key[0] == "exact" else int(x) + 1)
    rng = random.Random(3)
    for _ in range(5000):
        p, n = rng.uniform(0.0001, 99.9999), rng.randint(1, 1 << 40)
        assert H.h_nearest_rank(p, n) == fg.nearest_rank(p, n), (p, n)
    assert [H.h_nearest_rank(p, n) for p, n in ((0.1, 1), (99.9, 1), (0.1, 0), (49.9, 2), (50.1, 2))] == [1, 1, 1, 1, 2]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_model_against_oracle(oracle, tmp_path, case):
    """The model's files, thresholds, pair counts and orientation are the oracle's on the case's SAM texts."""
    t1, t2 = case.texts()
    i1, i2 = tmp_path / "i1.sam", tmp_path / "i2.sam"
    i1.write_bytes(t1)
    i2.write_bytes(t2)
    got = oracle.filter(i1, i2, orientation=case.orientation, low=case.low, high=case.high)
    m = fg.model(case)
    e1, e2 = case.expected_texts(m)
    assert (got["low"], got["high"], got["orientation"], list(got["pairs"])) == (m["low"], m["high"], m["orientation"], m["pairs"])
    assert got["out1"] == e1 and got["out2"] == e2
    assert got["after_count"] == m["n_pass"]
    assert 0 < m["n_pass"] < len(case.recs[0]) + len(case.recs[1])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_cases_are_sharp(case):
    """The correct radix select is the sorted one; each mistake the case is meant to catch changes a threshold and a verdict."""
    assert fg.model(case, None) == fg.model(case)
    for mu in case.sharp_for:
        assert fg.sharp(case, mu), mu


def test_every_mistake_is_caught():
    for mu in fg.MUTATIONS:
        assert sum(fg.sharp(c, mu) for c in CASES) >= 8, mu


def test_probes_sit_on_the_thresholds():
    """Every case has candidates at low - 1, low, high and high + 1 (where those are inserts), passing exactly at low and high."""
    for case in CASES:
        m = fg.model(case)
        want = {x for x in (m["low"] - 1, m["low"], m["high"], m["high"] + 1) if 1 <= x <= fg.MAX_COORD}
        seen = {}
        multi = {n for n, c in collections.Counter(r[0] for r in case.recs[0]).items() if c > 1}
        for i, r in enumerate(case.recs[0]):
            if r[1] != 0 or r[0] not in multi:
                continue
            for s in case.recs[1]:
                if s[0] == r[0] and s[1] == 0:
                    ins = fg.get_insert_size(r[2:], s[2:])
                    if ins in want and fg.get_orientation(r[2:], s[2:]) == m["orientation"]:
                        seen.setdefault(ins, set()).add(m["pass1"][i])
        assert set(seen) == want, case.name
        for ins, verdicts in seen.items():
            assert verdicts == {1 if m["low"] <= ins <= m["high"] else 0}, (case.name, ins)
