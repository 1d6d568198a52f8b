"""The depth runs (--depth-bedgraph) of the emulated kernels (tests/emu): k_tile's depth mode under the strict model of the chunk ring,
then k_status_heads<u64> and k_status_runs<u64>, against the run-length encoding of the oracle's --debug depth column, byte for byte;
and depth_tenths with the host's depth text against snprintf("%.1f").  CPU only."""
import math

import numpy as np
import pytest

import polypolish_b200 as pp
from tests import depthgen, emu_lib, endgen, fuzzgen, statusgen, walkgen


# ---- depth_tenths and the host's text ----------------------------------------------------------------------------------------------
def check_tenths(x):
    x = np.asarray(x, dtype=np.float64)
    t, bad = emu_lib.depth_tenths(x)
    assert bad == len(x), "depth_tenths(%r) = %d, snprintf says %s" % (x[bad], t[bad], "%.1f" % x[bad])
    assert t.tolist() == [depthgen.tenths(v) for v in x.tolist()]


def neighbours(x):
    """x and the doubles either side of it (depths are never negative)"""
    y = np.concatenate([np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf)])
    return y[y >= 0]


def test_tenths_twentieths():
    """Every n/20 up to 10^5 (all the decimal ties x.x5 and the tenths), each with the doubles either side of it."""
    x = neighbours(np.arange(0, 2_000_001, dtype=np.float64) / 20.0)
    t, bad = emu_lib.depth_tenths(x)
    assert bad == len(x), "depth_tenths(%r) = %d, snprintf says %s" % (x[bad], t[bad], "%.1f" % x[bad])


def test_tenths_exact_ties():
    """x.25 and x.75 are exact in binary: round half to even gives x.2 and x.8, never x.3 or x.7."""
    x = np.array([n + f for n in (0, 1, 2, 7, 100, 12345, 2 ** 31, 2 ** 32 - 1) for f in (0.25, 0.75)], dtype=np.float64)
    check_tenths(neighbours(x))
    t, _ = emu_lib.depth_tenths(np.array([0.25, 0.75, 1.25, 1.75]))
    assert t.tolist() == [2, 8, 12, 18]


def test_tenths_zero_and_large():
    """0, values near 2^32 (the largest cover) and near 2^36 / 10 tenths."""
    x = [0.0, 5e-324, 1e-300, 0.04999999999999999, 0.05, 0.95]
    x += [2.0 ** 32 + d for d in (-1.0, -0.95, -0.75, -0.5, -0.25, -0.05, 0.0, 0.05, 0.25, 0.75, 1.0)]
    x += [2.0 ** 36 / 10 + d for d in (-1.0, -0.45, -0.25, 0.0, 0.25, 0.45, 0.75)]
    check_tenths(neighbours(np.array(x)))


def test_tenths_random():
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.uniform(0, 1, 200_000), rng.uniform(0, 1000, 200_000), rng.uniform(0, 2.0 ** 32, 200_000),
                        np.exp(rng.uniform(-40, 22, 200_000))])
    check_tenths(x)


def test_depth_text():
    """The host formats the key with integers only: tenths / 10, ".", tenths % 10 - what snprintf("%.1f") prints of that many tenths."""
    keys = [0, 1, 9, 10, 11, 99, 100, 101, 12345, 10 ** 10 + 7, (1 << 36) - 1]
    want = b"".join(b"%.1f\n" % (k / 10) for k in keys[:-2]) + b"1000000000.7\n6871947673.5\n"
    assert emu_lib.depth_text(np.array(keys, np.uint64)) == want


# ---- the emulated kernels against the oracle ---------------------------------------------------------------------------------------
def check_depth(oracle, fa, sams, grid_tiles=2, with_changes=False, with_status=False, **opts):
    exp = oracle.polish(fa, sams, debug=True, **opts)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams, careful=opts.get("careful", False))
    r = emu_lib.polish(f, p, grid_tiles=grid_tiles, depth=True, changes=with_changes, status=with_status, **opts)
    assert "error" not in r, r
    assert emu_lib.fasta_bytes(f, r["sequences"]) == exp["fasta"]
    assert r["bedgraph"] == depthgen.bedgraph_from_debug_tsv(exp["debug_tsv"])
    assert sum(int(x.split(b"\t")[2]) - int(x.split(b"\t")[1]) for x in r["bedgraph"].splitlines()) == int(f.off[-1])
    if with_status:
        assert r["bed"] == statusgen.bed_from_debug_tsv(exp["debug_tsv"])
    # depth off: the same FASTA and statistics.  The total depth adds the walk's sum where depth mode walked and the fixed-point
    # estimate elsewhere (within n 2^-41 of each other per position), in atomics of no fixed order: equal to rounding
    plain = emu_lib.polish(f, p, grid_tiles=grid_tiles, **opts)
    assert plain["sequences"] == r["sequences"] and plain["changed"] == r["changed"] and plain["zero_depth"] == r["zero_depth"]
    assert all(math.isclose(a, b, rel_tol=1e-9, abs_tol=1e-9) for a, b in zip(plain["total_depth"], r["total_depth"])), (plain["total_depth"], r["total_depth"])
    return r, exp


def test_bedgraph_from_debug_tsv():
    tsv = (b"name\tpos\tbase\tdepth\tinvalid\tvalid\tcounts\tstatus\tnew\n"
           b"a\t0\tA\t0.0\t0\t5\t\tlow_depth\tA\na\t1\tA\t0.0\t0\t5\t\tlow_depth\tA\na\t2\tC\t9.0\t2\t5\tC:9\tkept\tC\n"
           b"b\t0\tG\t9.0\t2\t5\tG:9\tkept\tG\nb\t1\tG\t9.0\t2\t5\tG:9\tkept\tG\nb\t2\tG\t9.5\t2\t5\tG:9\tkept\tG\n")
    assert depthgen.bedgraph_from_debug_tsv(tsv) == b"a\t0\t2\t0.0\na\t2\t3\t9.0\nb\t0\t2\t9.0\nb\t2\t3\t9.5\n"


@pytest.mark.parametrize("seed", [100, 101, 104, 107, 112, 116, 121, 133, 140, 152, 164, 175])
def test_emu_depth_fuzz(oracle, tmp_path, seed):
    case = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0)
    fa, sams = case.write(tmp_path)
    try:
        oracle.polish(fa, sams, **case.opts)
    except Exception:
        pytest.skip("the reference rejects this input")
    check_depth(oracle, fa, sams, with_changes=seed % 2 == 1, with_status=seed % 3 == 0, **case.opts)


@pytest.mark.parametrize("seed", [300, 303, 307])
def test_emu_depth_deep_multimap(oracle, tmp_path, seed):
    """Non-dyadic k everywhere: most positions print from the bound, the rest from the ordered walk."""
    case = fuzzgen.make_case(seed, n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False))
    fa, sams = case.write(tmp_path)
    check_depth(oracle, fa, sams, with_status=seed == 303, **case.opts)


@pytest.mark.parametrize("name", sorted(depthgen.CASES) + sorted(depthgen.DYADIC))
def test_emu_depth_print_boundary(oracle, tmp_path, name):
    """P's depth prints one tenth in one SAM order and the tenth below in the other: the oracle's texts differ, the base does not,
    and the bound's lower end prints the wrong text for the "on" order, which only the depth walk rule opens."""
    on, off, spec = depthgen.case_pair(name)
    assert on.facts["tenths_lo"] != on.facts["tenths_ref"]
    assert on.facts["seq_bits"] == (8 if spec["eight_bit"] else 4)
    fastas = []
    for c, want in ((on, spec["on"]), (off, spec["off"])):
        d = tmp_path / ("on" if c is on else "off")
        d.mkdir()
        fa, sams = c.write(d)
        r, exp = check_depth(oracle, fa, sams, grid_tiles=1, **c.opts)
        assert depthgen.depth_at(exp["debug_tsv"], "probe", spec["P"]) == want
        fastas.append(exp["fasta"])
    assert fastas[0] == fastas[1]


@pytest.mark.parametrize("name", ["close-two", "depth-long", "multiple-three"])
def test_emu_depth_status_cases(oracle, tmp_path, name):
    """statusgen's boundary cases with both reports recorded in one call."""
    for c in statusgen.case_pair(name)[:2]:
        d = tmp_path / str(id(c))
        d.mkdir()
        fa, sams = c.write(d)
        check_depth(oracle, fa, sams, grid_tiles=1, with_status=True, **c.opts)


@pytest.mark.parametrize("name", ["W1-two", "W3-long", "W4-tile-start", "W5-contig-border", "W8-three-print"])
def test_emu_depth_walk_cases(oracle, tmp_path, name):
    """walkgen's merge-order cases: the walk's sum, not a concatenation of its runs, is what is printed."""
    lay, ks, target, side, opts, n_x, per_run, _ = walkgen.CASES[name]
    layout = walkgen.LAYOUTS[lay]()
    on, _ = walkgen.run_orders(5, ks, target, len(layout["runs"]), side=side, min_per_run=per_run)
    c = walkgen.walk_case(5, on, layout, x_reads=n_x, opts=opts)
    fa, sams = c.write(tmp_path)
    check_depth(oracle, fa, sams, grid_tiles=1, **c.opts)


@pytest.mark.parametrize("name,case", [("E", lambda: endgen.edges(41)), ("E8", lambda: endgen.edges(41, eight_bit=True))])
def test_emu_depth_contig_ends(oracle, tmp_path, name, case):
    """Contigs of 1-9 bp, contig starts at every residue mod 32, contigs no read covers (one 0.0 run each)."""
    c = case()
    fa, sams = c.write(tmp_path)
    r, _ = check_depth(oracle, fa, sams, with_status=True, **c.opts)
    assert r["bedgraph"].count(b"\n") >= len(c.facts["lens"])


@pytest.mark.parametrize("seed", [101, 116])
@pytest.mark.parametrize("min_depth", [0, 1, 2, 5])
def test_emu_depth_min_depth(oracle, tmp_path, seed, min_depth):
    """The depth report does not read the options, but the vote's shortcuts and walks do."""
    case = fuzzgen.make_case(seed)
    fa, sams = case.write(tmp_path)
    check_depth(oracle, fa, sams, **dict(case.opts, min_depth=min_depth))
