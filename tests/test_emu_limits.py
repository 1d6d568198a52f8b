"""The polish kernels past their size limits, on the CPU emulator (tests/emu) against the oracle: long other alleles (hashed
signatures compared against the reads), a compaction chunk too large to stage, read groups that cross 256-alignment blocks and the
in-block scan limit (global-k mode, ghost records of a shard), and depth boundaries with k > 32.  Every case first asserts that it
reaches its limit.  The node and output pools of the emulator never grow, so those repeats are tested on the GPU only
(tests/test_gpu_limits.py)."""
import types

import numpy as np
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import emu_lib, limitgen as lg
from tests.test_emu_polish import check


def pileup_alleles(debug_tsv):
    """(contig, position, allele, count) of every pileup entry of an oracle --debug TSV."""
    out = []
    for row in debug_tsv.decode("latin-1").split("\n")[1:]:
        if not row:
            continue
        c = row.split("\t")
        for e in filter(None, c[6].split(",")):
            a, _, n = e.rpartition("x")
            out.append((c[0], int(c[1]), a, int(n)))
    return out


LONG = [14, 15, 16, 17, 63, 64, 191, 254, 255, 256, 1000, 5000]
LONG8 = [7, 8, 9, 14, 15, 16, 17, 63, 64, 255, 256, 1000]


@pytest.mark.parametrize("kind", ["4bit", "8bit", "huge"])
def test_emu_long_alleles(oracle, tmp_path, kind):
    case = (lg.long_alleles(1, LONG) if kind == "4bit" else lg.long_alleles(2, LONG8, eight_bit=True) if kind == "8bit"
            else lg.long_alleles(3, [16, 300], huge=True))
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams, debug=True, **case.opts)
    # preconditions: the batch's pool, and every allele length at a changed locus (longer than the exact signature)
    p = pp.pack_sams(pp.load_fasta(fa), sams)
    assert p.view.seq_bits == case.facts["seq_bits"]
    lens = {len(a) for _, _, a, n in pileup_alleles(exp["debug_tsv"]) if n >= 5}
    assert set(case.facts["allele_lengths"]) <= lens
    assert max(lens) > (7 if kind == "8bit" else 15) and case.facts["hashed_reads"] > 0
    assert kind == "8bit" or case.facts["fast_walk_reads"] > 0
    assert sum(exp["changed"]) >= len(case.facts["allele_lengths"])
    check(oracle, fa, sams, grid_tiles=2, **case.opts)
    check(oracle, fa, sams, grid_tiles=1, min_depth=1, fraction_invalid=0.1)


def test_emu_unstaged_chunk(oracle, tmp_path):
    """Chunks that emit more than 4096 bytes write straight to the output, one of them across a contig boundary."""
    case = lg.output_growth(4, n_ins=24, ins_len=1000, contig_lens=(3000, 2500))
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams)
    f = pp.load_fasta(fa)
    got = sum(len(l) for l in exp["fasta"].split(b"\n")[1::2])
    assert got == case.facts["total"] < case.facts["G"] + case.facts["G"] // 4 + (1 << 20)       # (the emulator's output buffer)
    assert case.facts["chunk_bytes"][case.facts["boundary_chunk"]] > lg.CP_STAGE
    assert int(f.off[1]) // lg.CHUNK == case.facts["boundary_chunk"] and int(f.off[1]) % lg.CHUNK
    check(oracle, fa, sams, grid_tiles=2)


# (sizes, offset mod 256, first / last in the list, global-k mode).  A record scans the records of its group outside its own block,
# so a group switches modes only if some good record sees more than 8192 of them: never at 8193 (at most 8192 outside), at 8448
# only where a block holds a few of its records, at 9000 always.
GROUPS = [([2, 255, 256, 257, 511, 8192], 0, "first", False), ([8191, 8193], 1, "last", False), ([8448, 511], 255, "first", True),
          ([8448], 0, "last", False), ([9000], 0, "last", True)]


@pytest.mark.parametrize("sizes,offset,where,global_k", GROUPS, ids=["small-0-first", "8191-8193-1-last", "8448-255-first", "8448-0-last",
                                                                      "9000-0-last"])
def test_emu_read_groups(oracle, tmp_path, sizes, offset, where, global_k):
    case = lg.read_groups(21 + offset, sizes, offset=offset, where=where)
    fa, sams = case.write(tmp_path)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    rid = p.arrays()["read_id"]
    groups = dict(lg.group_records(rid))
    for g in case.facts["groups"]:
        assert groups[g["start"]] == g["size"] and g["start"] % 256 == offset
    first, last = case.facts["groups"][0], case.facts["groups"][-1]
    if where == "first":
        assert first["start"] == offset
    else:
        assert last["start"] + last["size"] == p.view.n_aln
    for opts in (dict(), dict(max_errors=0), dict(careful=True)):
        r = check(oracle, fa, sams, grid_tiles=2, **opts)
        assert r["global_k"] == lg.expect_global_k(rid, lg.record_good(case.sam_texts, **opts)), opts
    assert lg.expect_global_k(rid, lg.record_good(case.sam_texts)) == global_k


def test_emu_ghost_records_count_towards_k(oracle, tmp_path):
    """A group of 9,000 records over three contigs, sharded two ways: every shard holds the other shard's records as ghosts, which
    count towards k (k_classify_multi in global-k mode) but do not scatter."""
    case = lg.read_groups(7, [9000], offset=1, where="first")
    fa, sams = case.write(tmp_path)
    exp = oracle.polish(fa, sams)
    want = exp["fasta"].split(b"\n")[1::2]
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    sh = api.Shards(f.view, p.view, 2)
    n_ghost = 0
    for s in range(2):
        c, a, cmap, n_home = sh.get(s)
        n_ghost += a.n_aln - n_home
        off = np.ctypeslib.as_array(api.C.cast(c.off, api.C.POINTER(api.C.c_uint64)), shape=(c.n_contigs + 1,)).copy()
        r = emu_lib.polish(types.SimpleNamespace(view=c, off=off), types.SimpleNamespace(view=a), grid_tiles=2)
        assert r["global_k"]
        assert r["sequences"] == [want[i] for i in cmap]
        assert r["changed"] == [exp["changed"][i] for i in cmap]
        for got, i in zip(r["total_depth"], cmap):
            assert abs(got - exp["total_depth"][i]) <= 1e-9 * max(1.0, exp["total_depth"][i])
    assert n_ghost > 9000
    sh.close()


def chunk_cuts(text, threads, min_chunk):
    """Byte offsets where the threaded packer cuts a file into chunks (sam_pack.cpp pack_text_parallel): every
    max(min_chunk, size / threads + 1) bytes, moved on to the next line start."""
    n = len(text)
    want = max(min_chunk, n // threads + 1)
    cut = [0]
    while cut[-1] < n:
        nxt = cut[-1] + want
        if nxt >= n:
            break
        q = text.find(b"\n", nxt)
        cut.append(q + 1 if q >= 0 else n)
    return cut[1:]


def test_parallel_pack_rejoins_a_big_group(tmp_path):
    """The 20,000-record group parsed in chunks of 64 KB (it spans several chunk seams): the same arrays as the sequential packer."""
    case = lg.read_groups(9, [20_000], offset=0, where="first", filler=200)
    fa, sams = case.write(tmp_path)
    text = case.sam_texts[0].encode("latin-1")
    g = case.facts["groups"][0]
    line_start = [0]
    for line in text.split(b"\n"):
        line_start.append(line_start[-1] + len(line) + 1)
    lo, hi = line_start[g["start"]], line_start[g["start"] + g["size"]]
    assert len(text) >= 2 * (1 << 16)                                       # (smaller files are parsed in one piece)
    assert sum(1 for c in chunk_cuts(text, 4, 1 << 16) if lo < c < hi) >= 3   # seams inside the group
    out = []
    for threads, chunk in ((1, 1 << 30), (4, 1 << 16)):
        f = pp.load_fasta(fa)
        p = api.Packed(f)
        p.set_threads(threads, chunk)
        for s in sams:
            p.add_file(s)
        p.finish()
        out.append((f, p, p.arrays()))
    a1, a2 = out[0][2], out[1][2]
    assert max(n for _, n in lg.group_records(a1["read_id"])) == 20_000
    for k, v in a1.items():
        assert np.array_equal(v, a2[k]) if isinstance(v, np.ndarray) else v == a2[k], k


# k of the alignments over the probed position: the exact sum is the boundary (5 = min_depth, or 7 with fraction_invalid 0.5 at an
# allele seen 3 times); a seeded search finds one SAM order whose f64 sum is the boundary and one whose sum is one ulp below
K34_MIN = [1] * 4 + [34] * 34
K35_HALF = [1] * 6 + [35] * 35
K32_33 = [1] * 2 + [32] * 32 + [33] * 33 + [6] * 6
BOUNDARY_SETS = [(K34_MIN, 5.0), (K35_HALF, 7.0), (K32_33, 5.0)]


@pytest.mark.parametrize("ks,target", BOUNDARY_SETS, ids=["k34-min", "k35-half", "k32-k33-min"])
def test_emu_depth_boundary_past_the_table(oracle, tmp_path, ks, target):
    """k > 32: the ordered depth walk divides (__ddiv_rn) instead of reading its 1/k table."""
    half = target == 7.0
    opts = dict(min_depth=1, fraction_valid=0.9, fraction_invalid=0.5) if half else dict(min_depth=5)
    on, below = lg.boundary_orders(5, ks, target)
    for ks_, want in ((on, 1), (below, 0)):
        d = tmp_path / ("on" if want else "below")
        d.mkdir()
        fa, sam, P = lg.boundary_case(d, ks_, x_reads=3 if half else 0)
        exp = oracle.polish(fa, [sam], debug=True, **opts)
        row = exp["debug_tsv"].split(b"\n")[1 + P].split(b"\t")
        assert row[:2] == [b"probe", str(P).encode()] and exp["changed"][0] == want
        r = check(oracle, fa, [sam], grid_tiles=1, **opts)
        assert r["changed"][0] == want
