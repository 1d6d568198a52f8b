"""Read selection on the GPU against the oracle: the cases of tests/test_emu_select.py, each loaded once through both routes (pack_sams
+ upload, and the device tokeniser) and polished resident under its whole option grid, in a fixed order that ends with the first set
again, the change report on every other call.  Errors name the record the model names, and each call after a failed one is checked
like any other.  Case C runs on a context in global-k mode from its first call on; case B also crosses the alignment index where
k_goodk's grid-stride loop wraps on this device.  polish_packed, polish_files (both parsers, --debug, --changes) and
polish_files_multi (2 and 3 contexts: read groups whose records lie on contigs of different contexts) run a subset of the sets."""
import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import limitgen as lg, selectgen as sg
from tests.test_emu_ends import PANIC
from tests.test_emu_select import CASES, aligned_rows, load_careful, opt_sets, reference_message, run_oracle
from tests.test_gpu_changes import changed_rows
from tests.test_gpu_ends import check_message
from tests.test_gpu_limits import check_files, fasta_of, same_stats

pytestmark = pytest.mark.gpu
PR_THREADS = 256


@pytest.fixture(scope="module")
def ctx():
    import __graft_entry__ as g
    g.build()
    c = pp.Context(0)
    yield c
    c.close()


def goodk_wrap():
    """The first alignment index k_goodk's grid-stride loop reaches in its second round: grid = sm_count * 8 blocks of 256."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * PR_THREADS


def make(name):
    if name == "B":
        return sg.block_edges(12, wrap=goodk_wrap())
    return CASES[name]()


# the library's text for a device error (polish_kernels.cu err_text), by the model's kind
DEVICE_TEXT = {"unknown_contig": "query name in SAM but not in assembly", "seq_mismatch": "CIGAR string does not match read sequence",
               "bad_op": "unexpected character (other than M, =, X, I or D) in CIGAR string - did you use BWA MEM to generate your "
                         "alignments?",
               "oob": "alignment extends past the end of its reference sequence", "noseq": "no alignments for read contain sequence"}


def device_message(kind, aln):
    return "%s (alignment %d)" % (DEVICE_TEXT[kind], aln)


def check_changes(f, rows, debug_tsv):
    want = []
    for x in changed_rows(debug_tsv).split(b"\n")[1:-1]:
        cols = x.split(b"\t")
        want.append((int(f.off[f.names.index(cols[0].decode())]) + int(cols[1]), cols[8].decode()))
    assert [(x["pos"], x["new_base"]) for x in rows] == want


def resident_grid(ctx, oracle, case, fa, sams, f, grid, launches):
    """Every option set of `grid` on the context's resident dataset, the change report on odd calls."""
    for i, opts in enumerate(grid):
        m = lg.record_good(case.sam_texts, contigs=case.contigs, detail=True, **opts)
        changes = i % 2 == 1
        if m["error"]:
            with pytest.raises(pp.PolypolishError) as e:
                ctx.polish_resident(changes=changes, **opts)
            assert e.value.msg == device_message(*m["error"]), (i, opts, e.value.msg)
            assert reference_message(aligned_rows(case.sam_texts), *m["error"]) == run_oracle(oracle, fa, sams, opts)["error"]
            continue
        r = ctx.polish_resident(changes=changes, **opts)
        exp = oracle.polish(fa, sams, debug=changes, **opts)
        assert fasta_of(f, r["sequences"]) == exp["fasta"], (i, opts)
        same_stats(r, exp)
        assert r["n_aln_used"] == m["used"]
        assert r["timing"]["launches"] == launches(opts), (i, opts)
        if changes:
            check_changes(f, r["changes"], exp["debug_tsv"])


@pytest.mark.parametrize("route", ["upload", "tokenise"])
@pytest.mark.parametrize("name", list(CASES))
def test_resident_grid(ctx, oracle, tmp_path, name, route):
    case = make(name)
    fa, sams = case.write(tmp_path)
    f = pp.load_fasta(fa)
    careful = load_careful(name)
    p = None
    if route == "upload":
        p = pp.pack_sams(f, sams, careful=careful)
        ctx.upload(f.view, p.view)
    else:
        assert ctx.tokenise(f, sams, careful=careful)[0] == api.PP_OK
    grid = opt_sets(name) + [opt_sets(name)[0]]
    if name == "B":
        assert case.facts["n_aln"] > case.facts["wrap"]
        g = case.facts["groups"][-1]
        assert g["start"] < case.facts["wrap"] < g["start"] + g["size"]
    # C: the first call switches the context to global-k mode (k_classify_multi: 4 launches) and it stays there for every later call
    resident_grid(ctx, oracle, case, fa, sams, f, grid, lambda opts: 4 if name == "C" else 3)
    if p is not None:
        p.close()


SUBSET = [0, 2, 6]


@pytest.mark.parametrize("name", ["A", "B", "C", "D"])
def test_packed_and_files(ctx, oracle, tmp_path, name):
    case = CASES[name]()
    fa, sams = case.write(tmp_path)
    f = pp.load_fasta(fa)
    p = pp.pack_sams(f, sams)
    for j in SUBSET + ([1, 3, 5, 7] if name == "D" else []):
        opts = opt_sets(name)[j]
        m = lg.record_good(case.sam_texts, contigs=case.contigs, detail=True, **opts)
        d = tmp_path / ("o%d" % j)
        d.mkdir()
        if m["error"]:
            msg = reference_message(aligned_rows(case.sam_texts), *m["error"])
            with pytest.raises(pp.PolypolishError) as e:
                ctx.polish_packed(f.view, p.view, **opts)
            assert e.value.error_aln == m["error"][1]
            for parser in (0, 1):
                ctx.set_parser(parser)
                try:
                    with pytest.raises(pp.PolypolishError) as e:
                        ctx.polish_files(fa, sams, **opts)
                finally:
                    ctx.set_parser(0)
                check_message(e.value.msg, msg, PANIC.match(msg))
            continue
        r = ctx.polish_packed(f.view, p.view, **opts)
        exp = check_files(ctx, oracle, d, fa, sams, **opts)
        assert fasta_of(f, r["sequences"]) == exp["fasta"]
        same_stats(r, exp)
    p.close()


@pytest.mark.parametrize("name", ["A", "C"] + ["E-" + v for v in sg.NOSEQ_VARIANTS])
def test_multi_contexts(oracle, tmp_path, name):
    """2 and 3 contexts on one device, both parsers: a group's records on other contexts' contigs are ghosts there, which count
    towards k and make the group multi-record for --careful.  Case E loads with --careful as the call does, so its groups without
    SEQ are skipped (or the earlier group's error is raised)."""
    case = CASES[name]()
    fa, sams = case.write(tmp_path)
    grid = [dict(careful=True), dict(max_errors=256, careful=True)] if name.startswith("E") else [sg.OPTS[j] for j in SUBSET]
    for opts in grid:
        m = lg.record_good(case.sam_texts, contigs=case.contigs, detail=True, **opts)
        exp = run_oracle(oracle, fa, sams, opts)
        for n in (2, 3):
            for parser in (0, 1):
                if m["error"]:
                    with pytest.raises(pp.PolypolishError) as e:
                        api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser, **opts)
                    assert e.value.msg == exp["error"], (n, parser, opts)
                else:
                    assert api.polish_files_multi(fa, sams, devices=[0] * n, parser=parser, **opts) == exp["fasta"], (n, parser, opts)
    if not name.startswith("E"):                             # groups with records on several contigs, so on several contexts
        rows = aligned_rows(case.sam_texts)
        m = lg.record_good(case.sam_texts, contigs=case.contigs, detail=True)
        assert sum(1 for a, s in m["groups"] if s > 1 and len({rows[i][2] for i in range(a, a + s)}) > 1) > 10
