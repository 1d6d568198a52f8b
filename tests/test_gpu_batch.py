"""`polypolish batch` / pp_batch_files on the GPU: a mixed batch of whole jobs gives, job for job, the oracle's FASTA and reports and
the log of the job's own call, over 1, 2 and 3 contexts on one device; no per-job setting leaks from one job into the next; a failing
job fails alone with its own call's message; the CLI's files and stderr blocks are those of the single commands, in manifest order."""
import os
import re
import subprocess

import pytest

import polypolish_b200 as pp
from polypolish_b200 import api
from tests import depthgen, fuzzgen, statusgen, vcfgen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")
REPORTS = ("debug", "changes", "status", "vcf", "depth_bedgraph")
CLI_FLAG = dict(debug="--debug", changes="--changes", status="--status-bed", vcf="--vcf", depth_bedgraph="--depth-bedgraph")
OPT_FLAG = dict(fraction_invalid="-i", fraction_valid="-v", max_errors="-m", min_depth="-d")


@pytest.fixture(scope="module", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def changed_rows(debug_tsv):
    lines = debug_tsv.split(b"\n")
    return b"\n".join([lines[0]] + [x for x in lines[1:] if x.split(b"\t")[7:8] == [b"changed"]]) + b"\n"


def expected_report(kind, fa, debug_tsv):
    return {"debug": lambda: debug_tsv, "changes": lambda: changed_rows(debug_tsv), "status": lambda: statusgen.bed_from_debug_tsv(debug_tsv),
            "vcf": lambda: vcfgen.vcf_from_debug(fa, debug_tsv), "depth_bedgraph": lambda: depthgen.bedgraph_from_debug_tsv(debug_tsv)}[kind]()


def log_lines(text):
    """A log without its timing lines (they differ from run to run) and the CLI's start / end lines."""
    timing = ("SAM tokeniser", "GPU job", "read groups exchanged", "filter over", "device", "  phases", "Starting", "[timing]", "Finished")
    return [x for x in text.splitlines() if x and not x.startswith(timing)]


def eight_bit(case_dir, fa, sams):
    """The first long SEQ of the first SAM file gets a '.', which only the 8-bit pool holds."""
    text = open(sams[0], "rb").read().split(b"\n")
    for i, line in enumerate(text):
        c = line.split(b"\t")
        if len(c) > 10 and not line.startswith(b"@") and len(c[9]) > 20:
            c[9] = c[9][:10] + b"." + c[9][11:]
            text[i] = b"\t".join(c)
            break
    open(sams[0], "wb").write(b"\n".join(text))


@pytest.fixture(scope="module")
def mixed(tmp_path_factory, oracle):
    """The inputs of a mixed batch and what each job must give: (name, job without output, expected FASTA, {report: bytes}).  Every
    job's options and reports differ from its neighbours', so that a setting left behind by one job would change the next one."""
    d = tmp_path_factory.mktemp("batch_inputs")
    cases = []

    def add(name, kind, fa, sams, opts, reports=(), debug_exp=None, **extra):
        exp = oracle.polish(fa, sams, debug=True, **opts) if debug_exp is None else debug_exp
        job = dict(kind=kind, assembly=fa, **opts, **extra)
        if kind == "polish":
            job["sams"] = sams
        rep = {}
        for r in reports:
            job[r] = r
            rep[r] = expected_report(r, fa, exp["debug_tsv"])
        cases.append((name, job, exp["fasta"], rep))

    def case_dir(name):
        p = d / name
        p.mkdir()
        return p

    # fuzzgen: 8-bit (exotic SEQ) and 4-bit pools, a deep multi-map case
    for seed in (100, 101, 300):
        kw = dict(n_contigs=2, contig_len=(200, 400), depth=(150, 300), multimap=0.8, opts=dict(careful=False)) if seed >= 300 else {}
        c = fuzzgen.make_case(seed, exotic=0.5 if seed % 4 == 0 else 0.0, **kw)
        fa, sams = c.write(case_dir("fuzz%d" % seed))
        add("fuzz%d" % seed, "polish", fa, sams, dict(c.opts), reports=("changes", "status") if seed == 101 else ())
    # --careful with every other option away from its default, on a synthetic isolate with an 8-bit read
    syn = api.Synth(seed=21, n_contigs=2, contig_len=15_000, depth=40, draft_error_rate=2e-3)
    sd = case_dir("synth")
    fa, sams = syn.write(sd)
    eight_bit(sd, fa, sams)
    add("careful8", "polish", fa, sams, dict(careful=True, fraction_invalid=0.1, fraction_valid=0.6, max_errors=5, min_depth=3),
        reports=("vcf", "depth_bedgraph"))
    add("default8", "polish", fa, sams, {})
    # every report of polish, --debug included
    add("debug", "polish", fa, sams, dict(min_depth=4), reports=REPORTS)
    # no SAM files
    add("nosam", "polish", fa, [], {}, reports=("status",))
    # filter-polish with the filtered SAM files written
    syn2 = api.Synth(seed=22, n_contigs=3, contig_len=10_000, depth=50, draft_error_rate=1e-3)
    fd = case_dir("filter")
    fa2, sams2 = syn2.write(fd)
    ef = oracle.filter(sams2[0], sams2[1])
    f1, f2 = fd / "oracle_f1.sam", fd / "oracle_f2.sam"
    f1.write_bytes(ef["out1"])
    f2.write_bytes(ef["out2"])
    exp = oracle.polish(fa2, [f1, f2], debug=True, min_depth=3)
    add("filterpolish", "filter-polish", fa2, None, dict(min_depth=3), reports=("changes", "depth_bedgraph"), debug_exp=exp,
        in1=sams2[0], in2=sams2[1], out1="out1", out2="out2")
    cases[-1][3].update(out1=ef["out1"], out2=ef["out2"])
    return cases


def with_outputs(cases, out_dir):
    """The jobs with every output file (FASTA, reports, filtered SAM) under out_dir/<case name>."""
    jobs = []
    for name, job, _, rep in cases:
        j = dict(job)
        (out_dir / name).mkdir(parents=True, exist_ok=True)
        for key in rep:
            j[key] = out_dir / name / key
        j["output"] = out_dir / name / "polished.fasta"
        jobs.append(j)
    return jobs


def check_outputs(cases, out_dir):
    for name, _, fasta, rep in cases:
        got = sorted(os.listdir(out_dir / name))
        assert got == sorted(["polished.fasta"] + list(rep)), (name, got)        # nothing more: no report leaked into this job
        assert (out_dir / name / "polished.fasta").read_bytes() == fasta, name
        for key, want in rep.items():
            assert (out_dir / name / key).read_bytes() == want, (name, key)


def single_call(ctx, job, verbose=True):
    """The job through its own file-level call on ctx: (FASTA, stderr log) or the PolypolishError."""
    j = {k: v for k, v in job.items() if k not in ("kind", "output")}
    if job["kind"] == "polish":
        return ctx.polish_files(j.pop("assembly"), j.pop("sams"), verbose=verbose, **j)
    return ctx.filter_polish_files(j.pop("assembly"), j.pop("in1"), j.pop("in2"), verbose=verbose, **j)


@pytest.mark.parametrize("n_ctx", [1, 2, 3])
def test_mixed_batch(mixed, tmp_path, capfd, n_ctx):
    """Every job's FASTA and reports are the oracle's, and its log is its own call's, whichever context ran it."""
    ctxs = [pp.Context(0) for _ in range(n_ctx)]
    try:
        res = api.batch(with_outputs(mixed, tmp_path / "batch"), contexts=ctxs, verbose=True)
        assert capfd.readouterr().err == ""                          # every line of the library went into the results
        assert [r["ok"] for r in res] == [True] * len(mixed), [r["error"] for r in res]
        assert all(r["error"] is None and r["rc"] == 0 and r["wall_ms"] > 0 for r in res)
        assert all(0 <= r["context"] < n_ctx for r in res)
        check_outputs(mixed, tmp_path / "batch")
        # the single call's log, on a context of the batch
        for (name, job, fasta, rep), r in zip(mixed, res):
            one = with_outputs([(name, job, fasta, rep)], tmp_path / "single")[0]
            assert single_call(ctxs[-1], one) == fasta
            assert log_lines(r["log"]) == log_lines(capfd.readouterr().err), name
            assert r["log"].endswith("\n") and "Polishing " in r["log"]
    finally:
        for c in ctxs:
            c.close()


def test_state_does_not_leak(mixed, tmp_path):
    """The same jobs in reverse order, and every job twice in one batch, write the same bytes; a report-less job after a job with
    every report writes none (check_outputs lists each job's directory)."""
    with pp.Context(0) as c:
        fwd = api.batch(with_outputs(mixed, tmp_path / "fwd"), contexts=[c])
        rev = api.batch(with_outputs(mixed[::-1], tmp_path / "rev"), contexts=[c])
        twice = [(n + "_again" if i else n, j, f, r) for n, j, f, r in mixed for i in (0, 1)]
        tw = api.batch(with_outputs(twice, tmp_path / "twice"), contexts=[c], parser=1)     # and with the host parser throughout
    assert all(r["ok"] for r in fwd + rev + tw)
    for d in ("fwd", "rev"):
        check_outputs(mixed, tmp_path / d)
    check_outputs(twice, tmp_path / "twice")
    for name, *_ in mixed:
        for f in os.listdir(tmp_path / "fwd" / name):
            assert (tmp_path / "twice" / name / f).read_bytes() == (tmp_path / "twice" / (name + "_again") / f).read_bytes()


@pytest.fixture(scope="module")
def failing(mixed, tmp_path_factory):
    """Three failing jobs (a missing SAM file, an RNAME the assembly lacks, -i >= -v) between good ones."""
    d = tmp_path_factory.mktemp("failing")
    name, job, fasta, _ = [c for c in mixed if c[0] == "default8"][0]
    bad_sam = d / "unknown_rname.sam"
    lines = []
    for line in open(job["sams"][0], "rb").read().split(b"\n"):
        c = line.split(b"\t")
        if len(c) > 10 and not line.startswith(b"@") and c[2] != b"*":
            c[2] = b"no_such_contig"
        lines.append(b"\t".join(c))
    bad_sam.write_bytes(b"\n".join(lines))
    bad = [("missing_sam", dict(job, sams=[job["sams"][0], d / "missing.sam"])),
           ("unknown_rname", dict(job, sams=[bad_sam])),
           ("invalid_fractions", dict(job, fraction_invalid=0.5, fraction_valid=0.5))]
    good = [c for c in mixed if c[0] in ("fuzz101", "debug", "filterpolish", "nosam")]
    order = [good[0], bad[0], good[1], bad[1], good[2], bad[2], good[3]]
    return order, {n for n, _ in bad}


def test_failing_jobs(failing, tmp_path):
    """A failing job carries exactly its own call's error, creates no FASTA, and changes nothing for the others."""
    order, bad = failing
    cases = [(c[0], c[1], c[2] if len(c) > 2 else None, c[3] if len(c) > 3 else {}) for c in order]
    with pp.Context(0) as c1, pp.Context(0) as c2:
        res = api.batch(with_outputs(cases, tmp_path / "b"), contexts=[c1, c2], verbose=True)
        for (name, job, fasta, rep), r in zip(cases, res):
            if name not in bad:
                assert r["ok"], (name, r["error"])
                continue
            with pytest.raises(pp.PolypolishError) as e:
                single_call(c1, job, verbose=False)
            assert (r["ok"], r["rc"], r["error"]) == (False, e.value.code, e.value.msg), name
            assert not (tmp_path / "b" / name / "polished.fasta").exists()
    assert [n for (n, *_), r in zip(cases, res) if not r["ok"]] == [n for n, *_ in cases if n in bad]
    check_outputs([c for c in cases if c[0] not in bad], tmp_path / "b")


def cli_line(job, out_dir, name, rep):
    """A manifest line (and the same command line on its own) for a job, its outputs under out_dir/name."""
    (out_dir / name).mkdir(parents=True, exist_ok=True)
    args = [job["kind"]]
    for k, flag in OPT_FLAG.items():
        if k in job:
            args += [flag, str(job[k])]
    if job.get("careful"):
        args.append("--careful")
    for k in rep:
        if k in CLI_FLAG:
            args += [CLI_FLAG[k], str(out_dir / name / k)]
    if job["kind"] == "filter-polish":
        args += ["--in1", str(job["in1"]), "--in2", str(job["in2"]), "--out1", str(out_dir / name / "out1"), "--out2", str(out_dir / name / "out2")]
        args.append(str(job["assembly"]))
    else:
        args += [str(job["assembly"])] + [str(s) for s in job["sams"]]
    return args


def test_cli_batch(mixed, failing, tmp_path):
    """`polypolish batch` writes, job for job, the bytes of the single command; stderr has a start line, one block per job in
    manifest order (header, the single command's log, Finished! / Error:), a closing count; --quiet keeps only the failed jobs."""
    order, bad = failing
    cases = [(c[0], c[1], c[2] if len(c) > 2 else None, c[3] if len(c) > 3 else {}) for c in order]
    lines, singles = [], []
    for name, job, _, rep in cases:
        args = cli_line(job, tmp_path / "batch", name, rep)
        lines.append(" ".join(args + ["--output", str(tmp_path / "batch" / name / "polished.fasta")]))
        singles.append(cli_line(job, tmp_path / "single", name, rep))
    manifest = tmp_path / "jobs.txt"
    manifest.write_text("# isolates\n\n" + "\n".join(lines) + "\n")
    r = subprocess.run([EXE, "batch", "--gpus", "1", str(manifest)], capture_output=True, text=True)
    assert r.returncode == 1 and r.stdout == ""
    err = r.stderr
    assert err.startswith("Starting Polypolish batch (H100 build %s, %d jobs, 1 GPU)\n\n" % (pp.lib().pp_version().decode(), len(cases)))
    assert err.endswith("Batch finished: %d jobs, %d failed\n" % (len(cases), len(bad)))
    heads = list(re.finditer(r"^\[job (\d+)/(\d+)\] manifest line (\d+): (\S+) -> (\S+) \(GPU 0\)\n", err, flags=re.M))
    assert [(int(m.group(1)), int(m.group(3)), m.group(4)) for m in heads] == [(i + 1, i + 3, c[1]["kind"]) for i, c in enumerate(cases)]
    blocks = [err[m.end():(heads[i + 1].start() if i + 1 < len(heads) else err.rindex("Batch finished"))] for i, m in enumerate(heads)]
    for (name, job, fasta, rep), single, block in zip(cases, singles, blocks):
        s = subprocess.run([EXE] + single, capture_output=True)
        out = tmp_path / "batch" / name / "polished.fasta"
        if name in bad:
            assert s.returncode == 1 and not out.exists()
            msg = s.stderr.decode().rsplit("\nError: ", 1)[1]
            assert block.endswith("Error: " + msg + "\n"), name
            continue
        assert s.returncode == 0 and out.read_bytes() == s.stdout == fasta, name
        assert block.endswith("Finished!\n\n"), name
        assert log_lines(block) == log_lines(s.stderr.decode()), name
        for f in os.listdir(tmp_path / "single" / name):
            assert (tmp_path / "batch" / name / f).read_bytes() == (tmp_path / "single" / name / f).read_bytes(), (name, f)
    # --quiet: the header and the Error: line of each failed job, nothing else
    q = subprocess.run([EXE, "batch", "--quiet", str(manifest)], capture_output=True, text=True)
    assert q.returncode == 1 and q.stdout == ""
    want = "".join(err[m.start():m.end()] + blocks[i].splitlines(keepends=True)[-2] for i, m in enumerate(heads) if cases[i][0] in bad)
    assert q.stderr == want
    # a batch of good jobs only: exit 0
    good = tmp_path / "good.txt"
    good.write_text("\n".join(x.replace(str(tmp_path / "batch"), str(tmp_path / "again")) for x, c in zip(lines, cases) if c[0] not in bad) + "\n")
    for name, *_ in cases:
        (tmp_path / "again" / name).mkdir(parents=True, exist_ok=True)
    g = subprocess.run([EXE, "batch", "--quiet", str(good)], capture_output=True, text=True)
    assert (g.returncode, g.stdout, g.stderr) == (0, "", "")
