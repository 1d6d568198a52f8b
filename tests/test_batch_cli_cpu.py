"""`polypolish batch MANIFEST` without a GPU: every manifest error is a clap-style usage error (exit 2, nothing on stdout) that names the
manifest line and is decided before a GPU context is created; comments and blank lines are accepted; the help names the command.  The
batch structs and entry point of pp_abi.h match INTEGRATION.md and the Python mirror, and every C-linkage export is declared."""
import ctypes as C
import os
import re
import subprocess

import pytest

from tests import test_abi_layout as layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")
LIB = os.path.join(ROOT, "build", "libpolypolish_b200.so")


@pytest.fixture(scope="session", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def usage(msg):
    return f"error: {msg}\n\nFor more information, try '--help'.\n"


def run_manifest(tmp_path, text, *opts):
    m = tmp_path / "jobs.txt"
    m.write_text(text)
    return subprocess.run([EXE, "batch", *opts, str(m)], capture_output=True, text=True, cwd=tmp_path)


GOOD = "polish a.fa r1.sam r2.sam --output a.polished.fa\n"


@pytest.mark.parametrize("line,msg", [
    ("frob a.fa --output x.fa", "unrecognized command 'frob' (a job is `polish` or `filter-polish`)"),
    ("filter --in1 a --in2 b --out1 c --out2 d --output x.fa", "unrecognized command 'filter' (a job is `polish` or `filter-polish`)"),
    ("polish a.fa --output x.fa --device 1", "'--device' applies to every job: it belongs on the `polypolish batch` command line"),
    ("polish a.fa --output x.fa --gpus 2", "'--gpus' applies to every job: it belongs on the `polypolish batch` command line"),
    ("polish --gpus=2 a.fa --output x.fa", "'--gpus' applies to every job: it belongs on the `polypolish batch` command line"),
    ("filter-polish --in1 a --in2 b a.fa --output x.fa --gpu-count 2",
     "'--gpu-count' applies to every job: it belongs on the `polypolish batch` command line"),
    ("polish --quiet a.fa --output x.fa", "'--quiet' applies to every job: it belongs on the `polypolish batch` command line"),
    ("polish a.fa --host-parse --output x.fa", "'--host-parse' applies to every job: it belongs on the `polypolish batch` command line"),
    ("polish a.fa r.sam", "the following required arguments were not provided:\n  --output <FILE>"),
    ("polish a.fa --output", "a value is required for '--output <FILE>' but none was supplied"),
    # the subcommand's own argument errors, word for word
    ("polish --output x.fa", "the following required arguments were not provided:\n  <ASSEMBLY>"),
    ("polish a.fa -m x --output x.fa", "invalid value 'x' for '--max_errors <MAX_ERRORS>'"),
    ("polish a.fa --low=0.2 --output x.fa", "unexpected argument '--low' found"),
    ("polish a.fa --output x.fa --changes", "a value is required for '--changes <FILE>' but none was supplied"),
    ("filter-polish --in1 a a.fa --output x.fa", "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    ("filter-polish --in1 a --in2 b a.fa --debug d.tsv --output x.fa", "unexpected argument '--debug' found"),
    ("filter-polish --in1 a --in2 b a.fa --high=x --output x.fa", "invalid value 'x' for '--high <HIGH>': invalid float literal"),
    ("polish a.fa --output x.fa -h", "unexpected argument '-h' found"),
    # one output file named twice
    ("polish a.fa --output x.fa --vcf x.fa", "the output file 'x.fa' is also written by this line"),
    ("polish a.fa --output x.fa --changes c.tsv --status-bed ./c.tsv", "the output file './c.tsv' is also written by this line"),
    ("filter-polish --in1 a --in2 b a.fa --out1 f.sam --out2 f.sam --output x.fa", "the output file 'f.sam' is also written by this line"),
    ("polish b.fa --output a.polished.fa", "the output file 'a.polished.fa' is also written by line 2"),
    ("polish b.fa --output sub/../a.polished.fa", "the output file 'sub/../a.polished.fa' is also written by line 2"),
    ("polish b.fa --output y.fa --debug a.polished.fa", "the output file 'a.polished.fa' is also written by line 2"),
])
def test_manifest_line_errors(tmp_path, line, msg):
    """The bad line is line 4: a comment and a blank line come first, then a good job."""
    r = run_manifest(tmp_path, "# isolates\n" + GOOD + "\n" + line + "\n")
    assert (r.returncode, r.stdout, r.stderr) == (2, "", usage("manifest line 4: " + msg))


def test_a_job_may_not_read_another_jobs_output(tmp_path):
    r = run_manifest(tmp_path, GOOD + "polish a.polished.fa r1.sam --output b.fa\n")
    assert (r.returncode, r.stdout, r.stderr) == (2, "", usage("manifest line 2: the input file 'a.polished.fa' is written by line 1 "
                                                               "(jobs may run in any order)"))
    r = run_manifest(tmp_path, "filter-polish --in1 r1.sam --in2 r2.sam a.fa --out1 f1.sam --out2 f2.sam --output a.p.fa\n"
                               "polish b.fa f1.sam f2.sam --output b.p.fa\n")
    assert (r.returncode, r.stderr) == (2, usage("manifest line 2: the input file 'f1.sam' is written by line 1 (jobs may run in any order)"))


@pytest.mark.parametrize("text", ["", "# nothing\n\n   \n\t# indented comment\n"], ids=["empty", "comments"])
def test_manifest_without_jobs(tmp_path, text):
    r = run_manifest(tmp_path, text)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", usage('the manifest "%s" has no jobs' % (tmp_path / "jobs.txt")))


def test_unreadable_manifest(tmp_path):
    r = subprocess.run([EXE, "batch", str(tmp_path / "missing.txt")], capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", usage('unable to read the manifest "%s"' % (tmp_path / "missing.txt")))


@pytest.mark.parametrize("args,msg", [
    ([], "the following required arguments were not provided:\n  <MANIFEST>"),
    (["a.txt", "b.txt"], "unexpected argument 'b.txt' found"),
    (["--debug", "d", "a.txt"], "unexpected argument '--debug' found"),
    (["--gpu-count", "2", "a.txt"], "unexpected argument '--gpu-count' found"),
    (["--gpus", "x", "a.txt"], "invalid value 'x' for '--gpus'"),
])
def test_batch_command_line_errors(args, msg):
    r = subprocess.run([EXE, "batch"] + args, capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", usage(msg))


def test_comments_blank_lines_and_clap_forms_are_accepted(tmp_path):
    """A valid manifest gets past validation: the next thing is the GPU (no usable device here, exit 1) or, on a GPU, the jobs
    themselves (whose inputs do not exist, exit 1).  Never a usage error."""
    text = ("# two isolates\n\n" + GOOD.replace(" ", "\t", 2) + "   \n"
            "  filter-polish --in1=r1.sam --in2 r2.sam --low=0.2 -m5 -i0.1 --output=b.fa -- b.fa   \r\n"
            "polish -d=3 --careful c.fa --output c.out.fa --changes c.tsv --status-bed c.bed --vcf c.vcf --depth-bedgraph c.bg --debug c.dbg\n")
    r = run_manifest(tmp_path, text)
    assert r.returncode == 1 and r.stdout == "" and not r.stderr.startswith("error:"), r.stderr
    assert not any(os.path.exists(tmp_path / f) for f in ("a.polished.fa", "b.fa", "c.out.fa"))


def test_help_names_batch():
    r = subprocess.run([EXE, "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and re.search(r"^  batch +run many polish / filter-polish jobs", r.stdout, flags=re.M)
    r = subprocess.run([EXE, "batch", "-h"], capture_output=True, text=True)
    assert r.returncode == 0 and "Usage: polypolish batch [OPTIONS] <MANIFEST>" in r.stdout
    for words in ("--output <FILE>", "--gpus <N>", "--quiet", "--host-parse", "cannot contain whitespace", "'#'"):
        assert words in r.stdout, words


def test_batch_structs_match_the_header_and_the_mirror(tmp_path):
    """PpBatchJob / PpBatchResult in INTEGRATION.md and BatchJob / BatchResult in api.py have the layout of pp_abi.h's structs."""
    from polypolish_b200 import api
    c = layout.c_layout(tmp_path)
    r = layout.rust_structs()
    for rname, cname, cls in (("PpBatchJob", "pp_batch_job", api.BatchJob), ("PpBatchResult", "pp_batch_result", api.BatchResult)):
        size, _, offsets = layout.rust_layout(rname, r)
        assert (size, offsets) == (c[cname]["size"], c[cname]["fields"]), rname
        assert list(offsets) == list(c[cname]["fields"])
        assert C.sizeof(cls) == c[cname]["size"], cname
        assert [f for f, _ in cls._fields_] == list(c[cname]["fields"]), cname
        for fname, _ in cls._fields_:
            assert getattr(cls, fname).offset == c[cname]["fields"][fname], (cname, fname)


def test_every_c_export_is_declared():
    """Every C-linkage function the library exports is declared in pp_abi.h (pp_batch_files included)."""
    out = subprocess.check_output(["nm", "-D", "--defined-only", LIB], text=True)
    exports = {p[2] for p in (x.split() for x in out.splitlines()) if len(p) == 3 and p[1] == "T" and p[2].startswith("pp_")}
    header = re.sub(r"/\*.*?\*/", "", open(layout.HEADER).read(), flags=re.S)
    declared = set(re.findall(r"\b(pp_\w+)\s*\(", header))
    assert "pp_batch_files" in exports
    assert sorted(exports - declared) == []
