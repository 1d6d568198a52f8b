"""`--depth-bedgraph FILE` of `polish` and `filter-polish` without a GPU: its argument errors are clap's, word for word with exit code 2,
and are decided before a GPU context is created; `polish -h` names it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "polypolish")


@pytest.fixture(scope="session", autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


@pytest.mark.parametrize("args,msg", [
    (["polish", "--depth-bedgraph"], "a value is required for '--depth-bedgraph <FILE>' but none was supplied"),
    (["polish", "a.fa", "--depth-bedgraph"], "a value is required for '--depth-bedgraph <FILE>' but none was supplied"),
    (["filter-polish", "--in1", "a", "--in2", "b", "a.fa", "--depth-bedgraph"], "a value is required for '--depth-bedgraph <FILE>' but none was supplied"),
    # accepted, also as --depth-bedgraph=FILE: the next error is the missing positional
    (["polish", "--depth-bedgraph", "d.bedgraph"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["polish", "--depth-bedgraph=d.bedgraph"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["filter-polish", "--depth-bedgraph=d.bedgraph", "--gpu-count", "2"],
     "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["filter", "--depth-bedgraph", "d.bedgraph"], "unexpected argument '--depth-bedgraph' found"),
    (["filter", "--depth-bedgraph=d.bedgraph"], "unexpected argument '--depth-bedgraph' found"),
])
def test_depth_bedgraph_usage_errors(args, msg):
    r = subprocess.run([EXE] + args, capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", f"error: {msg}\n\nFor more information, try '--help'.\n")


def test_help_names_depth_bedgraph():
    """`polish -h` names the flag; `filter-polish -h` takes the options of `polish` (except --debug), so it names it through them."""
    r = subprocess.run([EXE, "polish", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--depth-bedgraph <FILE>" in r.stdout
    r = subprocess.run([EXE, "filter-polish", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "of `polish` (except --debug)" in r.stdout


def test_filter_help_does_not():
    r = subprocess.run([EXE, "filter", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--depth-bedgraph" not in r.stdout
