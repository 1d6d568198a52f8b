"""`--status-bed FILE` of `polish` and `filter-polish` without a GPU: its argument errors are clap's, word for word with exit code 2,
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
    (["polish", "--status-bed"], "a value is required for '--status-bed <FILE>' but none was supplied"),
    (["polish", "a.fa", "--status-bed"], "a value is required for '--status-bed <FILE>' but none was supplied"),
    (["filter-polish", "--in1", "a", "--in2", "b", "a.fa", "--status-bed"], "a value is required for '--status-bed <FILE>' but none was supplied"),
    # accepted, also as --status-bed=FILE: the next error is the missing positional
    (["polish", "--status-bed", "s.bed"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["polish", "--status-bed=s.bed"], "the following required arguments were not provided:\n  <ASSEMBLY>"),
    (["filter-polish", "--status-bed=s.bed", "--gpu-count", "2"],
     "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["filter", "--status-bed", "s.bed"], "unexpected argument '--status-bed' found"),
    (["filter", "--status-bed=s.bed"], "unexpected argument '--status-bed' found"),
])
def test_status_bed_usage_errors(args, msg):
    r = subprocess.run([EXE] + args, capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", f"error: {msg}\n\nFor more information, try '--help'.\n")


def test_help_names_status_bed():
    """`polish -h` names the flag; `filter-polish -h` takes the options of `polish` (except --debug), so it names it through them."""
    r = subprocess.run([EXE, "polish", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--status-bed <FILE>" in r.stdout
    r = subprocess.run([EXE, "filter-polish", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "of `polish` (except --debug)" in r.stdout


def test_filter_help_does_not():
    r = subprocess.run([EXE, "filter", "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--status-bed" not in r.stdout
