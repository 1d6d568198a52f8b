"""`--gpu-count N` of `filter` and `filter-polish` without a GPU: its argument errors are clap's, word for word with exit code 2, and
are decided before a GPU context is created; `filter -h` names it."""
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
    (["filter", "--gpu-count", "x"], "invalid value 'x' for '--gpu-count <N>'"),
    (["filter", "--gpu-count", "-1"], "invalid value '-1' for '--gpu-count <N>': invalid digit found in string"),
    (["filter", "--gpu-count"], "a value is required for '--gpu-count <N>' but none was supplied"),
    (["filter", "--gpu-count", "2", "--in1", "a"],
     "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  --out1 <OUT1>\n  --out2 <OUT2>"),
    (["filter-polish", "--gpu-count=y", "a.fa"], "invalid value 'y' for '--gpu-count <N>'"),
    (["filter-polish", "--gpu-count", "2", "a.fa"], "the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>"),
    (["polish", "--gpu-count", "2", "a.fa"], "unexpected argument '--gpu-count' found"),
])
def test_gpu_count_usage_errors(args, msg):
    r = subprocess.run([EXE] + args, capture_output=True, text=True)
    assert (r.returncode, r.stdout, r.stderr) == (2, "", f"error: {msg}\n\nFor more information, try '--help'.\n")


def test_filter_help_names_gpu_count():
    r = subprocess.run([EXE, "filter", "-h"], capture_output=True, text=True)
    assert r.returncode == 0 and "--gpu-count <N>" in r.stdout
