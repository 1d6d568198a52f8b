#!/usr/bin/env python
"""K synthetic isolates polished three ways from the same page-cache files: (a) K one-shot `polypolish polish` processes in sequence,
(b) one `polypolish batch --gpus 1`, (c) one batch over N contexts.  Prints the card name and its power limit with the times, the bytes
of SAM text, where a one-shot process spends its wall time (the POLYPOLISH_TIMING marks tools/cli_startup.sh reads), and checks that
every output file is byte-identical across the three arms.  With N up to the visible GPUs arm (c) is `polypolish batch --gpus N`;
with more, the N contexts share the visible GPUs round-robin through the Python API (pp_batch_files, as the CLI calls it), which
measures the overhead of the multi-context scheduler, not throughput over N GPUs.
usage: python tools/batch_bench.py [K (12)] [contig_len (1000000)] [depth (60)] [N (max(2, visible GPUs))] [seed (1)]"""
import filecmp
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
from polypolish_b200 import api  # noqa: E402

EXE = os.path.join(ROOT, "build", "polypolish")
K = int(sys.argv[1]) if len(sys.argv) > 1 else 12
clen = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
depth = float(sys.argv[3]) if len(sys.argv) > 3 else 60.0
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
cards = [x for x in q.stdout.strip().splitlines() if x.strip()]
n_gpus = len(cards)
N = int(sys.argv[4]) if len(sys.argv) > 4 else max(2, n_gpus)
seed = int(sys.argv[5]) if len(sys.argv) > 5 else 1
if n_gpus == 0:
    sys.exit("batch_bench: no GPU visible (nvidia-smi lists none); there is nothing to measure")
print("cards: %s; %d visible" % ("; ".join(cards), n_gpus), flush=True)
base = "/dev/shm" if os.path.isdir("/dev/shm") and shutil.disk_usage("/dev/shm").free > (8 << 30) else None
d = tempfile.mkdtemp(prefix="pp_bb_", dir=base)
try:
    isolates, sam_bytes = [], 0
    for i in range(K):
        idir = os.path.join(d, "iso%02d" % i)
        os.mkdir(idir)
        syn = api.Synth(seed=seed * 1000 + i, n_contigs=1, contig_len=clen, depth=depth)
        fa, sams = syn.write(idir)
        syn.close()
        sam_bytes += sum(os.path.getsize(s) for s in sams)
        isolates.append((fa, sams))
    print("%d isolates of %d bp x %g: %d bytes (%.2f GB) of SAM text (%s)" % (K, clen, depth, sam_bytes, sam_bytes / 1e9,
                                                                             "tmpfs" if base else "disk"), flush=True)

    def manifest(arm):
        os.makedirs(os.path.join(d, arm), exist_ok=True)
        lines = ["polish %s %s --output %s" % (fa, " ".join(sams), os.path.join(d, arm, "iso%02d.fasta" % i)) for i, (fa, sams) in enumerate(isolates)]
        p = os.path.join(d, arm + ".txt")
        open(p, "w").write("\n".join(lines) + "\n")
        return p

    # (a) K one-shot processes, each timed like tools/cli_startup.sh: wall clock around the process, POLYPOLISH_TIMING marks inside it
    os.makedirs(os.path.join(d, "a"))
    marks = {"contexts created": [], "command done": []}
    t0 = time.perf_counter()
    walls = []
    for i, (fa, sams) in enumerate(isolates):
        s = time.perf_counter()
        with open(os.path.join(d, "a", "iso%02d.fasta" % i), "wb") as out:
            r = subprocess.run([EXE, "polish", "--quiet", fa] + sams, stdout=out, stderr=subprocess.PIPE, text=True,
                               env=dict(os.environ, POLYPOLISH_TIMING="1"))
        walls.append(time.perf_counter() - s)
        if r.returncode:
            sys.exit("one-shot polish failed: " + r.stderr)
        for m in re.finditer(r"\[timing\]\s+([\d.]+) ms  (.*)", r.stderr):
            if m.group(2) in marks:
                marks[m.group(2)].append(float(m.group(1)))
    ta = time.perf_counter() - t0
    med = lambda v: sorted(v)[len(v) // 2] if v else float("nan")  # noqa: E731
    print("(a) %d one-shot `polypolish polish` processes: %.2f s (per process: wall median %.3f s, min %.3f, max %.3f; "
          "contexts created at %.0f ms, command done at %.0f ms, medians)" % (K, ta, med(walls), min(walls), max(walls),
                                                                             med(marks["contexts created"]), med(marks["command done"])), flush=True)

    # (b) one batch process, one GPU
    m = manifest("b")
    t0 = time.perf_counter()
    r = subprocess.run([EXE, "batch", "--quiet", "--gpus", "1", m], capture_output=True, text=True)
    tb = time.perf_counter() - t0
    if r.returncode:
        sys.exit("batch --gpus 1 failed: " + r.stderr)
    print("(b) `polypolish batch --gpus 1`, %d jobs: %.2f s (%.3f s per job)" % (K, tb, tb / K), flush=True)

    # (c) N contexts
    m = manifest("c")
    if N <= n_gpus:
        label = "`polypolish batch --gpus %d`" % N
        t0 = time.perf_counter()
        r = subprocess.run([EXE, "batch", "--quiet", "--gpus", str(N), m], capture_output=True, text=True)
        tc = time.perf_counter() - t0
        if r.returncode:
            sys.exit("batch --gpus %d failed: %s" % (N, r.stderr))
    else:
        label = "overhead only: %d contexts on %d GPU%s (Python API, contexts created inside the timing)" % (N, n_gpus, "s" if n_gpus > 1 else "")
        jobs = [dict(kind="polish", assembly=fa, sams=sams, output=os.path.join(d, "c", "iso%02d.fasta" % i)) for i, (fa, sams) in enumerate(isolates)]
        t0 = time.perf_counter()
        res = api.batch(jobs, devices=[i % n_gpus for i in range(N)])
        tc = time.perf_counter() - t0
        if not all(x["ok"] for x in res):
            sys.exit("batch over %d contexts failed: %s" % (N, [x["error"] for x in res if not x["ok"]]))
    print("(c) %s, %d jobs: %.2f s (%.3f s per job)" % (label, K, tc, tc / K), flush=True)

    same = all(filecmp.cmp(os.path.join(d, "a", f), os.path.join(d, arm, f), shallow=False)
               for f in sorted(os.listdir(os.path.join(d, "a"))) for arm in ("b", "c"))
    n_files = len(os.listdir(os.path.join(d, "a")))
    print("outputs: %d FASTA files per arm, %s across the three arms" % (n_files, "byte-identical" if same else "DIFFERENT"), flush=True)
    print("(a) / (b) = %.2fx, (a) / (c) = %.2fx" % (ta / tb, ta / tc), flush=True)
    if not same:
        sys.exit(1)
finally:
    shutil.rmtree(d, ignore_errors=True)
