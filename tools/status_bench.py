#!/usr/bin/env python
"""The status runs' cost: pp_polish_resident with status recorded (pp_polish_set_status) against without, steps alternated, on the
synthetic workload bench.py uses (seed 2, one contig, 150 bp multi-mapped pairs).  Wall time of the call (it ends in a device
synchronise; the run-length pass after the tile kernel is included, the fetch of the runs is not) and the library's CUDA-event time
of the polish stages.  With --files, also one `polish --status-bed` against one `polish --debug` from files, after one plain run.
Prints one JSON line with the card and its power limit.
usage: python tools/status_bench.py [contig_len] [depth] [steps] [--files]"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
import polypolish_b200 as pp  # noqa: E402
from polypolish_b200 import api  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
clen = int(args[0]) if len(args) > 0 else 5_000_000
depth = float(args[1]) if len(args) > 1 else 100.0
steps = int(args[2]) if len(args) > 2 else 50
syn = api.Synth(seed=2, n_contigs=1, contig_len=clen, depth=depth)
f = syn.fasta()
p = syn.pack(f)
wall = {False: [], True: []}
dev = {False: [], True: []}
runs = None
with pp.Context(0) as ctx:
    ctx.upload(f.view, p.view)
    for on in (False, True, False, True):                              # warm-up of both kernel instances
        ctx.polish_resident(fetch=False, status=on)
    for i in range(2 * steps):
        on = bool(i & 1)
        t0 = time.perf_counter()
        r = ctx.polish_resident(fetch=False, status=on)
        t1 = time.perf_counter()
        wall[on].append((t1 - t0) * 1e3)
        dev[on].append(r["timing"]["total_ms"])
        if on:
            runs = len(r["status"]["start"])
del p
files = None
if "--files" in sys.argv:
    exe = os.path.join(ROOT, "build", "polypolish")
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_stsb_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        fa, sams = syn.write(d)
        files = {}
        for name, extra in (("plain", []), ("status_bed", ["--status-bed", os.path.join(d, "s.bed")]), ("debug", ["--debug", os.path.join(d, "d.tsv")])):
            t0 = time.perf_counter()
            r = subprocess.run([exe, "polish", "--quiet"] + extra + [fa] + sams, capture_output=True)
            files[name + "_s"] = time.perf_counter() - t0
            assert r.returncode == 0, r.stderr.decode()
        files["status_bed_bytes"] = os.path.getsize(os.path.join(d, "s.bed"))
        files["debug_bytes"] = os.path.getsize(os.path.join(d, "d.tsv"))
    finally:
        shutil.rmtree(d, ignore_errors=True)
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip()
except Exception:
    card = None


def med(x):
    return sorted(x)[len(x) // 2]


print(json.dumps({"workload": "%d bp x %gx" % (clen, depth), "steps": steps, "runs": runs, "card": card,
                  "on_wall_ms_median": med(wall[True]), "off_wall_ms_median": med(wall[False]),
                  "on_device_ms_median": med(dev[True]), "off_device_ms_median": med(dev[False]),
                  "on_wall_ms_mean": sum(wall[True]) / steps, "off_wall_ms_mean": sum(wall[False]) / steps, "files": files}))
