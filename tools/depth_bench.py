#!/usr/bin/env python
"""The depth runs' cost: pp_polish_resident with depth recorded (pp_polish_set_depth) against without, steps alternated, on the
synthetic workload bench.py uses (seed 2, one contig, 150 bp multi-mapped pairs).  Wall time of the call (it ends in a device
synchronise; the run-length pass after the tile kernel is included), then apart from it the time of pp_polish_set_depth(ctx, 2) and of
fetching the runs; the library's CUDA-event time of the polish stages and of the tile kernel alone; the run count and the bedGraph's
size.  Then the same with recording left on from call to call ("kept": the keys are not allocated and released around every call).  With --files, also one `polish --depth-bedgraph` against one `polish --debug` from files, after one plain run.  With --walks
(a tools/build_tile_prof.sh library in POLYPOLISH_LIB), one call off and one on after the warm-up, each preceded by a marker line on
stderr, so that the library's "[tile prof]" lines can be told apart.  Prints one JSON line with the card and its power limit.
usage: python tools/depth_bench.py [contig_len] [depth] [steps] [--files] [--walks]"""
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
tile = {False: [], True: []}
stop, fetch = [], []
runs = bedgraph_bytes = None
L = api.lib()
with pp.Context(0) as ctx:
    ctx.upload(f.view, p.view)

    def call(on):
        """One resident call with depth recorded or not: its wall time (the run pass included) and result; with depth on also the
        time of pp_polish_set_depth(ctx, 2) (which releases the keys) and of fetching the runs."""
        if on:
            L.pp_polish_set_depth(ctx.h, 1)
        t0 = time.perf_counter()
        r = ctx.polish_resident(fetch=False)
        t1 = time.perf_counter()
        if on:
            L.pp_polish_set_depth(ctx.h, 2)
            t2 = time.perf_counter()
            r["depth"] = ctx.depth_runs()
            stop.append((t2 - t1) * 1e3)
            fetch.append((time.perf_counter() - t2) * 1e3)
        return (t1 - t0) * 1e3, r

    for on in (False, True, False, True):                              # warm-up of both kernel instances
        call(on)
    if "--walks" in sys.argv:
        for on in (False, True):
            print("== depth %s" % ("on" if on else "off"), file=sys.stderr, flush=True)
            call(on)
    for i in range(2 * steps):
        on = bool(i & 1)
        w, r = call(on)
        wall[on].append(w)
        dev[on].append(r["timing"]["total_ms"])
        tile[on].append(r["timing"][api.STAGES[3] + "_ms"])
        if on:
            d = r["depth"]
            runs = len(d["start"])
            bedgraph_bytes = len(f.names[0].encode()) * runs + sum(
                len("\t%d\t%d\t%d.%d\n" % (s, e, t // 10, t % 10)) for s, e, t in zip(d["start"].tolist(), d["end"].tolist(), d["tenths"].tolist()))
    # recording left on from call to call (the keys stay allocated): the kernels' own cost
    kept_wall, kept_tile = [], []
    L.pp_polish_set_depth(ctx.h, 1)
    for i in range(steps):
        t0 = time.perf_counter()
        r = ctx.polish_resident(fetch=False)
        kept_wall.append((time.perf_counter() - t0) * 1e3)
        kept_tile.append(r["timing"][api.STAGES[3] + "_ms"])
    L.pp_polish_set_depth(ctx.h, 0)
del p
files = None
if "--files" in sys.argv:
    exe = os.path.join(ROOT, "build", "polypolish")
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_depb_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        fa, sams = syn.write(d)
        files = {}
        for name, extra in (("plain", []), ("depth_bedgraph", ["--depth-bedgraph", os.path.join(d, "d.bedgraph")]),
                            ("debug", ["--debug", os.path.join(d, "d.tsv")])):
            t0 = time.perf_counter()
            r = subprocess.run([exe, "polish", "--quiet"] + extra + [fa] + sams, capture_output=True)
            files[name + "_s"] = time.perf_counter() - t0
            assert r.returncode == 0, r.stderr.decode()
        files["depth_bedgraph_bytes"] = os.path.getsize(os.path.join(d, "d.bedgraph"))
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


print(json.dumps({"workload": "%d bp x %gx" % (clen, depth), "steps": steps, "runs": runs, "bedgraph_bytes": bedgraph_bytes, "card": card,
                  "on_wall_ms_median": med(wall[True]), "off_wall_ms_median": med(wall[False]),
                  "on_device_ms_median": med(dev[True]), "off_device_ms_median": med(dev[False]),
                  "on_tile_ms_median": med(tile[True]), "off_tile_ms_median": med(tile[False]),
                  "stop_recording_ms_median": med(stop), "fetch_runs_ms_median": med(fetch),
                  "kept_on_wall_ms_median": med(kept_wall), "kept_on_tile_ms_median": med(kept_tile),
                  "on_wall_ms_mean": sum(wall[True]) / steps, "off_wall_ms_mean": sum(wall[False]) / steps, "files": files}))
