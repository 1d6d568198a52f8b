#!/usr/bin/env python
"""One per-position report's cost: pp_polish_resident with the report recorded against without, steps alternated, on the synthetic
workload bench.py uses (seed 2, one contig, 150 bp multi-mapped pairs).  Prints one JSON line with the card and its power limit.
  changes: the library's CUDA-event time of the call (pp_polish_set_changes); the fetch of the rows is not timed.
  status:  wall time of the call (it ends in a device synchronise; the run-length pass after the tile kernel and the fetch of the
           runs are included) and the library's CUDA-event time of the polish stages (pp_polish_set_status).
  depth:   wall time of the call (the run-length pass included), then apart from it the time of pp_polish_set_depth(ctx, 2) and of
           fetching the runs; the library's CUDA-event time of the polish stages and of the tile kernel alone; the run count and the
           bedGraph's size.  Then the same with recording left on from call to call ("kept": the keys are not allocated and released
           around every call).  With --walks (a tools/build_tile_prof.sh library in POLYPOLISH_LIB), one call off and one on after the
           warm-up, each preceded by a marker line on stderr, so that the library's "[tile prof]" lines can be told apart.
With --files, also one `polish` that writes the report against one `polish --debug` from files, after one plain run.
usage: python tools/report_bench.py --report changes|status|depth [contig_len] [depth] [steps] [--files] [--walks]"""
import argparse
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

ap = argparse.ArgumentParser()
ap.add_argument("--report", required=True, choices=("changes", "status", "depth"))
ap.add_argument("contig_len", nargs="?", type=int, default=5_000_000)
ap.add_argument("depth", nargs="?", type=float, default=100.0)
ap.add_argument("steps", nargs="?", type=int, default=50)
ap.add_argument("--files", action="store_true")
ap.add_argument("--walks", action="store_true")
a = ap.parse_args()
# per report: the CLI flag that writes it, and its name in the JSON
FILE_FLAG = {"changes": ("--changes", "changes"), "status": ("--status-bed", "status_bed"), "depth": ("--depth-bedgraph", "depth_bedgraph")}

g.build()
import polypolish_b200 as pp  # noqa: E402
from polypolish_b200 import api  # noqa: E402

clen, steps = a.contig_len, a.steps
syn = api.Synth(seed=2, n_contigs=1, contig_len=clen, depth=a.depth)
f = syn.fasta()
p = syn.pack(f)
L = api.lib()


def med(x):
    return sorted(x)[len(x) // 2]


def changes(ctx):
    for on in (False, True, False, True):                              # warm-up of both kernel instances
        ctx.polish_resident(fetch=False, changes=on)
    ms = {False: [], True: []}
    rows = None
    for i in range(2 * steps):
        on = bool(i & 1)
        r = ctx.polish_resident(fetch=False, changes=on)
        ms[on].append(r["timing"]["total_ms"])
        if on:
            rows = len(r["changes"])
    return {"rows": rows, "on_ms_per_call": sum(ms[True]) / steps, "off_ms_per_call": sum(ms[False]) / steps,
            "on_mbp_s": clen / 1e6 / (sum(ms[True]) / steps / 1e3), "off_mbp_s": clen / 1e6 / (sum(ms[False]) / steps / 1e3)}


def status(ctx):
    wall = {False: [], True: []}
    dev = {False: [], True: []}
    runs = None
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
    return {"runs": runs, "on_wall_ms_median": med(wall[True]), "off_wall_ms_median": med(wall[False]),
            "on_device_ms_median": med(dev[True]), "off_device_ms_median": med(dev[False]),
            "on_wall_ms_mean": sum(wall[True]) / steps, "off_wall_ms_mean": sum(wall[False]) / steps}


def depth(ctx):
    wall = {False: [], True: []}
    dev = {False: [], True: []}
    tile = {False: [], True: []}
    stop, fetch = [], []
    runs = bedgraph_bytes = None

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
    if a.walks:
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
    return {"runs": runs, "bedgraph_bytes": bedgraph_bytes, "on_wall_ms_median": med(wall[True]), "off_wall_ms_median": med(wall[False]),
            "on_device_ms_median": med(dev[True]), "off_device_ms_median": med(dev[False]),
            "on_tile_ms_median": med(tile[True]), "off_tile_ms_median": med(tile[False]),
            "stop_recording_ms_median": med(stop), "fetch_runs_ms_median": med(fetch),
            "kept_on_wall_ms_median": med(kept_wall), "kept_on_tile_ms_median": med(kept_tile),
            "on_wall_ms_mean": sum(wall[True]) / steps, "off_wall_ms_mean": sum(wall[False]) / steps}


with pp.Context(0) as ctx:
    ctx.upload(f.view, p.view)
    out = {"changes": changes, "status": status, "depth": depth}[a.report](ctx)
del p
files = None
if a.files:
    flag, name = FILE_FLAG[a.report]
    exe = os.path.join(ROOT, "build", "polypolish")
    shm = "/dev/shm"
    d = tempfile.mkdtemp(prefix="pp_repb_", dir=shm if os.path.isdir(shm) and shutil.disk_usage(shm).free > 6 << 30 else None)
    try:
        fa, sams = syn.write(d)
        files = {}
        for run, extra in (("plain", []), (name, [flag, os.path.join(d, "report")]), ("debug", ["--debug", os.path.join(d, "d.tsv")])):
            t0 = time.perf_counter()
            r = subprocess.run([exe, "polish", "--quiet"] + extra + [fa] + sams, capture_output=True)
            files[run + "_s"] = time.perf_counter() - t0
            assert r.returncode == 0, r.stderr.decode()
        files[name + "_bytes"] = os.path.getsize(os.path.join(d, "report"))
        files["debug_bytes"] = os.path.getsize(os.path.join(d, "d.tsv"))
    finally:
        shutil.rmtree(d, ignore_errors=True)
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip()
except Exception:
    card = None
print(json.dumps({"workload": "%d bp x %gx" % (clen, a.depth), "report": a.report, "steps": steps, **out, "card": card, "files": files}))
