#!/usr/bin/env python
"""The change report's cost: pp_polish_resident with the report on (pp_polish_set_changes) against off, steps alternated, on the
synthetic workload bench.py uses (seed 2, one contig, 150 bp multi-mapped pairs).  Device time of the call (CUDA events of the
library); the fetch of the rows is not timed.  Prints one JSON line with the card and its power limit.
usage: python tools/changes_bench.py [contig_len] [depth] [steps]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

g.build()
import polypolish_b200 as pp  # noqa: E402
from polypolish_b200 import api  # noqa: E402

clen = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
depth = float(sys.argv[2]) if len(sys.argv) > 2 else 100.0
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 50
syn = api.Synth(seed=2, n_contigs=1, contig_len=clen, depth=depth)
f = syn.fasta()
p = syn.pack(f)
with pp.Context(0) as ctx:
    ctx.upload(f.view, p.view)
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
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip()
except Exception:
    card = None
print(json.dumps({"workload": "%d bp x %gx" % (clen, depth), "steps": steps, "rows": rows, "card": card,
                  "on_ms_per_call": sum(ms[True]) / steps, "off_ms_per_call": sum(ms[False]) / steps,
                  "on_mbp_s": clen / 1e6 / (sum(ms[True]) / steps / 1e3), "off_mbp_s": clen / 1e6 / (sum(ms[False]) / steps / 1e3)}))
