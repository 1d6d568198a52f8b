#!/usr/bin/env python
"""`filter` and `filter-polish` from page-cache files at 1 and at N contexts, alternated (pp_filter_files_multi /
pp_filter_polish_files_multi through the Python mirror, contexts created once and reused).  Prints the card name and its power
limit with the times.  The assembly has N contigs (assembly_len / N bp each), so that the fused call, which like `polish` uses at
most one context per contig, runs on all N.  On a machine with fewer GPUs than N the N contexts share the visible devices round-robin:
that measures the overhead of the multi-context path (ranges, exchange of records by read name, reductions), not scaling over PCIe links.
usage: python tools/filter_multi_bench.py [n_contexts (8)] [assembly_len (5000000)] [depth (100)] [reps (3)]"""
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
import torch  # noqa: E402

import polypolish_b200 as pp  # noqa: E402
from polypolish_b200 import api  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 8
clen = int(sys.argv[2]) if len(sys.argv) > 2 else 5_000_000
depth = float(sys.argv[3]) if len(sys.argv) > 3 else 100.0
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 3
n_gpus = torch.cuda.device_count()
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print(f"cards: {q.stdout.strip() or 'unknown'}; {n_gpus} visible", flush=True)
label = "scaling over %d GPUs" % n if n_gpus >= n else "overhead only: %d contexts on %d GPU%s" % (n, n_gpus, "s" if n_gpus > 1 else "")
base = "/dev/shm" if os.path.isdir("/dev/shm") and shutil.disk_usage("/dev/shm").free > (8 << 30) else None
d = tempfile.mkdtemp(prefix="pp_fmb_", dir=base)
ctxs = [pp.Context(i % max(1, n_gpus)) for i in range(n)]
try:
    syn = api.Synth(seed=2, n_contigs=n, contig_len=clen // n, depth=depth)
    fa, sams = syn.write(d)
    sizes = sum(os.path.getsize(s) for s in sams)
    print(f"{n} contigs, {clen} bp x {depth:g}: {sizes / 1e9:.2f} GB of SAM text ({'tmpfs' if base else 'disk'}); {label}", flush=True)
    o1, o2 = os.path.join(d, "o1.sam"), os.path.join(d, "o2.sam")
    times = {}
    for rep in range(reps + 1):                     # the first round warms the page cache and the contexts' buffers
        for k in (1, n):
            t0 = time.perf_counter()
            api.filter_files_multi(sams[0], sams[1], o1, o2, contexts=ctxs[:k])
            t1 = time.perf_counter()
            api.filter_polish_files_multi(fa, sams[0], sams[1], contexts=ctxs[:k])
            t2 = time.perf_counter()
            if rep:
                times.setdefault(("filter", k), []).append((t1 - t0) * 1e3)
                times.setdefault(("filter-polish", k), []).append((t2 - t1) * 1e3)
    for (what, k), v in sorted(times.items()):
        v.sort()
        print(f"{what:14s} {k} context{'s' if k > 1 else ' '}: median {v[len(v) // 2]:.0f} ms (min {v[0]:.0f}, max {v[-1]:.0f}, {len(v)} runs)", flush=True)
finally:
    for c in ctxs:
        c.close()
    shutil.rmtree(d, ignore_errors=True)
