#!/usr/bin/env python
"""Roofline scan on a power-law graph (BASELINE.json config 5): R-MAT, one predicate, 2-hop pattern
?a p ?b . ?b p ?c as upload(frontier) -> k2u -> k2u, frontier sweep F = 1K .. 64M bindings (x4 steps).
The frontier is the first F entries of a seeded shuffle of the subject index [0|p|IN].
Prints one JSON line per (F, hop): CUDA-event time, algorithmic bytes (SURVEY.md §8d), GB/s, % of the measured HBM peak."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=int, default=26)
ap.add_argument("--edges", type=int, default=1_000_000_000)
ap.add_argument("--max-frontier", type=int, default=64 << 20)
ap.add_argument("--rbuf-gb", type=int, default=24)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
from wukong_b200 import capi, datagen, host  # noqa: E402

try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 3350.0    # H100 SXM data sheet
t0 = time.time()
tr = datagen.rmat(args.scale, args.edges, seed=42, typed=False)
t1 = time.time()
hs = host.HostStore(tr, num_normal_preds=datagen.RMAT_NUM_NORMAL_PREDS)
del tr
t2 = time.time()
gst = hs.upload(0)
subjects = hs.get_edges(0, datagen.RMAT_PRED, 0)          # [0|p|IN] = all subjects of p
print(json.dumps({"phase": "setup", "gen_s": round(t1 - t0, 1), "build_s": round(t2 - t1, 1), "upload_s": round(time.time() - t2, 1),
                  "keys": int(hs.num_keys), "edges_words": int(hs.num_edges), "subjects": int(subjects.shape[0])}), flush=True)
rng = np.random.default_rng(7)
perm = rng.permutation(subjects.shape[0])
eng = capi.Engine(gst, rbuf_bytes=args.rbuf_gb << 30)
eng.set_profiling(2)
cap_rows_3col = (args.rbuf_gb << 30) // 12
F = 1024
sizes = []
while F < min(args.max_frontier, subjects.shape[0]):
    sizes.append(F)
    F *= 4
sizes.append(min(args.max_frontier, subjects.shape[0]))
for F in sizes:
    frontier = subjects[perm[:F]].reshape(-1, 1)
    res = {}
    for rep in range(args.reps):
        eng.upload(frontier)
        eng.flush_l2()
        n1 = eng.known_to_unknown(0, datagen.RMAT_PRED, 1)
        s1 = eng.step_stats()[-1]
        # second hop, chunked so that the output fits the buffer: stop if even hop 1's table would overflow hop 2
        est = s1["out_rows"] * max(1.0, s1["out_rows"] / max(1, F))
        if est > cap_rows_3col * 0.9:
            res.setdefault(1, []).append(s1)
            break
        eng.flush_l2()
        try:
            n2 = eng.known_to_unknown(1, datagen.RMAT_PRED, 1)
            s2 = eng.step_stats()[-1]
            res.setdefault(2, []).append(s2)
        except capi.WukongError as ex:
            if ex.code != capi.WK_ERR_RBUF_OVERFLOW:
                raise
        res.setdefault(1, []).append(s1)
    for hop, lst in sorted(res.items()):
        us = float(np.median([x["device_us"] for x in lst]))
        s = lst[0]
        print(json.dumps({"frontier": F, "hop": hop, "in_rows": s["in_rows"], "out_rows": s["out_rows"], "buckets": s["buckets_visited"],
                          "algo_bytes": s["algo_bytes"], "us": round(us, 2), "gbs": round(s["algo_bytes"] / us / 1e3, 1),
                          "pct_of_peak": round(100 * s["algo_bytes"] / us / 1e3 / peak, 1)}), flush=True)
