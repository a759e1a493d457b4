#!/usr/bin/env python
"""Roofline scan on a power-law graph at 1 / 2 / 4 / 8 GPUs (BASELINE.json config 5): R-MAT (2^scale vertices, `edges` directed
edges, one predicate), store sharded by vid % N, 2-hop pattern ?a p ?b . ?b p ?c as
    frontier (this rank's share of a seeded shuffle of its subjects) -> known_to_unknown -> exchange by ?b -> known_to_unknown
Launch:  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 scripts/rmat_scan_sharded.py
One JSON line per frontier size: per hop the slowest rank's CUDA-event time, the algorithmic bytes of all ranks (SURVEY.md 8d),
aggregate and per-GPU GB/s against the measured HBM peak; for the exchange the bytes pushed over NVLink, GB/s per GPU and
direction against the measured peer-copy peak.  A second hop whose output does not fit the result buffers is run over
buffer-sized chunks of the first hop's output (wk_table_slice), the first --max-chunks of them, as SURVEY.md 8d prescribes.
Vertex labels are scrambled like Graph500's, so that vid % N shards carry equal shares of the hubs."""
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
ap.add_argument("--rbuf-gb", type=int, default=32)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--max-chunks", type=int, default=6)
args = ap.parse_args()
if int(os.environ.get("WORLD_SIZE", 1)) > 1:   # torchrun pins OMP_NUM_THREADS=1; the generator is OpenMP-parallel
    os.environ["OMP_NUM_THREADS"] = str(max(1, len(os.sched_getaffinity(0)) // int(os.environ["WORLD_SIZE"])))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from wukong_b200 import capi, datagen  # noqa: E402

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 3350.0    # H100 SXM data sheet
NVLINK = 450.0     # H100 SXM data sheet: NVLink 4, 900 GB/s per GPU both directions together
P = datagen.RMAT_PRED
t0 = time.time()
tr = datagen.rmat(args.scale, args.edges, seed=42, typed=False)
if world > 1:     # this rank's shard: triples whose subject or object it owns (base_loader.hpp:169-181)
    keep = (tr[:, 0] % world == rank) | (tr[:, 2] % world == rank)
    tr = tr[keep]
t1 = time.time()
gst = None
for lf in (55, 45, 35, 25):   # a skewed graph may outgrow a segment's ext extent at the default load factor
    try:
        gst = capi.Store.build(tr, datagen.RMAT_NUM_NORMAL_PREDS, num_servers=world, sid=rank, est_load_factor=lf, device=local)
        break
    except capi.WukongError as ex:
        if ex.code != capi.WK_ERR_STORE_FULL or lf == 25:
            raise
del tr
t2 = time.time()
subjects = gst.get_edges(0, P, 0, cap=1 << 27)          # [0|p|IN] restricted to this shard = the subjects it owns
eng = capi.Engine(gst, rbuf_bytes=args.rbuf_gb << 30)
if world > 1:
    allh = [None] * world
    dist.all_gather_object(allh, eng.p2p_export(world, rank))
    eng.p2p_import(b"".join(allh))
    dist.barrier()
nsub = torch.tensor([subjects.shape[0]], device="cuda", dtype=torch.int64)
if world > 1:
    dist.all_reduce(nsub)
nsub = int(nsub.item())
if rank == 0:
    print(json.dumps({"phase": "setup", "n_gpus": world, "gen_filter_s": round(t1 - t0, 1), "build_s": round(t2 - t1, 1),
                      "subjects_all_ranks": nsub, "build": {k: (round(v, 1) if isinstance(v, float) else v) for k, v in gst.build_stats.items()}}), flush=True)
rng = np.random.default_rng(7 + rank)
perm = rng.permutation(subjects.shape[0])
eng.set_profiling(2)
cap_rows = (args.rbuf_gb << 30) // 12
sizes, F = [], 1024
while F < min(args.max_frontier, nsub):
    sizes.append(F)
    F *= 4
sizes.append(min(args.max_frontier, nsub))


def allmax(x):
    t = torch.tensor([float(x)], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allsum(x):
    t = torch.tensor([float(x)], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t)
    return float(t.item())


def prepare(frontier):
    """frontier -> hop 1 -> exchange by ?b; returns (rows now on this rank, hop-1 stats, exchange stats)"""
    eng.upload(frontier)
    eng.flush_l2()
    eng.sync()
    if world > 1:
        dist.barrier()
    eng.known_to_unknown(0, P, 1)
    s1 = eng.step_stats()[-1]
    sx = None
    if world > 1:
        eng.flush_l2(); eng.sync(); dist.barrier()
        eng.exchange_p2p(1)
        sx = [x for x in eng.step_stats() if x["kind"] == "exchange"][-1]
    return eng.info()[0], s1, sx


def timed_hop2():
    """second hop over the current table; None when some rank's output did not fit"""
    eng.flush_l2(); eng.sync()
    if world > 1:
        dist.barrier()
    try:
        eng.known_to_unknown(1, P, 1)
        st, ok = eng.step_stats()[-1], 1.0
    except capi.WukongError as ex:
        if ex.code != capi.WK_ERR_RBUF_OVERFLOW:
            raise
        st, ok = None, 0.0
    return st if allsum(ok) == world else None


fan = 64.0          # rows out per row in of the last second hop that ran: sizes the chunks of the next one
for F in sizes:
    mine = min(subjects.shape[0], (F + world - 1) // world)
    frontier = subjects[perm[:mine]].reshape(-1, 1)
    acc = {"hop1": [], "xchg": [], "hop2": []}
    last = {}
    whole = True
    n_in = 0
    for rep in range(args.reps):
        n_in, s1, sx = prepare(frontier)
        acc["hop1"].append(s1["device_us"]); last["hop1"] = s1
        if sx is not None:
            acc["xchg"].append(sx["device_us"]); last["xchg"] = sx
        if not whole:
            continue
        # every rank takes the same decision
        if allmax(n_in * fan) > cap_rows * 0.7:
            whole = False
            continue
        s2 = timed_hop2()
        if s2 is None:
            whole = False
            acc["hop2"] = []
            continue
        acc["hop2"].append(s2["device_us"]); last["hop2"] = s2
        fan = max(1.0, allmax(s2["out_rows"] / max(1, s2["in_rows"])))
    line = {"frontier": F, "n_gpus": world}
    for name in ("hop1", "xchg", "hop2"):
        have = allsum(1.0 if acc[name] else 0.0)
        if have < world:
            continue
        us = allmax(float(np.median(acc[name])))
        st = last[name]
        by = allsum(st["algo_bytes"])
        e = {"us_max_rank": round(us, 2), "in_rows": int(allsum(st["in_rows"])), "out_rows": int(allsum(st["out_rows"])), "algo_bytes": int(by)}
        if name == "xchg":
            per_gpu = by / world / us / 1e3
            e.update({"nvlink_gbs_per_gpu": round(per_gpu, 1), "pct_of_nvlink_peak": round(100 * per_gpu / NVLINK, 1)})
        else:
            e.update({"gbs_all_gpus": round(by / us / 1e3, 1), "gbs_per_gpu": round(by / world / us / 1e3, 1),
                      "pct_of_hbm_peak_per_gpu": round(100 * by / world / us / 1e3 / peak, 1)})
        line[name] = e
    if not whole:
        # chunked second hop: B rows of the (exchanged) first-hop output at a time, sized from the last fan-out seen and halved
        # until every rank's output fits; the first max_chunks chunks are timed
        nmax = int(allmax(n_in))
        B = int(max(1024, min(nmax, cap_rows * 0.5 / fan)))
        tries = 0
        while True:
            prepare(frontier)
            eng.slice(0, B)
            s2 = timed_hop2()
            tries += 1
            if s2 is not None or B <= 1024 or tries > 24:
                break
            B //= 2
        if s2 is not None:
            nchunks_all = (nmax + B - 1) // B
            K = int(min(args.max_chunks, nchunks_all))
            us_sum, by_sum, in_sum, out_sum = allmax(s2["device_us"]), allsum(s2["algo_bytes"]), allsum(s2["in_rows"]), allsum(s2["out_rows"])
            done = 1
            for k in range(1, K):
                prepare(frontier)
                eng.slice(k * B, B)
                sk = timed_hop2()
                if sk is None:     # a chunk full of hubs: leave it out, say so
                    continue
                us_sum += allmax(sk["device_us"]); by_sum += allsum(sk["algo_bytes"])
                in_sum += allsum(sk["in_rows"]); out_sum += allsum(sk["out_rows"])
                done += 1
            fan = max(1.0, out_sum / max(1.0, in_sum)) * 1.5
            line["hop2"] = {"us_max_rank": round(us_sum, 2), "in_rows": int(in_sum), "out_rows": int(out_sum), "algo_bytes": int(by_sum),
                            "gbs_all_gpus": round(by_sum / us_sum / 1e3, 1), "gbs_per_gpu": round(by_sum / world / us_sum / 1e3, 1),
                            "pct_of_hbm_peak_per_gpu": round(100 * by_sum / world / us_sum / 1e3 / peak, 1),
                            "chunked": {"rows_per_chunk_per_rank": B, "chunks_timed": done, "chunks_total": int(nchunks_all),
                                        "note": "sum over the timed chunks of the slowest rank's time; every chunk after its own L2 flush"}}
        else:
            line["note"] = "second hop: no chunk size down to 1024 rows fits the result buffers"
    if rank == 0:
        print(json.dumps(line), flush=True)
eng.close()
gst.close()
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
