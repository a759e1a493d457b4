"""CPU: the JSON line bench.py prints -- keys and types a consumer reads.  The reference arm runs here (tiny scale); the
GPU arm's line is checked on the committed output of a 1-GPU run on an H100 (profiles/bench_lubm2560_h100.json) and, when
present, on committed sharded lines (profiles/r2_bench_sharded_*gpu_lubm10240.json)."""
import json
import os
import subprocess
import sys

from conftest import ROOT

BASE_KEYS = {"metric": str, "value": float, "unit": str, "n_gpus": int, "steps": int, "warmup": int, "ms_per_step": float,
             "higher_is_better": bool, "scaling": str, "dtype": str, "data": str, "config": dict, "e2e": dict}


def _check_base(d):
    for k, t in BASE_KEYS.items():
        assert k in d and isinstance(d[k], t), k
    assert "vs_baseline" in d and (d["vs_baseline"] is None or isinstance(d["vs_baseline"], float))
    assert d["metric"] == "lubm_q1_q7_geomean_queries_per_sec" and d["unit"] == "queries/s" and d["higher_is_better"] is True
    assert "workload" in d["config"] and "model" not in d["config"]
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"], k
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] > 0 and cb["unit"] == "queries/s" and cb["sample"]


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--scale", "1", "--steps", "2",
                          "--warmup", "1"], capture_output=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr.decode()[-2000:]
    lines = [l for l in out.stdout.decode().splitlines() if l.strip()]
    assert len(lines) == 1, lines                       # ONE line on stdout; libraries' chatter goes to stderr
    d = json.loads(lines[0])
    _check_base(d)
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["vs_baseline"] is None                     # the published figure is for LUBM-2560 only


def test_committed_gpu_line_has_the_contract_keys():
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_lubm2560_h100.json")))
    _check_base(d)
    assert "impl" not in d or d["impl"] != "reference"
    assert d["n_gpus"] == 1 and d["dtype"] == "u32" and d["data"] == "synthetic" and d["gpu_launches"] > 0
    assert "LUBM-2560" in d["config"]["workload"]
    r = d["roofline"]
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r, k
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3
    assert d["roofline_expand"]["frac"] >= 0.6          # the north-star's bar for the expand kernel
    c = d["clocks"]
    assert c["sm_mhz"] and c["sm_max_mhz"] and isinstance(c["reasons"], list)
    assert not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["value"] < d["value"]
    assert d["value"] / d["cpu_baseline"]["value"] >= 10    # the north-star's throughput bar, same box: blind vs blind
    assert d["e2e"]["value"] / d["cpu_baseline"]["e2e_value"] >= 10    # ... and non-blind end to end vs the CPU arm's non-blind
    assert d["parity"]["match"] is True and d["parity"]["queries"] == 7   # table digests equal the CPU arm's at full scale
    assert d["cpu_baseline"]["kind"] == "reference" and d["cpu_baseline"]["cores"] == d["cpu_baseline"]["host_cpus"]["usable"]


def test_committed_sharded_lines_have_the_contract_keys():
    import glob
    files = sorted(glob.glob(os.path.join(ROOT, "profiles", "r2_bench_sharded_*gpu_lubm10240.json")))
    for f in files:
        d = json.load(open(f))
        for k, t in BASE_KEYS.items():
            assert k in d and isinstance(d[k], t), (f, k)
        assert d["n_gpus"] > 1 and d["scaling"] == "strong" and "LUBM-10240" in d["config"]["workload"] and "sharded" in d["config"]["parallelism"]
        assert d["comm"]["bytes_pushed_per_step_all_ranks"] > 0 and d["comm"]["nvlink"]["achieved_gbs_per_gpu_per_direction"] > 0
        want = {"q1": 2542, "q2": 11069032, "q3": 0, "q4": 9, "q5": 13, "q6": 146, "q7": 383460}   # one GPU, same store (profiles)
        assert d["rows"] == want, f
        if d.get("secondary"):                              # the line carries the single-GPU run of the same store itself
            assert d["secondary"]["single_gpu_same_store"]["rows"] == want, f
        assert d["gpu_launches"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0


def test_spin_barrier_of_the_sharded_bench_on_two_gloo_ranks(tmp_path):
    """CPU: bench.SpinBarrier (dist.barrier + a generation counter per rank in /dev/shm, spun on) with two gloo ranks: no rank
    passes generation g before every rank has reached it, the shared file is gone afterwards"""
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    code = r'''
import os, sys, time
sys.path.insert(0, %r)
import numpy as np
import torch.distributed as dist
import bench
rank, world = int(sys.argv[1]), 2
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d", rank=rank, world_size=world)
bar = bench.SpinBarrier(rank, world, dist)
assert bar.a is not None and bar.a.shape[0] == 8 * world
seen = []
for g in range(1, 51):
    if rank == 1 and g %% 10 == 0:
        time.sleep(0.02)                     # a late rank: the other one must wait for it
    bar.wait()
    seen.append([int(x) for x in bar.slots])
    assert min(seen[-1]) >= g, (g, seen[-1])  # nobody is past a barrier the other has not reached
dist.barrier()
assert not [f for f in os.listdir("/dev/shm") if f.startswith("wk_bench_%%d_" %% os.getpid())]
dist.destroy_process_group()
print("ok", rank)
''' % (ROOT, port)
    procs = [subprocess.Popen([sys.executable, "-c", code, str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, cwd=ROOT) for r in range(2)]
    outs = [p.communicate(timeout=300)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0 and "ok" in o, o[-2000:]
