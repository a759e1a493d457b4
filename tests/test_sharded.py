"""Sharded (vid % n) execution: world_size-2/3 gloo run on CPU for the host-side logic, NCCL run on GPUs."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import sparql_mini as M
from conftest import PLANS, ROOT, load_query, rows_equal
from wukong_b200 import capi, datagen


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_world(world, mode, tmp_path, univs=2, seed=7):
    port = _free_port()
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "sharded_worker.py"), "--rank", str(r), "--world",
                               str(world), "--port", str(port), "--mode", mode, "--univs", str(univs), "--seed", str(seed),
                               "--out", str(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
             for r in range(world)]
    outs = [p.communicate(timeout=900)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    return [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]


def _check_against_bruteforce(results, univs, seed):
    tr = datagen.lubm(univs, seed=seed)
    for q in range(1, 8):
        _, _, req, raw = load_query(q, PLANS[0])
        bf = M.bruteforce_bgp(tr, raw, req)
        for plan in PLANS:
            name = "q%d_%s" % (q, plan)
            got = np.concatenate([r[name].reshape(-1, len(req)) for r in results])
            assert rows_equal(got, bf), name


def test_exchange_plan():
    # Q7, optimal10240 plan: SURVEY appendix walk-through: 3 exchanges (by ?X, ?Y, ?Z)
    pats, nvars, req, _ = load_query(7, "optimal10240_plan")
    ex = capi.plan_exchanges(pats, nvars)
    assert [e for e in ex if e != -1] == [1, 0, 2] and ex[0] == -1 and ex[1] == -1 and ex[2] == -1
    # Q2: type-index seed then ?X name ?Y on the same (local) variable: no exchange at all
    pats, nvars, req, _ = load_query(2, "osdi16_plan")
    assert capi.plan_exchanges(pats, nvars) == [-1, -1]
    # a type-index lookup of a known variable must be replicated to every shard (sparql.hpp:1091-1110)
    assert capi.plan_exchanges([(18, 1, 0, -1), (-1, 5, 0, -2), (-2, 1, 0, -3)], 3)[2] == -2


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_cpu_gloo(world, tmp_path):
    """product shard builder + product exchange plan + gloo all_to_all, probed with the oracle primitives"""
    res = _run_world(world, "cpu", tmp_path)
    _check_against_bruteforce(res, 2, 7)


@pytest.mark.gpu
def test_partition_counts_single_gpu(lubm1):
    from wukong_b200 import host
    gst = host.HostStore(lubm1).upload(0)
    eng = capi.Engine(gst, rbuf_bytes=64 << 20)
    rng = np.random.default_rng(0)
    tbl = rng.integers(1 << 17, 1 << 24, (100003, 3), dtype=np.uint32)
    for nparts, col in ((2, 0), (8, 2), (5, 1)):
        eng.upload(tbl)
        got = eng.partition(col, nparts)
        assert np.array_equal(got, np.bincount(tbl[:, col] % nparts, minlength=nparts).astype(np.uint64))
    eng.close()
    gst.close()


@pytest.mark.gpu
def test_sharded_gpu_nccl(tmp_path):
    if capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(capi.device_count(), 4)
    res = _run_world(world, "gpu", tmp_path)
    _check_against_bruteforce(res, 2, 7)
    st = res[0]["__stats__"]
    assert st[0] > 0          # exchanges happened


@pytest.mark.gpu
def test_sharded_gpu_peer_memory(tmp_path):
    """same queries, exchange through CUDA-IPC peer memory (kernel stores over NVLink, no NCCL, no host sync)"""
    if capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(capi.device_count(), 4)
    res = _run_world(world, "gpu_p2p", tmp_path)
    _check_against_bruteforce(res, 2, 7)
    assert res[0]["__stats__"][0] > 0
    tot = sum(np.asarray(r["__stats__"], dtype=np.uint64) for r in res)      # exchanges, rows sent, rows received
    assert tot[1] == tot[2] and tot[1] > 0                                    # every row pushed to a peer arrived


@pytest.mark.gpu
def test_sharded_gpu_in_place_light_queries(tmp_path):
    """const-start plans answered by the constant's owner alone, probing the other shards through peer memory (the
    reference's in-place mode with one-sided reads); a table that outgrows shared memory falls back to the exchange path"""
    if capi.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(capi.device_count(), 4)
    res = _run_world(world, "gpu_inplace", tmp_path)
    _check_against_bruteforce(res, 2, 7)
    # light queries no longer exchange: fewer exchanges than the all-collective run of the same workload would need,
    # and every row of a light answer sits on ONE rank (the owner of Department0 / University0)
    for q in (4, 5, 6):
        name = "q%d_%s" % (q, PLANS[0])
        holders = [r for r in range(world) if res[r][name].size]
        assert len(holders) <= 1, (name, holders)
    want = _spill_want(datagen.lubm(2, seed=7))
    got = np.concatenate([r["spill"].reshape(-1, 3) for r in res])
    assert want.shape[0] > 1024 and rows_equal(got, want)


def _spill_want(tr):
    """members of Department0.University0 x their courses x the courses' teachers, by plain numpy joins"""
    d0 = M.lubm_str2id("<http://www.Department0.University0.edu>")
    P = {n: i for i, n in enumerate(M.LUBM_INDEX)}
    t = np.unique(tr, axis=0)
    mem = t[(t[:, 1] == P[M.UB + "memberOf>"]) & (t[:, 2] == d0)][:, 0]
    tc = t[(t[:, 1] == P[M.UB + "takesCourse>"]) & np.isin(t[:, 0], mem)]
    to = t[t[:, 1] == P[M.UB + "teacherOf>"]]
    return np.array([(x, c, y) for x, _, c in tc.tolist() for y, _, c2 in to[to[:, 2] == c].tolist()], dtype=np.uint32).reshape(-1, 3)


# ---- the same sharded execution with all shards on ONE GPU: engines of this process as a peer-memory group
# (wk_comm_local_group), one host thread per rank.  Runs on a single GPU under `-m gpu`. ----------
def _local_group(world, univs=2, seed=7, rbuf=128 << 20):
    from wukong_b200 import host
    stores, engs = [], []
    for r in range(world):
        tr = datagen.lubm_shard(univs, world, r, seed=seed, chunk=1)
        stores.append(host.HostStore(tr, num_servers=world, sid=r, kvstore_bytes=48 << 20).upload(0))
        engs.append(capi.Engine(stores[-1], rbuf_bytes=rbuf))
    capi.local_group(engs)
    return stores, engs


def _run_ranks(engs, fn):
    """fn(rank, engine) on one thread per rank (ctypes releases the GIL: the ranks' kernels are in flight together)"""
    import threading
    out, errs = [None] * len(engs), []

    def work(r):
        try:
            out[r] = fn(r, engs[r])
        except Exception as ex:   # noqa: BLE001
            import traceback
            errs.append("rank %d: %s" % (r, traceback.format_exc()))

    th = [threading.Thread(target=work, args=(r,)) for r in range(len(engs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, "\n".join(errs)
    return out


def _spill_plan():
    from oracle import oracle as O
    P = {n: i for i, n in enumerate(M.LUBM_INDEX)}
    d0 = M.lubm_str2id("<http://www.Department0.University0.edu>")
    return ([(d0, P[M.UB + "memberOf>"], O.IN, -1), (-1, P[M.UB + "takesCourse>"], O.OUT, -2),
             (-2, P[M.UB + "teacherOf>"], O.IN, -3)], 3, [-1, -2, -3])


@pytest.mark.gpu
@pytest.mark.parametrize("world,resident", [(2, 1), (3, 1), (2, 0)])
def test_sharded_local_group_single_gpu(world, resident):
    """Q1-Q7 x 3 plan sets + a const-start plan that outgrows shared memory, `world` shards on device 0: exchange through
    the single-pass peer-memory push, light plans in place on the constant's owner -- by the resident servers of all shards
    (owner walks the shards, peers wait for its verdict, nobody launches) or by one launch per rank -- all against the
    brute-force joiner"""
    stores, engs = _local_group(world)
    for e in engs:
        e.set_resident(bool(resident))
    queries = {"q%d_%s" % (q, plan): load_query(q, plan)[:3] for q in range(1, 8) for plan in PLANS}
    queries["spill"] = _spill_plan()

    def run(rank, eng):
        res = {}
        for name, (pats, nvars, req) in queries.items():
            rc, rows, cols, tbl = eng.query_sharded(pats, nvars, req)
            assert rc == 0, (name, rc)
            res[name] = tbl.copy() if rows else np.zeros((0, len(req)), np.uint32)
            rc, rows_b, _, _ = eng.query_sharded(pats, nvars, req, blind=True)
            assert rc == 0 and rows_b == rows, name
        res["__stats__"] = eng.comm_stats()
        res["__requests__"] = eng.get_option(capi.WK_INFO_RESIDENT_REQUESTS)
        return res

    res = _run_ranks(engs, run)
    _check_against_bruteforce(res, 2, 7)
    for r in res:   # every rank's server took part in every light query (as owner or as waiter), or none did
        assert (r["__requests__"] >= 2 * 3 * 3) if resident else (r["__requests__"] == 0), r["__requests__"]
    want = _spill_want(datagen.lubm(2, seed=7))
    got = np.concatenate([r["spill"].reshape(-1, 3) for r in res])
    assert want.shape[0] > 1024 and rows_equal(got, want)
    sent = sum(r["__stats__"]["rows_sent"] for r in res)
    recv = sum(r["__stats__"]["rows_recv"] for r in res)
    assert sent == recv and sent > 0 and res[0]["__stats__"]["exchanges"] > 0
    for q in (4, 5, 6):   # in place: every row of a light answer sits on the constant's owner
        assert len([r for r in range(world) if res[r]["q%d_%s" % (q, PLANS[0])].size]) <= 1
    for e in engs:
        e.close()
    for s in stores:
        s.close()


@pytest.mark.gpu
def test_exchange_local_group_tables_and_overflow():
    """wk_exchange_p2p on uploaded tables (1-9 columns, ragged tiles, replicate mode) against numpy; a receive buffer that
    is too small fails on EVERY rank with WK_ERR_RBUF_OVERFLOW and leaves the group usable"""
    world = 3
    stores, engs = _local_group(world, univs=1, seed=1, rbuf=8 << 20)
    rng = np.random.default_rng(5)
    # 700 K and 400 K rows: more tiles than the grid has CTAs, so space is reserved per chunk of several tiles (wk_sharded.cuh)
    for C, n in ((1, 700001), (2, 400003), (3, 50000), (5, 33333), (9, 4099), (2, 0)):
        tabs = [rng.integers(1 << 17, 1 << 26, (n + 13 * r, C), dtype=np.uint32) for r in range(world)]
        col = C // 2

        def run(rank, eng, tabs=tabs, col=col):
            eng.upload(tabs[rank], ncols=tabs[rank].shape[1])
            rows = eng.exchange_p2p(col)
            t = eng.download()
            return t[:rows]

        got = _run_ranks(engs, run)
        allrows = np.concatenate(tabs)
        for r in range(world):
            want = allrows[allrows[:, col] % world == r]
            assert got[r].shape[0] == want.shape[0], (C, n, r)
            if want.shape[0]:
                assert rows_equal(got[r].reshape(-1, C), want), (C, n, r)
    # replicate mode (the table of a type-index lookup, sparql.hpp:1091-1110): every rank ends up with every rank's rows;
    # 250 K rows per rank = more tiles than CTAs (chunked reservations), 1 000 rows = one tile per rank
    for nrep in (250007, 1000):
        tabs = [rng.integers(1 << 17, 1 << 26, (nrep + 5 * r, 2), dtype=np.uint32) for r in range(world)]

        def run_dup(rank, eng, tabs=tabs):
            eng.upload(tabs[rank], ncols=2)
            rows = eng.exchange_p2p(-2)
            return eng.download()[:rows]

        got = _run_ranks(engs, run_dup)
        allrows = np.concatenate(tabs)
        for r in range(world):
            assert got[r].shape[0] == allrows.shape[0] and rows_equal(got[r].reshape(-1, 2), allrows), (nrep, r)
    # overflow: 2 M words per buffer; rank 0 would receive 3 x 300 K rows x 3 columns
    tabs = [np.full((300000, 3), 3 * 1000 + 0, dtype=np.uint32) for _ in range(world)]   # every row is owned by rank 0

    def run_ovf(rank, eng):
        eng.upload(tabs[rank])
        try:
            eng.exchange_p2p(0)
        except capi.WukongError as ex:
            return ex.code
        return 0

    assert _run_ranks(engs, run_ovf) == [capi.WK_ERR_RBUF_OVERFLOW] * world
    # the group is still in step: a small exchange afterwards works
    tabs2 = [rng.integers(1 << 17, 1 << 20, (1000, 2), dtype=np.uint32) for _ in range(world)]

    def run2(rank, eng):
        eng.upload(tabs2[rank])
        rows = eng.exchange_p2p(1)
        return eng.download()[:rows]

    got = _run_ranks(engs, run2)
    allrows = np.concatenate(tabs2)
    for r in range(world):
        assert rows_equal(got[r].reshape(-1, 2), allrows[allrows[:, 1] % world == r])
    for e in engs:
        e.close()
    for s in stores:
        s.close()


def test_sharded_refuses_const_to_known():
    # a pattern that starts from a constant after the first step cannot be forked: OBJ_ERROR like need_fork_join (sparql.hpp:808)
    pats = [(18, 1, 0, -1), (131072, 5, 1, -1)]
    lib = capi.lib()
    import ctypes as C
    p = np.array(pats, dtype=np.int32)
    out = np.zeros(2, dtype=np.int32)
    assert lib.wk_plan_exchanges(p.ctypes.data_as(C.c_void_p), 2, 1, out.ctypes.data_as(C.c_void_p)) == 7   # WK_OBJ_ERROR
