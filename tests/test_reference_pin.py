"""CPU: the oracle against the reference's OWN compiled code (oracle/_ref/libwukong_ref.so: StaticGStore + SPARQLEngine of a
Wukong checkout behind C shims, see oracle/Makefile).  The reference's answers are stored under tests/golden/ (ref_answers.py):
where oracle/_ref is built they are recomputed live and must equal the stored ones, elsewhere the stored ones are used."""
import hashlib
import json
import os

import numpy as np
import pytest

import random_bgp as R
import sparql_mini as M
from conftest import PLANS, load_query
from oracle import oracle as O
from oracle import ref as REF
from ref_answers import EdgeDigest, answers, exact_digest, rows_digest
from wukong_b200 import host

HERE = os.path.dirname(os.path.abspath(__file__))


def table_digest(t):
    t = M.sort_rows(np.asarray(t, dtype=np.uint32))
    return hashlib.sha256(t.tobytes()).hexdigest()


def _occupied(v):
    """slots holding a key (slot 7 of a bucket is the chain pointer)"""
    idx = np.arange(v.shape[0])
    return (idx % 8 != 7) & (v[:, 0] != 0)


def _decode(k, p):
    """-> vid, pid, dir, edge count, edge offset of one slot"""
    return k >> 18, (k >> 1) & 0x1FFFF, k & 1, p & ((1 << 28) - 1), (p >> 28) & ((1 << 34) - 1)


def _ordered(vid, e):
    """index lists: their order follows hash-map iteration in the reference, a set is the contract; normal keys: the sorted run"""
    return np.sort(e) if vid == 0 else e


def _key_set(v):
    return hashlib.sha256(np.sort(v[_occupied(v), 0]).tobytes()).hexdigest()


def _segs(rows):
    return sorted([int(x) for x in r[:8]] for r in rows)


def _oracle_segs(o):
    return sorted([x.index, x.dir, x.pid, x.num_keys, x.num_buckets, x.bucket_start, x.num_edges, x.edge_start] for x in o.segs())


def _ref_edges(rs, keys):
    dg = EdgeDigest()
    for k in keys:
        vid, pid, d, _, _ = _decode(k, 0)
        dg.add(k, _ordered(vid, rs.get_edges(vid, pid, d)))
    return dg.hexdigest()


def _oracle_edges(oe, keys, ptrs):
    dg, n_index = EdgeDigest(), 0
    for k, p in zip(keys, ptrs):
        vid, _, _, size, off = _decode(k, p)
        n_index += vid == 0
        dg.add(k, _ordered(vid, oe[off:off + size]))
    return dg.hexdigest(), n_index


def test_store_matches_reference_store(lubm1):
    """segment table, key set and every key's edge list: the reference's StaticGStore::init + GStore::get_edges"""
    o = O.Store.build(lubm1, kvstore_bytes=1 << 30, num_engines=1, gpu_ext_mode=False)
    ov, oe = o.vertices(), o.edges()
    occ = _occupied(ov)
    keys, ptrs = ov[occ, 0].tolist(), ov[occ, 1].tolist()

    def compute(lib):
        rs = lib.RefStore(lubm1)
        return {"num_slots": int(rs.num_slots), "segs": _segs(rs.segs()), "keys": _key_set(rs.vertices()),
                "num_edges": int(rs.edges().shape[0]), "edges": _ref_edges(rs, keys)}
    ref = answers("store_lubm1", compute)
    assert ov.shape[0] == ref["num_slots"]
    assert _oracle_segs(o) == ref["segs"]
    assert _key_set(ov) == ref["keys"]                   # same key set
    assert oe.shape[0] == ref["num_edges"]
    edges, n_index = _oracle_edges(oe, keys, ptrs)
    assert edges == ref["edges"] and n_index > 30
    # the product host builder is bit-identical to the oracle (test_host_builder.py), hence pinned through it
    hs = host.HostStore(lubm1, kvstore_bytes=1 << 30, gpu_ext_extents=False)
    assert np.array_equal(hs.vertices(), ov) and np.array_equal(hs.edges(), oe)


def _extra_queries():
    univ0 = M.lubm_str2id("<http://www.University0.edu>")
    P = {n: i for i, n in enumerate(M.LUBM_INDEX)}
    # const_to_known in the middle of a plan (sparql.hpp:144-186): departments of graduate students that belong to University0
    c2k = [(P[M.UB + "GraduateStudent>"], 1, 0, -1), (-1, P[M.UB + "memberOf>"], 1, -2),
           (univ0, P[M.UB + "subOrganizationOf>"], 0, -2), (-2, P[M.UB + "name>"], 1, -3)]
    # known_to_unknown through the type index (pid == TYPE_ID && d == IN, sparql.hpp:339-340): professors -> their types ->
    # every instance of those types
    tidx = [(P[M.UB + "FullProfessor>"], 1, 0, -1), (-1, 1, 1, -2), (-2, 1, 0, -3)]
    errors = [([(-1, 5, 1, -2)], 2, [-1]), ([(18, 1, 0, -1), (univ0, 7, 0, -2)], 2, [-1]),
              ([(18, 5, 0, -1)], 1, [-1]), ([(18, 1, 0, -1)], 1, [])]
    return (c2k, 3, [-1, -3]), (tidx, 3, [-1, -2, -3]), errors


def test_engine_matches_reference_engine(lubm1, ostore1):
    """Q1-Q7 x 3 plan sets x mt 1/3, blind, DISTINCT / OFFSET / LIMIT, error codes: SPARQLEngine vs the oracle"""
    c2k, tidx, errors = _extra_queries()

    def compute(lib):
        rs, out = lib.RefStore(lubm1), {}
        for q in range(1, 8):
            for plan in PLANS:
                pats, nvars, req, _ = load_query(q, plan)
                name = "q%d_%s" % (q, plan)
                for mt in (1, 3):
                    rc, rows, cols, t = rs.query(pats, nvars, req, mt_factor=mt)
                    out["%s_mt%d" % (name, mt)] = [rc, rows, cols, rows_digest(t)]
                out[name + "_blind"] = list(rs.query(pats, nvars, req, blind=True)[:2])
                rc, rows, _, t = rs.query(pats, nvars, req, distinct=True, offset=1, limit=40)
                out[name + "_distinct"] = [rc, rows, exact_digest(t) if rows else None]
        for name, (pats, nv, req) in (("c2k", c2k), ("type_index", tidx)):
            rc, rows, cols, t = rs.query(pats, nv, req)
            out[name] = [rc, rows, cols, rows_digest(t)]
        out["errors"] = [rs.query(pats, nv, req)[0] for pats, nv, req in errors]
        return out
    ref = answers("engine_pin_lubm1", compute)
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, req, _ = load_query(q, plan)
            name = "q%d_%s" % (q, plan)
            for mt in (1, 3):
                want = O.run_query([ostore1], pats, nvars, req, mt_factor=mt)
                rc, rows, cols, dg = ref["%s_mt%d" % (name, mt)]
                assert rc == 0 and rows == want.rows, (q, plan, mt)
                if rows:
                    assert cols == want.cols and dg == rows_digest(want.table), (q, plan, mt)
            assert ref[name + "_blind"] == [0, want.rows]
            wd = O.run_query([ostore1], pats, nvars, req, distinct=True, offset=1, limit=40)
            rc, rows, dg = ref[name + "_distinct"]
            assert rc == 0 and rows == wd.rows and (rows == 0 or dg == exact_digest(wd.table)), (q, plan)
    for name, (pats, nv, req), least in (("c2k", c2k, 0), ("type_index", tidx, 1000)):
        want = O.run_query([ostore1], pats, nv, req)
        rc, rows, cols, dg = ref[name]
        assert rc == 0 and rows == want.rows > least and dg == rows_digest(want.table), name
    assert ref["errors"] == [O.run_query([ostore1], pats, nv, req).status for pats, nv, req in errors]


@pytest.mark.parametrize("gseed", [3, 11, 12])
def test_random_graph_matches_reference_engine(gseed):
    """random graphs (hubs, self loops, duplicates, multi-typed vertices) and 60 random plans each, chains of every primitive,
    through the reference engine"""
    tr, meta = R.graph(gseed, nv=300, ntriples=2500)
    npreds = meta["num_normal_preds"]
    ost = O.Store.build(tr, kvstore_bytes=8 << 20, num_engines=2, num_normal_preds=npreds)
    plans = {}
    for qseed in range(60):
        planned, _, nvars, req = R.query(7000 + 100 * gseed + qseed, tr, meta)
        if O.run_query([ost], planned, nvars, req, blind=True).rows <= 200_000:
            plans[str(qseed)] = (planned, nvars, req)

    def compute(lib):
        rs, out = lib.RefStore(tr, num_normal_preds=npreds), {}
        for k, (planned, nvars, req) in plans.items():
            rc, rows, _, t = rs.query(planned, nvars, req)
            drc, drows, _, dt = rs.query(planned, nvars, req, distinct=True)
            out[k] = [rc, rows, rows_digest(t), drc, drows, exact_digest(dt) if drows else None]
        return out
    ref = answers("random_graph_%d" % gseed, compute)
    assert sorted(ref) == sorted(plans) and len(plans) >= 45
    for k, (planned, nvars, req) in plans.items():
        rc, rows, dg, drc, drows, ddg = ref[k]
        want = O.run_query([ost], planned, nvars, req)
        assert rc == want.status == 0 and rows == want.rows, (k, planned)
        if rows:
            assert dg == rows_digest(want.table), (k, planned)
        wd = O.run_query([ost], planned, nvars, req, distinct=True)
        assert drc == 0 and drows == wd.rows and (drows == 0 or ddg == exact_digest(wd.table)), (k, planned)


@pytest.mark.parametrize("which", [1, 2])
def test_oracle_matches_reference_engine_fixture(ostore1, ostore2, which):
    """always runs: the reference engine's answers on LUBM-1 (seed 1) and LUBM-2 (seed 7), committed as row counts + digests of
    the sorted tables"""
    G = json.load(open(os.path.join(HERE, "golden", "ref_engine_lubm%d.json" % which)))
    ostore1 = ostore1 if which == 1 else ostore2
    assert G["queries"]
    for name, e in G["queries"].items():
        q, plan = int(name.split("_")[0][1:]), name.split("_", 1)[1]
        pats, nvars, req, _ = load_query(q, plan)
        got = O.run_query([ostore1], pats, nvars, req)
        assert got.status == 0 and got.rows == e["rows"], name
        if got.rows:
            assert table_digest(got.table) == e["sha256"], name
        d = O.run_query([ostore1], pats, nvars, req, distinct=True, offset=1, limit=40)
        assert d.rows == e["distinct_rows"] and (d.rows == 0 or hashlib.sha256(d.table.tobytes()).hexdigest() == e["distinct_sha256"]), name


CUSTOM_FMT = "# plan\n{\n 3 <\n\n1 >>\n  2 <<\n4 >\n5 <\n6 >\n1 >\n}\n9 >\n"
BAD_FMTS = ("1 <\n", "", "# nothing\n")


def test_set_plan_matches_reference_planner():
    """Planner::set_plan + set_direction (core/planner.hpp:1647-1754) vs the oracle's restatement and the independent Python
    reader (the C++ host mirror is held to the same reader in test_host_surface.py)"""
    from conftest import WORKLOADS

    def fmt_of(q, plan):
        return open(os.path.join(WORKLOADS, plan, "lubm_q%d.fmt" % q)).read()
    raw7 = load_query(7, "osdi16_plan")[3]

    def compute(lib):
        out = {"q%d_%s" % (q, plan): lib.set_plan(load_query(q, plan)[3], fmt_of(q, plan)) for q in range(1, 8) for plan in PLANS}
        # comments, blank lines, braces, reordering, every direction token, more plan lines than patterns
        out["custom"] = lib.set_plan(raw7, CUSTOM_FMT)
        out["bad"] = [lib.set_plan(raw7, bad) for bad in BAD_FMTS]
        return out
    ref = answers("set_plan", compute)
    for q in range(1, 8):
        for plan in PLANS:
            planned, _, _, raw = load_query(q, plan)
            planned = [list(t) for t in planned]
            assert ref["q%d_%s" % (q, plan)] == planned == [list(t) for t in O.set_plan(raw, fmt_of(q, plan))], (q, plan)
    assert ref["custom"] == [list(t) for t in O.set_plan(raw7, CUSTOM_FMT)] == [list(t) for t in M.apply_plan(raw7, CUSTOM_FMT)]
    assert ref["bad"] == [None] * len(BAD_FMTS)          # fewer plan lines than patterns: refused
    for bad in BAD_FMTS:
        with pytest.raises(ValueError):
            O.set_plan(raw7, bad)


FORK_PATS = [(18, 1, 0, -1), (-1, 5, 0, -2), (-2, 1, 1, -3), (-3, 1, 0, -4)]   # a type-index lookup of a bound variable
SPLITS = ((2, 0), (3, 2), (8, 1))


def test_fork_join_decisions_and_split_match_reference(lubm1):
    """row a15: which steps exchange (SPARQLEngine::need_fork_join + the replicate rule of dispatch) and how rows are split
    (generate_sub_query), against the product's host-side exchange planner and the `row[col] % n` rule of its kernels"""
    from wukong_b200 import capi
    tbl = np.random.default_rng(5).integers(1 << 17, 1 << 31, (5000, 3), dtype=np.uint32)

    def compute(lib):
        rs = lib.RefStore(lubm1)
        out = {"q%d_%s" % (q, plan): list(rs.fork_plan(*load_query(q, plan)[:2], 4)) for q in range(1, 8) for plan in PLANS}
        out["replicate"] = list(rs.fork_plan(FORK_PATS, 4, 3))
        out["split"] = [[exact_digest(part) for part in rs.split(tbl, col, n)] for n, col in SPLITS]
        return out
    ref = answers("fork_join", compute)
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, _, _ = load_query(q, plan)
            assert ref["q%d_%s" % (q, plan)] == [0, capi.plan_exchanges(pats, nvars)], (q, plan)
    assert ref["replicate"] == [0, capi.plan_exchanges(FORK_PATS, 4)] and -2 in ref["replicate"][1]
    for (n, col), parts in zip(SPLITS, ref["split"]):
        assert parts == [exact_digest(tbl[tbl[:, col] % n == i]) for i in range(n)]       # same rows, original order


def test_sharded_store_matches_reference_store(lubm1):
    """server 1 of 2 (OUT edges with the subject's owner, IN edges with the object's, index lists of local vertices only):
    the reference's partition + StaticGStore::init against the oracle's per-server build"""
    o = O.Store.build(lubm1, num_servers=2, sid=1, kvstore_bytes=1 << 30, num_engines=1, gpu_ext_mode=False)
    ov, oe = o.vertices(), o.edges()
    occ = _occupied(ov)
    pick = np.random.default_rng(1).permutation(int(occ.sum()))[:20000]
    idxkeys = ov[occ][(ov[occ, 0] >> np.uint64(18)) == 0]
    keys = ov[occ, 0][pick].tolist() + idxkeys[:, 0].tolist()
    ptrs = ov[occ, 1][pick].tolist() + idxkeys[:, 1].tolist()

    def compute(lib):
        rs = lib.RefStore(lubm1, num_servers=2, sid=1)
        return {"segs": _segs(rs.segs()), "keys": _key_set(rs.vertices()), "edges": _ref_edges(rs, keys)}
    ref = answers("sharded_store_lubm1", compute)
    assert _oracle_segs(o) == ref["segs"]
    assert _key_set(ov) == ref["keys"]
    assert _oracle_edges(oe, keys, ptrs)[0] == ref["edges"]


@pytest.mark.parametrize("n", [2, 3])
def test_simulated_reference_cluster(lubm1, n):
    """n shard stores built by the reference (refs_build with the loader's owner rule) and one reference engine per shard; the
    plan is driven by execute_one_pattern / need_fork_join / generate_sub_query exactly as execute_patterns does, with an
    in-process work list instead of the transport.  Answers must equal the brute-force joiner's and the oracle's cluster's."""
    def compute(lib):
        shards = [lib.RefStore(lubm1, num_servers=n, sid=i) for i in range(n)]
        out = {}
        for q in range(1, 8):
            for plan in PLANS:
                pats, nvars, req, _ = load_query(q, plan)
                rc, rows, _, t = lib.cluster_query(shards, pats, nvars, req)
                out["q%d_%s" % (q, plan)] = [rc, rows, rows_digest(t)]
        return out
    ref = answers("cluster_%d" % n, compute)
    oshards = [O.Store.build(lubm1, num_servers=n, sid=i, kvstore_bytes=32 << 20, num_engines=2) for i in range(n)]
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, req, raw = load_query(q, plan)
            bf = M.bruteforce_bgp(lubm1, raw, req)
            rc, rows, dg = ref["q%d_%s" % (q, plan)]
            assert rc == 0 and rows == bf.shape[0], (n, q, plan)
            if rows:
                assert dg == rows_digest(bf), (n, q, plan)
            mine = O.run_query(oshards, pats, nvars, req)
            assert mine.status == 0 and mine.rows == rows


def test_config_loader_matches_reference(tmp_path):
    """load_config(fname, nsrvs) + reload_config(str) of the host mirror (csrc/host/global.hpp) against the reference's own
    (core/config.hpp:42-230, compiled in oracle/_ref; non-GPU build, no RDMA device): every Global item, for the reference's
    sample config, for files that leave items at their defaults, repeat keys, carry unknown keys and comment lines, and for
    reloads that try to change immutable items"""
    from wukong_b200 import host
    sample = ("# general\nglobal_num_proxies              4\nglobal_num_engines              16\nglobal_data_port_base           5500\n"
              "global_ctrl_port_base           9576\nglobal_mt_threshold             8\nglobal_enable_workstealing      0\n"
              "global_stealing_pattern         0\nglobal_enable_planner           1\nglobal_generate_statistics      1\n"
              "global_enable_vattr             0\nglobal_silent                   1\n\n# kvstore\n"
              "global_input_folder             /path/to/input/rdfdata/id_lubm_40/\nglobal_memstore_size_gb         40\n"
              "global_est_load_factor          55\n\n# RDMA\nglobal_rdma_buf_size_mb         128\nglobal_rdma_rbf_size_mb         32\n"
              "global_use_rdma                 1\nglobal_rdma_threshold           300\nglobal_enable_caching           0\n\n# GPU\n"
              "global_num_gpus                 0\nglobal_gpu_rdma_buf_size_mb     64\nglobal_gpu_rbuf_size_mb         32\n"
              "global_gpu_kvcache_size_gb      10\nglobal_gpu_key_blk_size_mb      16\nglobal_gpu_value_blk_size_mb    4\n"
              "global_gpu_enable_pipeline      1\n")
    cases = [sample,
             sample.replace("global_mt_threshold             8", "global_mt_threshold             64"),     # clamped to num_engines
             "global_num_engines 4\n# c\n\nglobal_input_folder /a/b\nglobal_mt_threshold 2\nglobal_silent 0\nfoo_bar 3\nglobal_num_engines 6\n",
             "global_input_folder x/\nglobal_est_load_factor 35\nglobal_gpu_rbuf_size_mb 4096\nglobal_enable_planner 0 trailing words\n"]
    reloads = ["", "global_silent 0 global_mt_threshold 100 global_num_engines 99 global_use_rdma 1 global_enable_planner 0",
               "global_rdma_threshold 7\nglobal_enable_caching 1\nglobal_memstore_size_gb 1"]
    files = []
    for i, text in enumerate(cases):
        f = tmp_path / ("c%d.cfg" % i)
        f.write_text(text)
        files.append(str(f))

    def compute(lib):
        return {"%d_%d_%d" % (i, nsrvs, j): lib.load_config(f, nsrvs, rl)
                for i, f in enumerate(files) for nsrvs in (1, 3) for j, rl in enumerate(reloads)}
    ref = answers("config_loader", compute)
    assert len(ref) == len(files) * 2 * len(reloads)
    for i, f in enumerate(files):
        for nsrvs in (1, 3):
            for j, rl in enumerate(reloads):
                want = ref["%d_%d_%d" % (i, nsrvs, j)]
                got = host.load_config(f, nsrvs, rl)
                assert got == want, (i, nsrvs, rl, {k: (want[k], got[k]) for k in want if want[k] != got[k]})
    assert host.load_config(str(tmp_path / "missing.cfg"), 1) is None


def test_set_plan_with_union_and_optional_blocks():
    """.fmt plans with UNION { } / OPTIONAL { } blocks (core/planner.hpp:1722-1738): the host mirror's Planner::set_plan on
    pattern-group trees against the reference's own, for the union / optional workloads (workloads/lubm/{union,optional}), a
    nested block, blocks interleaved with the group's own lines, a sub-plan the block refuses, and refused plans"""
    from conftest import ROOT
    X, Y, S, UG, MAS, DOC = -1, -2, -1, -2, -3, -4
    T, NAME, WORKS, UGD, MASD, DOCD = 1, 8, 9, 2, 11, 12
    grp = lambda pats, unions=(), optionals=(): ([(s, p, 1, o) for (s, p, o) in pats], list(unions), list(optionals))   # noqa: E731
    def fmt(rel):
        return open(os.path.join(ROOT, "workloads", "lubm", rel)).read()
    cases = [
        (grp([], unions=[grp([(X, T, 20), (X, NAME, Y)]), grp([(X, T, 21), (X, NAME, Y)])]), fmt("union/manual_plan/q1.fmt")),
        (grp([(X, WORKS, 131072 + 5)], unions=[grp([(X, T, 22), (X, NAME, Y)]), grp([(X, T, 23), (X, NAME, Y)]), grp([(X, T, 24), (X, NAME, Y)])]),
         fmt("union/manual_plan/q4.fmt")),
        (grp([(S, UGD, UG)], optionals=[grp([(S, DOCD, DOC)])]), fmt("optional/manual_plan/q1.fmt")),
        (grp([(S, UGD, UG)], optionals=[grp([(S, MASD, MAS), (MAS, NAME, 131072 + 9)]), grp([(S, DOCD, DOC)])]), fmt("optional/manual_plan/q3.fmt")),
        # own lines before, between and after the blocks; an optional nested in a union; upper / lower case keywords
        (grp([(X, T, 20), (X, NAME, Y), (X, WORKS, -3)],
             unions=[grp([(X, UGD, -4)], optionals=[grp([(-4, NAME, -5)])]), grp([(X, MASD, -4)])],
             optionals=[grp([(X, DOCD, -6), (-6, NAME, -7)])]),
         "2 <\nunion {\n 1 >\n OPTIONAL {\n  1 <\n }\n}\n1 >\nUnion{\n 1 <<\n}\n3 >\noptional {\n 2 <\n 1 >>\n}\n"),
        # the second block lists fewer lines than it has patterns: refused for that block only
        (grp([(X, T, 20)], unions=[grp([(X, NAME, Y)]), grp([(X, NAME, Y), (X, WORKS, -3)])]), "1 <\nUNION {\n 1 >\n}\nUNION {\n 1 >\n}\n"),
        # the group itself lists fewer lines than it has patterns: no plan
        (grp([(X, T, 20), (X, NAME, Y)], unions=[grp([(X, WORKS, -3)])]), "1 <\nUNION {\n 1 >\n}\n"),
    ]

    def compute(lib):
        out = []
        for group, text in cases:
            w = lib.set_plan_tree(group, text)
            out.append(None if w is None else REF.encode_group(w))
        return out
    ref = answers("set_plan_tree", compute)
    assert len(ref) == len(cases)
    for (group, text), want in zip(cases, ref):
        got = host.set_plan_tree(REF.encode_group(group), text)
        assert (got is None) == (want is None), (group, text)
        if want is not None:
            assert got == want, (group, text, REF.decode_group(want)[0], REF.decode_group(got)[0])
    # at least one of each outcome was seen
    assert ref[0] is not None and ref[-1] is None
