"""GPU: the engine against the reference's OWN compiled code (the file name sorts last so that it runs after the other GPU tests).

* the committed answers of the reference engine (tests/golden/ref_engine_lubm1.json, made by tests/golden/make_ref_engine.py
  from oracle/_ref) -- always runs;
* a store BUILT BY THE REFERENCE (StaticGStore::init, CPU build with many 256-bucket ext extents, unsorted index lists),
  uploaded as is with wk_store_create and queried on the GPU -- runs where oracle/_ref is built;
* a random graph against the reference engine's stored answers (tests/golden/ref_random_graph_gpu.json) -- always runs."""
import numpy as np
import pytest

import sparql_mini as M
from conftest import PLANS, load_query, rows_equal
from oracle import oracle as O
from wukong_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng1(gstore1):
    e = capi.Engine(gstore1, rbuf_bytes=64 << 20)
    yield e
    e.close()


@pytest.fixture(scope="module")
def eng2(gstore2):
    e = capi.Engine(gstore2, rbuf_bytes=64 << 20)
    yield e
    e.close()


@pytest.mark.parametrize("which", [1, 2])
def test_matches_reference_engine_fixture(eng1, eng2, which):
    """the answers of the reference's OWN compiled engine on this dataset (tests/golden/ref_engine_lubm1.json, produced by
    tests/golden/make_ref_engine.py from oracle/_ref): row counts and digests of the sorted tables, exact tables under DISTINCT"""
    import hashlib
    import json
    import os
    G = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_engine_lubm%d.json" % which)))
    eng1 = eng1 if which == 1 else eng2
    for name, e in G["queries"].items():
        q, plan = int(name.split("_")[0][1:]), name.split("_", 1)[1]
        pats, nvars, req, _ = load_query(q, plan)
        rc, rows, cols, tbl = eng1.query(pats, nvars, req)
        assert rc == 0 and rows == e["rows"], name
        if rows:
            assert hashlib.sha256(M.sort_rows(tbl).tobytes()).hexdigest() == e["sha256"], name
        rc, rows, cols, tbl = eng1.query(pats, nvars, req, distinct=True, offset=1, limit=40)
        assert rc == 0 and rows == e["distinct_rows"], name
        if rows:
            assert hashlib.sha256(np.ascontiguousarray(tbl).tobytes()).hexdigest() == e["distinct_sha256"], name


def test_reference_built_store_runs_on_the_gpu(lubm1, ostore1):
    from oracle import ref as REF
    try:
        ok = REF.available()
    except OSError:
        ok = False
    if not ok:
        pytest.skip("oracle/_ref is not built (needs a Wukong checkout)")
    rs = REF.RefStore(lubm1)
    segs = []
    for r in rs.segs():
        m = capi.SegMeta()
        m.index, m.dir, m.pid = int(r[0]), int(r[1]), int(r[2])
        m.num_keys, m.num_buckets, m.bucket_start, m.num_edges, m.edge_start = (int(x) for x in r[3:8])
        m.ext_start, m.ext_num = int(r[9]), int(r[10])        # first extent only (informational: probes follow chain pointers)
        segs.append(m)
    v = rs.vertices()
    v = v[: (v.shape[0] // 8) * 8]      # GStore's slot count need not be a multiple of 8; no bucket id reaches the partial tail
    gst = capi.Store(v, rs.edges(), segs)
    eng = capi.Engine(gst, rbuf_bytes=64 << 20)
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, req, _ = load_query(q, plan)
            want = O.run_query([ostore1], pats, nvars, req)
            rc, rows, cols, tbl = eng.query(pats, nvars, req)
            assert rc == 0 and rows == want.rows, (q, plan)
            if rows:
                assert rows_equal(tbl, want.table), (q, plan)
    s, p, o = (int(x) for x in lubm1[4321])
    assert np.array_equal(gst.get_edges(s, p, O.OUT), rs.get_edges(s, p, O.OUT))
    eng.close()
    gst.close()


def test_random_graph_against_reference_engine():
    """a random graph (tests/random_bgp.py) answered by the GPU engine and by the reference's compiled engine (its answers stored
    in tests/golden/ref_random_graph_gpu.json, recomputed live where oracle/_ref is built)"""
    import random_bgp as R
    from ref_answers import answers, rows_digest
    tr, meta = R.graph(0, nv=400, ntriples=4000)
    npreds = meta["num_normal_preds"]
    ost = O.Store.build(tr, kvstore_bytes=16 << 20, num_engines=1, num_normal_preds=npreds)
    plans = {}
    for qseed in range(40):
        planned, _, nvars, req = R.query(qseed, tr, meta)
        if O.run_query([ost], planned, nvars, req, blind=True).rows <= 300_000:
            plans[str(qseed)] = (planned, nvars, req)

    def compute(lib):
        rs, out = lib.RefStore(tr, num_normal_preds=npreds), {}
        for k, (planned, nvars, req) in plans.items():
            rc, rows, _, t = rs.query(planned, nvars, req)
            out[k] = [rc, rows, rows_digest(t)]
        return out
    ref = answers("random_graph_gpu", compute)
    assert sorted(ref) == sorted(plans)
    gst = capi.Store.build(tr, npreds)
    eng = capi.Engine(gst, rbuf_bytes=256 << 20)
    checked = 0
    for k, (planned, nvars, req) in plans.items():
        rc, rows, cols, tbl = eng.query(planned, nvars, req)
        if rc == capi.WK_ERR_RBUF_OVERFLOW:
            continue
        rrc, rrows, rdg = ref[k]
        assert rc == 0 and rrc == 0 and rrows == rows and (rows == 0 or rows_digest(tbl) == rdg), (k, planned)
        checked += 1
    assert checked >= 30
    eng.close()
    gst.close()
