"""Generates tests/golden/ref_engine_lubm1.json from the reference's OWN engine (oracle/_ref/libwukong_ref.so, built by
`make -C oracle ref`): LUBM-1 (wukong_b200.datagen.lubm(1, seed=1)), Q1-Q7 x 3 plan sets -> row count and sha256 of the
lexicographically sorted result table, plus the same under DISTINCT OFFSET 1 LIMIT 40 (exact order).

    make -C oracle ref REFERENCE=<wukong checkout> && python tests/golden/make_ref_engine.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import sparql_mini as M  # noqa: E402
from conftest import PLANS, load_query  # noqa: E402
from oracle import ref as REF  # noqa: E402
from wukong_b200 import datagen  # noqa: E402


def make(univs, seed, fname):
    rs = REF.RefStore(datagen.lubm(univs, seed=seed))
    out = {"source": "SPARQLEngine (core/engine/sparql.hpp) over StaticGStore, compiled by oracle/Makefile `ref`",
           "dataset": "wukong_b200.datagen.lubm(%d, seed=%d)" % (univs, seed), "queries": {}}
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, req, _ = load_query(q, plan)
            rc, rows, cols, t = rs.query(pats, nvars, req)
            assert rc == 0
            e = {"rows": rows, "cols": cols,
                 "sha256": hashlib.sha256(M.sort_rows(t).tobytes()).hexdigest() if rows else None}
            rc, drows, _, dt = rs.query(pats, nvars, req, distinct=True, offset=1, limit=40)
            assert rc == 0
            e["distinct_rows"] = drows
            e["distinct_sha256"] = hashlib.sha256(np.ascontiguousarray(dt).tobytes()).hexdigest() if drows else None
            out["queries"]["q%d_%s" % (q, plan)] = e
    with open(os.path.join(HERE, fname), "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", fname, len(out["queries"]), "entries")


if __name__ == "__main__":
    make(1, 1, "ref_engine_lubm1.json")      # the dataset of the lubm1 / ostore1 / gstore1 fixtures (tests/conftest.py)
    make(2, 7, "ref_engine_lubm2.json")      # ... of lubm2 / ostore2 / gstore2
