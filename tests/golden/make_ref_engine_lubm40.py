"""Generates tests/golden/ref_engine_lubm40.json from the reference's OWN engine (oracle/_ref/libwukong_ref.so, built by
`make -C oracle ref`) at BASELINE config 2: LUBM-40 (wukong_b200.datagen.lubm(40, seed=1), ~5.5 M triples), Q1-Q7 x 3 plan
sets -> row count, column count, sha256 of the lexicographically sorted result table, and the order-independent 64-bit
digest (oracle.ref.table_digest) that bench.py also uses at LUBM-2560.  The store is the reference's own StaticGStore
build of the same triples.

    make -C oracle ref REFERENCE=<wukong checkout> && python tests/golden/make_ref_engine_lubm40.py
"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sparql_mini as M  # noqa: E402
from conftest import PLANS, load_query  # noqa: E402
from oracle import ref as REF  # noqa: E402
from wukong_b200 import datagen  # noqa: E402


def main():
    t0 = time.time()
    tr = datagen.lubm(40, seed=1)
    rs = REF.RefStore(tr, memstore_gb=4)
    print("reference store built in %.1f s (%d triples)" % (time.time() - t0, tr.shape[0]))
    out = {"source": "SPARQLEngine (core/engine/sparql.hpp) over StaticGStore, compiled by oracle/Makefile `ref`",
           "dataset": "wukong_b200.datagen.lubm(40, seed=1)", "triples": int(tr.shape[0]), "queries": {}}
    for q in range(1, 8):
        for plan in PLANS:
            pats, nvars, req, _ = load_query(q, plan)
            rc, rows, cols, t = rs.query(pats, nvars, req)
            assert rc == 0, (q, plan, rc)
            out["queries"]["q%d_%s" % (q, plan)] = {
                "rows": rows, "cols": cols,
                "sha256": hashlib.sha256(M.sort_rows(t).tobytes()).hexdigest() if rows else None,
                "digest": REF.table_digest(t) if rows else 0}
            print("q%d %s: %d rows" % (q, plan, rows))
    with open(os.path.join(HERE, "ref_engine_lubm40.json"), "w") as f:
        json.dump(out, f, indent=0)
    print("wrote ref_engine_lubm40.json in %.1f s" % (time.time() - t0))


if __name__ == "__main__":
    main()
