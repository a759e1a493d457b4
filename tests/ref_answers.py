"""Answers of the reference's own compiled code (oracle/_ref), stored as tests/golden/ref_<name>.json so that the tests that
compare against the reference run without a Wukong checkout.  Where oracle/_ref is built, the answers are recomputed live
and must equal the stored ones; with WUKONG_WRITE_GOLDEN=1 the live answers replace the stored file instead."""
import hashlib
import json
import os

import numpy as np

import sparql_mini as M
from oracle import ref as REF

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def live():
    try:
        return REF.build()
    except OSError:
        return False


def answers(name, compute):
    """compute(REF) -> JSON-able answers of the live reference; returns them, or the stored ones where there is no reference"""
    path = os.path.join(GOLDEN, "ref_%s.json" % name)
    if not live():
        with open(path) as f:
            return json.load(f)
    got = json.loads(json.dumps(compute(REF)))
    if os.environ.get("WUKONG_WRITE_GOLDEN"):
        with open(path, "w") as f:
            json.dump(got, f, separators=(",", ":"), sort_keys=True)
    else:
        with open(path) as f:
            assert got == json.load(f), "the live reference disagrees with " + path
    return got


def rows_digest(t):
    """sha256 of a table as a multiset of rows (None for no table)"""
    if t is None:
        return None
    t = np.asarray(t, dtype=np.uint32)
    if t.size == 0:
        return None
    return hashlib.sha256(M.sort_rows(t).tobytes()).hexdigest()


def exact_digest(t):
    """sha256 of a table in its row order"""
    return hashlib.sha256(np.ascontiguousarray(t, dtype=np.uint32).tobytes()).hexdigest()


class EdgeDigest:
    """running sha256 over (key, edge list) pairs"""

    def __init__(self):
        self.h = hashlib.sha256()

    def add(self, key, edges):
        e = np.ascontiguousarray(edges, dtype=np.uint32)
        self.h.update(np.array([key, e.size], dtype=np.uint64).tobytes())
        self.h.update(e.tobytes())

    def hexdigest(self):
        return self.h.hexdigest()
