import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

WORKLOADS = os.path.join(ROOT, "workloads", "lubm", "basic")
PLANS = ["osdi16_plan", "optimal2560_plan", "optimal10240_plan"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _ensure_built():
    from wukong_b200 import build
    from oracle import oracle as O
    build.build_all()
    O.build()


@pytest.fixture(scope="session", autouse=True)
def built():
    _ensure_built()


def load_query(q, plan):
    """-> (planned patterns, nvars, required_vars, raw patterns) via the independent Python reader."""
    import sparql_mini as M
    text = open(os.path.join(WORKLOADS, "lubm_q%d" % q)).read()
    fmt = open(os.path.join(WORKLOADS, plan, "lubm_q%d.fmt" % q)).read()
    pats, nvars, req = M.parse_query(text)
    return M.apply_plan(pats, fmt), nvars, req, pats


@pytest.fixture(scope="session")
def lubm1():
    from wukong_b200 import datagen
    return datagen.lubm(1, seed=1)


@pytest.fixture(scope="session")
def lubm2():
    from wukong_b200 import datagen
    return datagen.lubm(2, seed=7)


@pytest.fixture(scope="session")
def ostore1(lubm1):
    from oracle import oracle as O
    return O.Store.build(lubm1, kvstore_bytes=32 << 20, num_engines=4)


@pytest.fixture(scope="session")
def ostore2(lubm2):
    from oracle import oracle as O
    return O.Store.build(lubm2, kvstore_bytes=48 << 20, num_engines=3)


def has_gpu():
    try:
        from wukong_b200 import capi
        return capi.device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gstore1(ostore1):
    from wukong_b200 import capi
    st = capi.Store(ostore1.vertices(), ostore1.edges(), ostore1.segs())
    yield st
    st.close()


@pytest.fixture(scope="session")
def gstore2(ostore2):
    from wukong_b200 import capi
    st = capi.Store(ostore2.vertices(), ostore2.edges(), ostore2.segs())
    yield st
    st.close()


def rows_equal(a, b):
    """bit-exact equality of two binding tables as multisets of rows"""
    import sparql_mini as M
    a = np.asarray(a, dtype=np.uint32)
    b = np.asarray(b, dtype=np.uint32)
    if a.size == 0 and b.size == 0:
        return True
    if a.shape != b.shape:
        return False
    return bool((M.sort_rows(a) == M.sort_rows(b)).all())
