"""TEST INFRASTRUCTURE ONLY: ctypes access to oracle/_ref/libwukong_ref.so -- the reference's OWN store (StaticGStore) and
query engine (SPARQLEngine) compiled from a Wukong source checkout ($WUKONG_REFERENCE) behind C shims
(oracle/ref_store_shim.cpp, ref_engine_shim.cpp, third-party stand-ins in oracle/ref_stubs/).  Exists only where
`make -C oracle ref REFERENCE=...` has run.  Used to pin the oracle and to make the fixtures under tests/golden/; never by
the product."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libwukong_ref.so")
_lib = None


GPU_LIB = os.path.join(HERE, "_ref", "libwukong_ref_gpu.so")
_gpu_lib = None


def available():
    return os.path.exists(LIB)


def gpu_binding_available():
    return os.path.exists(GPU_LIB)


def gpu_lib():
    """the reference's GPUEngine over integration/gpu_engine_cuda.hpp (ref_gpu_engine_shim.cpp); needs a GPU to run a query"""
    global _gpu_lib
    if _gpu_lib is None:
        L = C.CDLL(GPU_LIB)
        u64, vp, ci = C.c_uint64, C.c_void_p, C.c_int
        L.refs_build.restype = vp
        L.refs_build.argtypes = [vp, u64, ci, ci, ci, ci, ci]
        L.refg_query.argtypes = [vp, vp, ci, ci, vp, ci, ci, ci, vp, u64, C.POINTER(u64), C.POINTER(ci)]
        L.refs_get_edges.restype = u64
        L.refs_get_edges.argtypes = [vp, C.c_uint32, C.c_uint32, ci, C.POINTER(vp)]
        _gpu_lib = L
    return _gpu_lib


class RefGpuEngine:
    """a store built by the reference's StaticGStore::init, queried through the reference's GPUEngine::execute_one_pattern
    whose backend is the replacement GPUEngineCuda (calls into libwukong_b200.so)"""

    def __init__(self, triples, num_normal_preds=31, memstore_gb=1):
        t = np.ascontiguousarray(triples, dtype=np.uint32).reshape(-1, 3)
        self.h = gpu_lib().refs_build(t.ctypes.data_as(C.c_void_p), t.shape[0], 1, 0, 1, memstore_gb, num_normal_preds)
        self._out = np.empty(1 << 24, dtype=np.uint32)

    def get_edges(self, vid, pid, d):
        """GStore::get_edges of the store built under -DUSE_GPU (CPU probe)"""
        p = C.c_void_p()
        n = gpu_lib().refs_get_edges(self.h, vid, pid, d, C.byref(p))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint32)), shape=(n,)).copy() if n else np.zeros(0, np.uint32)

    def query(self, patterns, nvars, required, blind=False, rbuf_mb=64):
        """-> (status, rows, cols, raw table of the pattern phase: one column per bound variable, in binding order)"""
        p = np.array(patterns, dtype=np.int32).reshape(-1, 4)
        rq = np.array(required, dtype=np.int32)
        rows, cols = C.c_uint64(0), C.c_int(0)
        rc = gpu_lib().refg_query(self.h, p.ctypes.data_as(C.c_void_p), p.shape[0], nvars, rq.ctypes.data_as(C.c_void_p) if len(rq) else None,
                                  len(rq), 1 if blind else 0, rbuf_mb, self._out.ctypes.data_as(C.c_void_p), self._out.size,
                                  C.byref(rows), C.byref(cols))
        tbl = None
        if rc == 0 and not blind and cols.value:
            tbl = self._out[: rows.value * cols.value].reshape(rows.value, cols.value).copy()
        return rc, rows.value, cols.value, tbl


def reference_tree():
    """the Wukong source checkout named by $WUKONG_REFERENCE, or None"""
    p = os.environ.get("WUKONG_REFERENCE", "")
    return p if p and os.path.isdir(os.path.join(p, "core")) else None


def build():
    """(re)build oracle/_ref when a reference tree is given ($WUKONG_REFERENCE); returns availability"""
    ref = reference_tree()
    if ref:
        import subprocess
        subprocess.check_call(["make", "-C", HERE, "ref", "REFERENCE=" + ref], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        u64, vp, ci, i64 = C.c_uint64, C.c_void_p, C.c_int, C.c_int64
        L.refs_build.restype = vp
        L.refs_build.argtypes = [vp, u64, ci, ci, ci, ci, ci]
        for n in ("refs_num_slots", "refs_num_buckets", "refs_num_entries", "refs_last_ext", "refs_last_entry"):
            getattr(L, n).restype = u64
            getattr(L, n).argtypes = [vp]
        L.refs_vertices.restype = vp
        L.refs_vertices.argtypes = [vp]
        L.refs_edges.restype = vp
        L.refs_edges.argtypes = [vp]
        L.refs_num_segs.argtypes = [vp]
        L.refs_segs.restype = vp
        L.refs_segs.argtypes = [vp]
        L.refs_get_edges.restype = u64
        L.refs_get_edges.argtypes = [vp, C.c_uint32, C.c_uint32, ci, C.POINTER(vp)]
        L.refe_query.argtypes = [vp, vp, ci, ci, vp, ci, ci, ci, ci, i64, i64, vp, u64, C.POINTER(u64), C.POINTER(ci)]
        L.refs_adopt.restype = vp
        L.refs_adopt.argtypes = [vp, u64, u64, vp, u64, vp, ci, ci]
        L.refe_time_query.argtypes = [vp, vp, ci, ci, vp, ci, ci, ci, ci, ci, vp, C.POINTER(u64)]
        L.refe_time_query_digest.argtypes = [vp, vp, ci, ci, vp, ci, ci, ci, ci, ci, vp, C.POINTER(u64), C.POINTER(u64)]
        L.refe_cluster_query.argtypes = [vp, ci, vp, ci, ci, vp, ci, ci, vp, u64, C.POINTER(u64), C.POINTER(ci)]
        L.refp_set_plan.argtypes = [vp, ci, C.c_char_p, vp, ci]
        L.refe_fork_plan.argtypes = [vp, vp, ci, ci, ci, vp]
        L.refe_split.argtypes = [vp, vp, u64, ci, ci, ci, vp, vp]
        _lib = L
    return _lib


def encode_group(group):
    """group = (patterns, unions, optionals) with patterns a list of (s, p, d, o) and unions / optionals lists of groups
    -> the int32 tree the shims and the host mirror exchange"""
    pats, unions, optionals = group
    out = [len(pats)]
    for t in pats:
        out += [int(x) for x in t]
    out.append(len(unions))
    for u in unions:
        out += encode_group(u)
    out.append(len(optionals))
    for o in optionals:
        out += encode_group(o)
    return out


def decode_group(a, pos=0):
    n = a[pos]; pos += 1
    pats = [tuple(int(x) for x in a[pos + 4 * i: pos + 4 * i + 4]) for i in range(n)]
    pos += 4 * n
    subs = []
    for _ in range(2):
        k = a[pos]; pos += 1
        lst = []
        for _ in range(k):
            g, pos = decode_group(a, pos)
            lst.append(g)
        subs.append(lst)
    return (pats, subs[0], subs[1]), pos


def set_plan_tree(group, fmt_text):
    """Planner::set_plan on a group tree (UNION / OPTIONAL blocks, core/planner.hpp:1722-1738) -> planned tree or None"""
    a = np.array(encode_group(group), dtype=np.int32)
    out = np.zeros(4096, dtype=np.int32)
    L = lib()
    L.refp_set_plan_tree.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int]
    n = L.refp_set_plan_tree(a.ctypes.data_as(C.c_void_p), a.size, fmt_text.encode(), out.ctypes.data_as(C.c_void_p), out.size)
    if n < 0:
        return None
    return decode_group(out[:n].tolist())[0]


def load_config(fname, nsrvs, reload=""):
    """the reference's load_config(fname, nsrvs) [+ reload_config(reload)] (core/config.hpp:160-230, non-GPU build without an
    RDMA device) -> dict of the Global items in the order of wukong_b200.host.CONFIG_ITEMS, plus input_folder"""
    from wukong_b200.host import CONFIG_ITEMS
    L = lib()
    L.refc_load_config.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    out = np.zeros(len(CONFIG_ITEMS), dtype=np.int32)
    folder = C.create_string_buffer(4096)
    n = L.refc_load_config(fname.encode(), nsrvs, reload.encode(), out.ctypes.data_as(C.c_void_p), len(out), folder, 4096)
    assert n == len(CONFIG_ITEMS), n
    d = {k: int(v) for k, v in zip(CONFIG_ITEMS, out)}
    d["input_folder"] = folder.value.decode()
    return d


def table_digest(table):
    """order-independent digest of a binding table (a multiset of rows): sum over rows of a 64-bit mix of the row's words,
    modulo 2^64 -- the same function as row_digest() in ref_engine_shim.cpp"""
    t = np.asarray(table, dtype=np.uint32)
    if t.size == 0:
        return 0
    t = t.reshape(t.shape[0], -1)
    with np.errstate(over="ignore"):
        h = np.full(t.shape[0], 0x9E3779B97F4A7C15, dtype=np.uint64)
        for c in range(t.shape[1]):
            h = (h ^ t[:, c].astype(np.uint64)) * np.uint64(0xBF58476D1CE4E5B9)
            h ^= h >> np.uint64(29)
        h *= np.uint64(0x94D049BB133111EB)
        h ^= h >> np.uint64(32)
        return int(h.sum(dtype=np.uint64))


def cluster_query(stores, patterns, nvars, required):
    """one query over n shard stores (RefStore(..., num_servers=n, sid=i)) driven by the reference's per-server functions:
    execute_one_pattern, need_fork_join, generate_sub_query, final_process.  -> (status, rows, cols, table or None)"""
    n = len(stores)
    arr = (C.c_void_p * n)(*[s.h for s in stores])
    p = np.array(patterns, dtype=np.int32).reshape(-1, 4)
    rq = np.array(required, dtype=np.int32)
    out = np.empty(1 << 24, dtype=np.uint32)
    rows, cols = C.c_uint64(0), C.c_int(0)
    rc = lib().refe_cluster_query(C.cast(arr, C.c_void_p), n, p.ctypes.data_as(C.c_void_p), p.shape[0], nvars,
                                  rq.ctypes.data_as(C.c_void_p) if len(rq) else None, len(rq), 0,
                                  out.ctypes.data_as(C.c_void_p), out.size, C.byref(rows), C.byref(cols))
    tbl = out[: rows.value * cols.value].reshape(rows.value, cols.value).copy() if (rc == 0 and cols.value) else None
    return rc, rows.value, cols.value, tbl


def set_plan(patterns, fmt_text):
    """Planner::set_plan + set_direction (core/planner.hpp:1647-1754) -> planned patterns, or None when refused"""
    a = np.array(patterns, dtype=np.int32).reshape(-1, 4)
    out = np.zeros((64, 4), dtype=np.int32)
    n = lib().refp_set_plan(a.ctypes.data_as(C.c_void_p), a.shape[0], fmt_text.encode(), out.ctypes.data_as(C.c_void_p), 64)
    if n < 0:
        return None
    return [tuple(int(x) for x in row) for row in out[:n]]


class RefStore:
    """One server's store built by the reference's StaticGStore::init (CPU build: 256-bucket ext extents; 1 GiB kvstore)."""

    def __init__(self, triples, num_servers=1, sid=0, num_normal_preds=31, memstore_gb=1):
        t = np.ascontiguousarray(triples, dtype=np.uint32).reshape(-1, 3)
        self.h = lib().refs_build(t.ctypes.data_as(C.c_void_p), t.shape[0], num_servers, sid, 1, memstore_gb, num_normal_preds)
        self._out = np.empty(1 << 22, dtype=np.uint32)

    @classmethod
    def adopt(cls, vertices, edges, segs, num_normal_preds=31):
        """a reference GStore over existing store arrays (e.g. the host builder's); segs: objects with the wk_segmeta_t fields"""
        self = cls.__new__(cls)
        v = np.ascontiguousarray(vertices, dtype=np.uint64).reshape(-1, 2)
        e = np.ascontiguousarray(edges, dtype=np.uint32)
        rows = np.array([[x.index, x.dir, x.pid, x.num_keys, x.num_buckets, x.bucket_start, x.num_edges, x.edge_start,
                          x.ext_start, x.ext_num] for x in segs], dtype=np.uint64)
        main = int(max(int(r[5]) + int(r[4]) for r in rows))
        self._keep = (v, e, rows)
        self.h = lib().refs_adopt(v.ctypes.data_as(C.c_void_p), v.shape[0], main, e.ctypes.data_as(C.c_void_p), e.shape[0],
                                  rows.ctypes.data_as(C.c_void_p), rows.shape[0], num_normal_preds)
        self._out = np.empty(1 << 22, dtype=np.uint32)
        return self

    def time_query(self, patterns, nvars, required, reps=1, mt_factor=1, threaded=True, blind=False, digest=False):
        """-> (status, usec[reps], rows[, digest]): wall time of pattern phase (mt_factor slices on host threads) + merge +
        final_process; digest = table_digest() of the last repetition's final table (computed outside the timed region)"""
        p = np.array(patterns, dtype=np.int32).reshape(-1, 4)
        rq = np.array(required, dtype=np.int32)
        us = np.zeros(reps, dtype=np.float64)
        rows, dg = C.c_uint64(0), C.c_uint64(0)
        rc = lib().refe_time_query_digest(self.h, p.ctypes.data_as(C.c_void_p), p.shape[0], nvars,
                                          rq.ctypes.data_as(C.c_void_p) if len(rq) else None, len(rq), 1 if blind else 0, mt_factor,
                                          1 if threaded else 0, reps, us.ctypes.data_as(C.c_void_p), C.byref(rows),
                                          C.byref(dg) if digest else None)
        if digest:
            return rc, us, rows.value, dg.value
        return rc, us, rows.value

    @property
    def num_slots(self):
        return lib().refs_num_slots(self.h)

    def vertices(self):
        n = self.num_slots
        return np.frombuffer((C.c_uint64 * (2 * n)).from_address(lib().refs_vertices(self.h)), dtype=np.uint64).reshape(n, 2)

    def edges(self):
        n = lib().refs_last_entry(self.h)
        return np.frombuffer((C.c_uint32 * max(n, 1)).from_address(lib().refs_edges(self.h)), dtype=np.uint32)[:n]

    def segs(self):
        """rows of (index, dir, pid, num_keys, num_buckets, bucket_start, num_edges, edge_start, n_ext, ext0_start, ext0_num)"""
        n = lib().refs_num_segs(self.h)
        return np.frombuffer((C.c_uint64 * (11 * n)).from_address(lib().refs_segs(self.h)), dtype=np.uint64).reshape(n, 11).copy()

    def get_edges(self, vid, pid, d):
        """GStore::get_edges_local (gstore.hpp:393-410)"""
        out = C.c_void_p()
        n = lib().refs_get_edges(self.h, vid, pid, d, C.byref(out))
        if n == 0 or not out.value:
            return np.zeros(0, dtype=np.uint32)
        return np.frombuffer((C.c_uint32 * n).from_address(out.value), dtype=np.uint32).copy()

    def fork_plan(self, patterns, nvars, n):
        """per step: -1 no exchange, -2 replicate, c >= 0 re-shard by column c -- need_fork_join / dispatch decisions of the
        reference engine for a store sharded over n servers (RDMA rule, threshold 0).  -> (status, list)"""
        p = np.array(patterns, dtype=np.int32).reshape(-1, 4)
        out = np.zeros(p.shape[0], dtype=np.int32)
        rc = lib().refe_fork_plan(self.h, p.ctypes.data_as(C.c_void_p), p.shape[0], nvars, n, out.ctypes.data_as(C.c_void_p))
        return rc, out.tolist()

    def split(self, table, col, n):
        """SPARQLEngine::generate_sub_query: -> list of n sub-tables"""
        t = np.ascontiguousarray(table, dtype=np.uint32)
        out = np.empty_like(t)
        counts = np.zeros(n, dtype=np.uint64)
        lib().refe_split(self.h, t.ctypes.data_as(C.c_void_p), t.shape[0], t.shape[1], col, n, out.ctypes.data_as(C.c_void_p),
                         counts.ctypes.data_as(C.c_void_p))
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        return [out[offs[i]:offs[i + 1]] for i in range(n)]

    def query(self, patterns, nvars, required, blind=False, mt_factor=1, distinct=False, offset=0, limit=-1):
        """SPARQLEngine::execute_one_pattern until done, then final_process.  -> (status, rows, cols, table or None)"""
        p = np.array(patterns, dtype=np.int32).reshape(-1, 4)
        rq = np.array(required, dtype=np.int32)
        while True:
            rows, cols = C.c_uint64(0), C.c_int(0)
            rc = lib().refe_query(self.h, p.ctypes.data_as(C.c_void_p), p.shape[0], nvars,
                                  rq.ctypes.data_as(C.c_void_p) if len(rq) else None, len(rq), 1 if blind else 0, mt_factor,
                                  1 if distinct else 0, offset, limit, self._out.ctypes.data_as(C.c_void_p), self._out.size,
                                  C.byref(rows), C.byref(cols))
            if rc == -1:   # table larger than the staging buffer
                self._out = np.empty(self._out.size * 4, dtype=np.uint32)
                continue
            break
        tbl = None
        if rc == 0 and not blind and cols.value:
            tbl = self._out[: rows.value * cols.value].reshape(rows.value, cols.value).copy()
        return rc, rows.value, cols.value, tbl
