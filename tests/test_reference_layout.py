"""CPU: the data-structure layer of oracle and product against the reference's OWN compiled headers.

tests/golden/ref_layout.json holds outputs of core/store/vertex.hpp (ikey_t, iptr_t, is_tpid, is_vid),
utils/math.hpp (hash_u64, hash_mod, hash_prime_u64) and core/type.hpp (triple sort orders) compiled from the
reference tree (oracle/Makefile `ref`, tests/golden/make_ref_layout.py).  When oracle/_ref exists (build
container) the live library is checked against the fixture as well."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from wukong_b200 import capi

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "ref_layout.json")))


def test_constants():
    c = G["consts"]
    assert (c["NBITS_DIR"], c["NBITS_IDX"], c["NBITS_VID"]) == (1, capi.WK_NBITS_IDX if hasattr(capi, "WK_NBITS_IDX") else 17, 46)
    assert (c["NBITS_SIZE"], c["NBITS_PTR"], c["NBITS_TYPE"]) == (28, 34, 2)
    assert (c["PREDICATE_ID"], c["TYPE_ID"]) == (O.PREDICATE_ID, O.TYPE_ID)


def test_key_layout_and_hash():
    L, Lo = capi.lib(), O.lib()
    for vid, pid, d, raw, h in G["keys"]:
        assert Lo.wko_make_key(vid, pid, d) == raw
        assert Lo.wko_hash_u64(raw) == h                       # ikey_t::hash() == hash_u64(raw bits)
        assert L.wk_selftest_make_key(vid, pid, d) == raw
        assert L.wk_selftest_hash(raw) == h
    for x, h in G["hash_u64"]:
        assert Lo.wko_hash_u64(x) == h and L.wk_selftest_hash(x) == h


def test_pointer_layout():
    L, Lo = capi.lib(), O.lib()
    for size, off, raw in G["ptrs"]:
        assert Lo.wko_make_ptr(size, off) == raw
        assert L.wk_selftest_ptr_size(raw) == size and L.wk_selftest_ptr_off(raw) == off


def test_bucket_prime_owner_and_id_classes():
    Lo = O.lib()
    for up, p in G["hash_prime_u64"]:
        assert Lo.wko_hash_prime_u64(up) == p
    for v, n, o in G["owner"]:
        assert v % n == o                                      # math::hash_mod: the sharding rule used everywhere
    for i, tp, vd in G["id_class"]:
        assert Lo.wko_is_tpid(i) == tp
        assert (1 if i >= (1 << 17) else 0) == vd


def test_triple_sort_orders():
    Lo = O.lib()
    for a, b, pso, pos in G["triple_order"]:
        a = np.array(a, dtype=np.uint32); b = np.array(b, dtype=np.uint32)
        assert Lo.wko_less_pso(a.ctypes.data, b.ctypes.data) == pso
        assert Lo.wko_less_pos(a.ctypes.data, b.ctypes.data) == pos
        # the product builders order by the packed (p, s, o) / (p, o, s) tuple
        assert int(tuple(a[[1, 0, 2]]) < tuple(b[[1, 0, 2]])) == pso
        assert int(tuple(a[[1, 2, 0]]) < tuple(b[[1, 2, 0]])) == pos


def test_fixture_matches_live_reference_headers():
    from oracle import ref as REF
    REF.build()                      # builds oracle/_ref where $WUKONG_REFERENCE names a Wukong checkout
    lib = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libwukong_ref_layout.so")
    if not os.path.exists(lib):
        pytest.skip("oracle/_ref not built (needs a Wukong checkout in $WUKONG_REFERENCE)")
    L = C.CDLL(lib)
    u64 = C.c_uint64
    for n, k in (("ref_key_raw", 3), ("ref_key_hash", 3), ("ref_ptr_raw", 3), ("ref_hash_u64", 1), ("ref_hash_prime_u64", 1)):
        getattr(L, n).restype = u64
        getattr(L, n).argtypes = [u64] * k
    for vid, pid, d, raw, h in G["keys"]:
        assert L.ref_key_raw(vid, pid, d) == raw and L.ref_key_hash(vid, pid, d) == h
    for size, off, raw in G["ptrs"]:
        assert L.ref_ptr_raw(size, off, 0) == raw
    for x, h in G["hash_u64"]:
        assert L.ref_hash_u64(x) == h
    for up, p in G["hash_prime_u64"]:
        assert L.ref_hash_prime_u64(up) == p
