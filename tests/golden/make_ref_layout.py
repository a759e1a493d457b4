"""Generates tests/golden/ref_layout.json from the reference's OWN compiled headers
(oracle/_ref/libwukong_ref_layout.so, built by `make -C oracle ref` from core/store/vertex.hpp of a Wukong checkout,
utils/math.hpp and core/type.hpp).  Run where a Wukong checkout is available:

    make -C oracle ref REFERENCE=<wukong checkout> && python tests/golden/make_ref_layout.py
"""
import ctypes as C
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def load():
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libwukong_ref_layout.so"))
    u64 = C.c_uint64
    for n, args in (("ref_key_raw", [u64] * 3), ("ref_key_hash", [u64] * 3), ("ref_ptr_raw", [u64] * 3),
                    ("ref_hash_u64", [u64]), ("ref_hash_prime_u64", [u64])):
        getattr(L, n).restype = u64
        getattr(L, n).argtypes = args
    L.ref_hash_mod.argtypes = [u64, C.c_int]
    L.ref_is_tpid.argtypes = [C.c_int64]
    L.ref_is_vid.argtypes = [C.c_int64]
    L.ref_less_pso.argtypes = [C.c_void_p, C.c_void_p]
    L.ref_less_pos.argtypes = [C.c_void_p, C.c_void_p]
    return L


def main():
    L = load()
    rng = np.random.default_rng(20260922)
    out = {"source": "reference headers core/store/vertex.hpp, utils/math.hpp, core/type.hpp compiled by oracle/Makefile `ref`",
           "consts": {n: L.ref_consts(i) for i, n in enumerate(
               ["NBITS_DIR", "NBITS_IDX", "NBITS_VID", "PREDICATE_ID", "TYPE_ID", "NBITS_SIZE", "NBITS_PTR", "NBITS_TYPE"])}}
    keys = []
    vids = [0, 1, (1 << 17), (1 << 17) + 1, (1 << 32) - 1, (1 << 46) - 1] + [int(x) for x in rng.integers(0, 1 << 46, 60)]
    for i, vid in enumerate(vids):
        pid = [0, 1, 2, 17, (1 << 17) - 1][i % 5] if i < 10 else int(rng.integers(0, 1 << 17))
        d = i & 1
        keys.append([vid, pid, d, L.ref_key_raw(vid, pid, d), L.ref_key_hash(vid, pid, d)])
    out["keys"] = keys                                        # vid, pid, dir, raw bits, ikey_t::hash()
    ptrs = []
    for i in range(40):
        size = [0, 1, (1 << 28) - 1][i] if i < 3 else int(rng.integers(0, 1 << 28))
        off = [0, 1, (1 << 34) - 1][i] if i < 3 else int(rng.integers(0, 1 << 34))
        ptrs.append([size, off, L.ref_ptr_raw(size, off, 0)])
    out["ptrs"] = ptrs                                        # size, off, raw bits (type = sid)
    hs = [0, 1, 2, (1 << 64) - 1, 0x123456789ABCDEF] + [int(x) for x in rng.integers(0, 1 << 63, 60)]
    out["hash_u64"] = [[x, L.ref_hash_u64(x)] for x in hs]
    ups = [98317, 98318, 196612, 196613, 1 << 20, 3145739, 50331653 + 7, 123456789, 1610612741, (1 << 31) - 1] + \
          [int(x) for x in rng.integers(98317, 1 << 31, 30)]
    out["hash_prime_u64"] = [[x, L.ref_hash_prime_u64(x)] for x in ups]
    out["owner"] = [[int(v), int(n), L.ref_hash_mod(int(v), int(n))] for v, n in
                    zip(rng.integers(0, 1 << 32, 30), rng.integers(1, 9, 30))]
    ids = [-5, -1, 0, 1, 2, 3, (1 << 17) - 1, 1 << 17, (1 << 17) + 1, 1 << 30]
    out["id_class"] = [[i, L.ref_is_tpid(i), L.ref_is_vid(i)] for i in ids]
    tri = rng.integers(1, 6, (60, 2, 3)).astype(np.uint32)    # small domain: many ties on every component
    less = []
    for a, b in tri:
        a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
        less.append([a.tolist(), b.tolist(), L.ref_less_pso(a.ctypes.data, b.ctypes.data), L.ref_less_pos(a.ctypes.data, b.ctypes.data)])
    out["triple_order"] = less                                # a, b, pso(a<b), pos(a<b)
    with open(os.path.join(HERE, "ref_layout.json"), "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", len(keys), "keys,", len(ptrs), "ptrs,", len(hs), "hashes")


if __name__ == "__main__":
    main()
