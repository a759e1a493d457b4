// TEST INFRASTRUCTURE ONLY.  Compiles the reference's OWN headers (core/store/vertex.hpp,
// utils/math.hpp, core/type.hpp -- read in place from a Wukong checkout, never copied) behind a tiny
// C interface, so that the key / pointer bit layout, the hash functions, the bucket-count prime
// table, the id classes and the triple sort orders of oracle and product can be checked against
// the reference's compiled code.  This pins the DATA-STRUCTURE layer only: the store build and the
// query engine of the reference need Boost/TBB/MPI/ZeroMQ/hwloc and cannot be compiled here.
// Built by `make -C oracle ref` into oracle/_ref/ (git-ignored); tests/golden/make_ref_layout.py
// turns its outputs into the committed fixture tests/golden/ref_layout.json.
#include <stdint.h>
#include <string.h>

#include "store/vertex.hpp"   // -I $(REFERENCE)/core -I $(REFERENCE)/utils

static_assert(sizeof(ikey_t) == 8 && sizeof(iptr_t) == 8 && sizeof(vertex_t) == 16 && sizeof(edge_t) == 4,
              "reference slot / edge sizes");

extern "C" {

uint64_t ref_key_raw(uint64_t vid, uint64_t pid, uint64_t dir) {
    ikey_t k(vid, pid, dir);
    uint64_t raw;
    memcpy(&raw, &k, 8);
    return raw;
}
uint64_t ref_key_hash(uint64_t vid, uint64_t pid, uint64_t dir) { return ikey_t(vid, pid, dir).hash(); }
uint64_t ref_ptr_raw(uint64_t size, uint64_t off, uint64_t type) {
    iptr_t p(size, off, type);
    uint64_t raw;
    memcpy(&raw, &p, 8);
    return raw;
}
uint64_t ref_hash_u64(uint64_t x) { return wukong::math::hash_u64(x); }
int ref_hash_mod(uint64_t n, int m) { return wukong::math::hash_mod(n, m); }   // owner of a vertex: vid % num_servers
uint64_t ref_hash_prime_u64(uint64_t upper) { return wukong::math::hash_prime_u64(upper); }
int ref_is_tpid(int64_t id) { return is_tpid((ssid_t)id) ? 1 : 0; }
int ref_is_vid(int64_t id) { return is_vid((ssid_t)id) ? 1 : 0; }
int ref_less_pso(const uint32_t *a, const uint32_t *b) { return triple_sort_by_pso()(triple_t(a[0], a[1], a[2]), triple_t(b[0], b[1], b[2])) ? 1 : 0; }
int ref_less_pos(const uint32_t *a, const uint32_t *b) { return triple_sort_by_pos()(triple_t(a[0], a[1], a[2]), triple_t(b[0], b[1], b[2])) ? 1 : 0; }
int ref_consts(int which) {
    switch (which) {
    case 0: return NBITS_DIR;
    case 1: return NBITS_IDX;
    case 2: return NBITS_VID;
    case 3: return PREDICATE_ID;
    case 4: return TYPE_ID;
    case 5: return NBITS_SIZE;
    case 6: return NBITS_PTR;
    case 7: return NBITS_TYPE;
    default: return -1;
    }
}

}  // extern "C"
