// =============================================================================================
// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product.
//
// CPU restatement of the reference's (SJTU-IPADS/wukong) graph-exploration hot path, written
// from the behaviour of the files cited below.  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load this library; the product path
// (wukong_b200/) never does and fails loudly when its CUDA library is missing.
//
// PARITY PINNING: the reference's own tests hold NO golden vectors for this path (SURVEY.md §4, §8c), and its build
// (CMake + Boost / TBB / ZeroMQ / MPI / hwloc, none in this image) cannot be run.  What IS done: the reference's OWN
// sources are compiled in place, behind C shims and std-based stand-ins for those third-party containers
// (oracle/Makefile `ref`, oracle/ref_*_shim.cpp, oracle/ref_stubs/), into oracle/_ref:
//   * core/store/vertex.hpp, utils/math.hpp, core/type.hpp        -> key / pointer layout, hashes, primes, sort orders
//   * core/store/static_gstore.hpp + gstore.hpp + meta.hpp + mem.hpp -> store build (StaticGStore::init) and probe
//   * core/engine/sparql.hpp + core/query.hpp                     -> SPARQLEngine: dispatch, every pattern function,
//                                                                     final_process (DISTINCT / OFFSET / LIMIT / projection)
// tests/test_reference_layout.py and tests/test_reference_pin.py hold this oracle to that compiled code: segment tables,
// key sets and every key's edge list on LUBM-1; Q1-Q7 x 3 plan sets x mt 1/3, blind counts, modifiers, error codes; a
// random graph x 60 random plans; and the committed fixtures tests/golden/ref_layout.json, ref_engine_lubm1.json.
// Not covered by the pin: the loader's file reading, the fork-join transport, the proxy (and the stand-ins are mine).
// Further, independent checks: the gsck invariants (gchecker.hpp:132-360) restated in wko_store_check, and a brute-force
// triple-scan joiner (tests/sparql_mini.py) on LUBM and on random graphs.
//
// All file:line citations are relative to the root of a Wukong checkout.
// =============================================================================================
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

namespace wko {

typedef uint32_t sid_t;   // core/type.hpp:34-38 (DTYPE_64BIT off)
typedef int32_t ssid_t;
static const sid_t BLANK_ID = UINT32_MAX;

enum { DIR_IN = 0, DIR_OUT = 1 };            // core/type.hpp:127
enum { PREDICATE_ID = 0, TYPE_ID = 1 };      // store/vertex.hpp:38
enum { NBITS_DIR = 1, NBITS_IDX = 17, NBITS_VID = 46 };  // store/vertex.hpp:33-35
enum { NBITS_SIZE = 28, NBITS_PTR = 34 };    // store/vertex.hpp:112-114
static const int ASSOCIATIVITY = 8;          // store/gstore.hpp:967

static inline bool is_tpid(int64_t id) { return id > 1 && id < (1 << NBITS_IDX); }  // vertex.hpp:40

// error codes, utils/errors.hpp:28-43
enum { SUCCESS = 0, UNKNOWN_ERROR, SYNTAX_ERROR, UNKNOWN_PATTERN, ATTR_DISABLE, NO_REQUIRED_VAR,
       UNSUPPORT_UNION, OBJ_ERROR, VERTEX_INVALID, UNKNOWN_SUB, SETTING_ERROR, FIRST_PATTERN_ERROR,
       UNKNOWN_FILTER };
struct OracleError { int code; };
#define O_ASSERT_CODE(cond, code) do { if (!(cond)) throw OracleError{code}; } while (0)
#define O_ASSERT(cond) do { if (!(cond)) { fprintf(stderr, "oracle assert failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); abort(); } } while (0)

// ---- key / pointer bit layout: store/vertex.hpp:47-66 (ikey_t), :116-119 (iptr_t) -------------
// ikey_t bitfields are declared dir:1, pid:17, vid:46 (LSB first on x86-64 gcc).
static inline uint64_t make_key(uint64_t vid, uint64_t pid, uint64_t dir) {
    return (vid << (NBITS_IDX + NBITS_DIR)) | (pid << NBITS_DIR) | dir;
}
static inline uint64_t key_vid(uint64_t k) { return k >> (NBITS_IDX + NBITS_DIR); }
static inline uint64_t key_pid(uint64_t k) { return (k >> NBITS_DIR) & ((1u << NBITS_IDX) - 1); }
static inline uint64_t key_dir(uint64_t k) { return k & 1; }
// iptr_t bitfields: size:28, off:34, type:2
static inline uint64_t make_ptr(uint64_t size, uint64_t off) { return size | (off << NBITS_SIZE); }
static inline uint64_t ptr_size(uint64_t p) { return p & ((1ull << NBITS_SIZE) - 1); }
static inline uint64_t ptr_off(uint64_t p) { return (p >> NBITS_SIZE) & ((1ull << NBITS_PTR) - 1); }

struct vertex_t { uint64_t key, ptr; };  // store/vertex.hpp:152-155 (128-bit slot)

// Thomas Wang 64-bit mix — utils/math.hpp:58-67.  ikey_t::hash() (vertex.hpp:88-96) rebuilds
// exactly the raw key bits (vid<<18 | pid<<1 | dir) before hashing.
static inline uint64_t hash_u64(uint64_t key) {
    key = (~key) + (key << 21);
    key = key ^ (key >> 24);
    key = (key + (key << 3)) + (key << 8);
    key = key ^ (key >> 14);
    key = (key + (key << 2)) + (key << 4);
    key = key ^ (key >> 28);
    key = key + (key << 31);
    return key;
}

// utils/math.hpp:105-131
struct triple_t;
static bool less_pso(const triple_t &a, const triple_t &b);   // type.hpp:88-99
static bool less_pos(const triple_t &a, const triple_t &b);   // type.hpp:101-112

static uint64_t hash_prime_u64(uint64_t upper) {
    static const uint64_t P[] = {1610612741ull, 805306457ull, 402653189ull, 201326611ull, 100663319ull,
                                 50331653ull, 25165843ull, 12582917ull, 6291469ull, 3145739ull, 1572869ull,
                                 786433ull, 393241ull, 196613ull, 98317ull};
    if (upper >= (1ull << 31)) return upper;  // "too large" warning path
    for (uint64_t p : P)
        if (upper >= p) return p;
    return upper;  // "too small" warning path
}

struct triple_t { sid_t s, p, o; };
static bool less_pso(const triple_t &a, const triple_t &b) {
    if (a.p != b.p) return a.p < b.p;
    if (a.s != b.s) return a.s < b.s;
    return a.o < b.o;
}
static bool less_pos(const triple_t &a, const triple_t &b) {
    if (a.p != b.p) return a.p < b.p;
    if (a.o != b.o) return a.o < b.o;
    return a.s < b.s;
}

// ---- segment metadata: store/meta.hpp:53-204 ---------------------------------------------------
struct ext_extent_t { uint64_t num_ext_buckets, off, start; };
struct seg_meta_t {
    uint64_t num_keys = 0, num_buckets = 0, bucket_start = 0, num_edges = 0, edge_start = 0;
    std::vector<ext_extent_t> ext;
    uint64_t get_ext_bucket() {  // meta.hpp:107-115
        for (auto &e : ext)
            if (e.off < e.num_ext_buckets) return e.start + e.off++;
        return 0;
    }
};
struct segid_t {
    int index; int dir; sid_t pid;
    bool operator<(const segid_t &o) const {  // meta.hpp:172-182
        if (pid != o.pid) return pid < o.pid;
        if (index != o.index) return index < o.index;
        return dir < o.dir;
    }
};
static inline segid_t segid_of_key(uint64_t key) {  // meta.hpp:143-153
    segid_t s;
    s.dir = (int)key_dir(key);
    if (key_vid(key) == 0) { s.index = 1; s.pid = PREDICATE_ID; }
    else { s.index = 0; s.pid = (sid_t)key_pid(key); }
    return s;
}

// =============================================================================================
// Graph store: loader (core/loader/base_loader.hpp) + StaticGStore (store/static_gstore.hpp)
//              + GStore (store/gstore.hpp)
// =============================================================================================
struct Store {
    int sid = 0, num_servers = 1, num_engines = 1;
    bool gpu_ext_mode = true;   // -DUSE_GPU build: one 15% extent per segment (meta.hpp:38-40)
    int num_normal_preds = 0;   // (#lines of str_index) - 1, base_loader.hpp:409-424

    uint64_t num_slots = 0, num_buckets = 0, num_buckets_ext = 0, num_entries = 0;
    uint64_t last_ext = 0, last_entry = 0, main_hdr_off = 0;
    std::vector<vertex_t> vert_own;
    std::vector<sid_t> edge_own;
    vertex_t *vertices = nullptr;   // may point at foreign arrays (wko_store_wrap)
    sid_t *edges = nullptr;
    std::map<segid_t, seg_meta_t> seg_map;
    bool build_failed = false;
    std::string fail_msg;

    // build-time state
    std::vector<sid_t> all_local_preds;
    std::map<sid_t, std::vector<sid_t>> pidx_in_map, pidx_out_map, tidx_map;
    uint64_t num_segments = 0;
    // alloc_buckets_to_seg keeps function-local statics (gstore.hpp:437-438); one store => members
    bool nfb_init = false;
    uint64_t num_free_buckets = 0;

    void fail(const std::string &m) { if (!build_failed) { build_failed = true; fail_msg = m; } }

    // ---- sizing: GStore ctor, gstore.hpp:1013-1025; HD_RATIO/MHD_RATIO gstore.hpp:979-992 -----
    void size_regions(uint64_t kvstore_bytes) {
        const uint64_t HD_RATIO = (128 * 100 / (128 + 3 * 32));  // = 57 for 32-bit sid_t
        const uint64_t MHD_RATIO = 80;
        uint64_t header_region = kvstore_bytes * HD_RATIO / 100;
        uint64_t entry_region = kvstore_bytes - header_region;
        num_slots = header_region / sizeof(vertex_t);
        num_buckets = hash_prime_u64((num_slots / ASSOCIATIVITY) * MHD_RATIO / 100);
        num_buckets_ext = (num_slots / ASSOCIATIVITY) - num_buckets;
        num_entries = entry_region / sizeof(sid_t);
        vert_own.assign(num_slots, vertex_t{0, 0});   // StaticGStore::refresh, static_gstore.hpp:456-463
        edge_own.assign(num_entries, 0);
        vertices = vert_own.data();
        edges = edge_own.data();
    }

    uint64_t alloc_edges(uint64_t n) {  // static_gstore.hpp:36-47
        uint64_t orig = last_entry;
        last_entry += n;
        if (last_entry >= num_entries) fail("out of entry region");
        return orig;
    }
    uint64_t alloc_edges_to_seg(uint64_t n) { return n > 0 ? alloc_edges(n) : 0; }  // :49-51

    uint64_t alloc_ext_buckets(uint64_t n) {  // gstore.hpp:414-426
        uint64_t orig = last_ext;
        last_ext += n;
        if (last_ext >= num_buckets_ext) fail("out of indirect-header region");
        return num_buckets + orig;
    }
    uint64_t ext_extent_len(uint64_t nb) const {  // meta.hpp:38-43
        return gpu_ext_mode ? (nb * 15 / 100 + 1) : 256;
    }

    void alloc_buckets_to_seg(seg_meta_t &seg, uint64_t total_num_keys) {  // gstore.hpp:428-472
        uint64_t nbuckets;
        if (seg.num_keys == 0) {
            nbuckets = 0;
        } else {  // global_auto_bkt_alloc == true (gstore.hpp:153)
            if (!nfb_init) { num_free_buckets = num_buckets - num_segments; nfb_init = true; }
            double ratio = static_cast<double>(seg.num_keys) / total_num_keys;
            nbuckets = ratio * num_free_buckets;
        }
        const uint64_t min_buckets_per_seg = 1;  // gstore.hpp:187
        seg.num_buckets = std::max(nbuckets, min_buckets_per_seg);
        seg.bucket_start = main_hdr_off;
        main_hdr_off += seg.num_buckets;
        if (main_hdr_off > num_buckets) fail("main header overflow");
        if (seg.num_buckets > 0) {
            uint64_t n = ext_extent_len(seg.num_buckets);
            uint64_t start_off = alloc_ext_buckets(n);
            seg.ext.push_back(ext_extent_t{n, 0, start_off});
        }
    }

    uint64_t bucket_local(uint64_t key) {  // gstore.hpp:242-248
        seg_meta_t &seg = seg_map[segid_of_key(key)];
        O_ASSERT(seg.num_buckets > 0);
        return seg.bucket_start + hash_u64(key) % seg.num_buckets;
    }

    uint64_t insert_key(uint64_t key) {  // gstore.hpp:789-856
        if (build_failed) return 0;
        uint64_t bucket_id = bucket_local(key);
        uint64_t slot_id = bucket_id * ASSOCIATIVITY;
        while (slot_id < num_slots) {
            for (int i = 0; i < ASSOCIATIVITY - 1; i++, slot_id++) {
                if (vertices[slot_id].key == key) { fail("duplicate key"); return slot_id; }
                if (vertices[slot_id].key == 0) {   // ikey_t::is_empty, vertex.hpp:76
                    vertices[slot_id].key = key;
                    return slot_id;
                }
            }
            if (vertices[slot_id].key != 0) {   // chain pointer lives in key.vid of the last slot
                slot_id = key_vid(vertices[slot_id].key) * ASSOCIATIVITY;
                continue;
            }
            seg_meta_t &seg = seg_map[segid_of_key(key)];
            uint64_t ext_bucket_id = seg.get_ext_bucket();
            if (ext_bucket_id == 0) {
                if (gpu_ext_mode) { fail("segment exceeded its single ext extent (EXT_BUCKET_LIST_CAPACITY 1)"); return 0; }
                uint64_t n = ext_extent_len(seg.num_buckets);
                uint64_t start_off = alloc_ext_buckets(n);
                if (build_failed) return 0;
                seg.ext.push_back(ext_extent_t{n, 0, start_off});
                ext_bucket_id = seg.get_ext_bucket();
            }
            vertices[slot_id].key = make_key(ext_bucket_id, 0, 0);   // key.vid = ext bucket id
            slot_id = ext_bucket_id * ASSOCIATIVITY;
            vertices[slot_id].key = key;
            return slot_id;
        }
        fail("slot id out of range");
        return 0;
    }

    void collect_idx_info(uint64_t slot_id) {  // gstore.hpp:858-888
        uint64_t k = vertices[slot_id].key;
        sid_t vid = (sid_t)key_vid(k), pid = (sid_t)key_pid(k);
        uint64_t sz = ptr_size(vertices[slot_id].ptr), off = ptr_off(vertices[slot_id].ptr);
        if (key_dir(k) == DIR_IN) {
            if (pid == PREDICATE_ID) {}
            else if (pid == TYPE_ID) { O_ASSERT(false); }
            else pidx_out_map[pid].push_back(vid);
        } else {
            if (pid == PREDICATE_ID) {}
            else if (pid == TYPE_ID) { for (uint64_t e = 0; e < sz; e++) tidx_map[edges[off + e]].push_back(vid); }
            else pidx_in_map[pid].push_back(vid);
        }
    }

    // ---- loader: base_loader.hpp:308-378 (aggregate_data), :81-95 (dedup) --------------------
    static void dedup(std::vector<triple_t> &t) {
        if (t.size() <= 1) return;
        uint64_t n = 1;
        for (uint64_t i = 1; i < t.size(); i++) {
            if (t[i].s == t[i - 1].s && t[i].p == t[i - 1].p && t[i].o == t[i - 1].o) continue;
            t[n++] = t[i];
        }
        t.resize(n);
    }
    void load(const sid_t *tr, uint64_t n, std::vector<std::vector<triple_t>> &pso,
              std::vector<std::vector<triple_t>> &pos) {
        pso.assign(num_engines, {});
        pos.assign(num_engines, {});
        for (uint64_t i = 0; i < n; i++) {
            sid_t s = tr[3 * i], p = tr[3 * i + 1], o = tr[3 * i + 2];
            if ((int)(s % num_servers) == sid) pso[s % num_engines].push_back(triple_t{s, p, o});
            if ((int)(o % num_servers) == sid) pos[o % num_engines].push_back(triple_t{s, p, o});
        }
        for (int t = 0; t < num_engines; t++) {
            std::sort(pso[t].begin(), pso[t].end(), less_pso);
            std::sort(pos[t].begin(), pos[t].end(), less_pos);
            dedup(pos[t]);
            dedup(pso[t]);
        }
    }

    // ---- StaticGStore::init, static_gstore.hpp:383-454 ----------------------------------------
    void build(const sid_t *tr, uint64_t n) {
        std::vector<std::vector<triple_t>> pso, pos;
        load(tr, n, pso, pos);
        const int npreds = num_normal_preds;
        num_segments = (uint64_t)npreds * 2 + 2;   // PREDICATE_NSEGS*preds + INDEX_NSEGS, :386

        // init_triples_map (gstore.hpp:475-527): per (pid,dir) concatenation over engine tids
        std::map<std::pair<sid_t, int>, std::vector<triple_t>> triples_map;
        for (int t = 0; t < num_engines; t++) {
            for (auto &x : pso[t]) triples_map[{x.p, DIR_OUT}].push_back(x);
            for (auto &x : pos[t]) triples_map[{x.p, DIR_IN}].push_back(x);
        }

        // init_seg_metas (gstore.hpp:530-786)
        struct cnt_t { uint64_t in = 0, out = 0; };
        std::map<sid_t, cnt_t> normal_cnt, index_cnt;
        for (int i = 0; i <= npreds; ++i) {
            index_cnt[i]; normal_cnt[i];
            for (int d = 0; d <= 1; d++) seg_map[segid_t{0, d, (sid_t)i}];
        }
        seg_map[segid_t{1, DIR_IN, PREDICATE_ID}];
        seg_map[segid_t{1, DIR_OUT, PREDICATE_ID}];
        for (int t = 0; t < num_engines; t++) {
            auto &a = pso[t];
            uint64_t s = 0;
            while (s < a.size()) {
                uint64_t e = s + 1;
                while (e < a.size() && a[s].s == a[e].s && a[s].p == a[e].p) {
                    if (a[e].p == TYPE_ID && is_tpid(a[e].o)) index_cnt[a[e].o].in++;
                    e++;
                }
                normal_cnt[a[s].p].out += (e - s);
                index_cnt[a[s].p].in++;
                if (a[s].p == TYPE_ID && is_tpid(a[s].o)) index_cnt[a[s].o].in++;
                s = e;
            }
            auto &b = pos[t];
            uint64_t type_triples = 0;
            while (type_triples < b.size() && is_tpid(b[type_triples].o)) type_triples++;
            s = type_triples;
            while (s < b.size()) {
                uint64_t e = s + 1;
                while (e < b.size() && b[s].o == b[e].o && b[s].p == b[e].p) e++;
                normal_cnt[b[s].p].in += (e - s);
                index_cnt[b[s].p].out++;
                s = e;
            }
        }
        uint64_t total_num_keys = 0, num_typeid = 0;
        for (int i = 1; i <= npreds; ++i) {
            if (normal_cnt[i].in + normal_cnt[i].out > 0) {
                all_local_preds.push_back(i);
                total_num_keys += index_cnt[i].in + index_cnt[i].out;
            } else if (index_cnt[i].in > 0) {
                num_typeid++;
            }
        }
        total_num_keys += all_local_preds.size() * 2 + num_typeid;

        seg_meta_t &idx_out_seg = seg_map[segid_t{1, DIR_OUT, PREDICATE_ID}];
        seg_meta_t &idx_in_seg = seg_map[segid_t{1, DIR_IN, PREDICATE_ID}];
        for (sid_t pid = 1; pid <= (sid_t)npreds; ++pid) {
            seg_meta_t &out_seg = seg_map[segid_t{0, DIR_OUT, pid}];
            seg_meta_t &in_seg = seg_map[segid_t{0, DIR_IN, pid}];
            out_seg.num_edges = normal_cnt[pid].out;
            in_seg.num_edges = normal_cnt[pid].in;
            idx_out_seg.num_edges += index_cnt[pid].out;
            idx_in_seg.num_edges += index_cnt[pid].in;
            uint64_t normal_nkeys[2] = {index_cnt[pid].out, index_cnt[pid].in};
            out_seg.num_keys = (out_seg.num_edges == 0) ? 0 : normal_nkeys[DIR_OUT];
            in_seg.num_keys = (in_seg.num_edges == 0) ? 0 : normal_nkeys[DIR_IN];
            out_seg.edge_start = alloc_edges_to_seg(out_seg.num_edges);
            in_seg.edge_start = alloc_edges_to_seg(in_seg.num_edges);
            alloc_buckets_to_seg(out_seg, total_num_keys);
            alloc_buckets_to_seg(in_seg, total_num_keys);
        }
        idx_out_seg.edge_start = alloc_edges_to_seg(idx_out_seg.num_edges);
        idx_out_seg.num_keys = all_local_preds.size();
        alloc_buckets_to_seg(idx_out_seg, total_num_keys);
        idx_in_seg.edge_start = alloc_edges_to_seg(idx_in_seg.num_edges);
        idx_in_seg.num_keys = all_local_preds.size() + num_typeid;
        alloc_buckets_to_seg(idx_in_seg, total_num_keys);
        if (build_failed) return;

        // insert_triples per predicate, OUT then IN (static_gstore.hpp:64-161, 410-416)
        for (sid_t pid : all_local_preds) {
            for (int dir : {DIR_OUT, DIR_IN}) {
                seg_meta_t &seg = seg_map[segid_t{0, dir, pid}];
                if (seg.num_edges == 0) continue;
                auto it = triples_map.find({pid, dir});
                O_ASSERT(it != triples_map.end());
                const std::vector<triple_t> &v = it->second;
                uint64_t off = seg.edge_start, s = 0;
                if (dir == DIR_OUT) {
                    while (s < v.size()) {
                        uint64_t e = s + 1;
                        while (e < v.size() && v[s].s == v[e].s && v[s].p == v[e].p) e++;
                        uint64_t slot = insert_key(make_key(v[s].s, v[s].p, DIR_OUT));
                        if (build_failed) return;
                        vertices[slot].ptr = make_ptr(e - s, off);
                        for (uint64_t i = s; i < e; i++) edges[off++] = v[i].o;
                        collect_idx_info(slot);
                        s = e;
                    }
                } else {
                    uint64_t type_triples = 0;
                    while (type_triples < v.size() && is_tpid(v[type_triples].o)) type_triples++;
                    s = type_triples;
                    while (s < v.size()) {
                        uint64_t e = s + 1;
                        while (e < v.size() && v[s].o == v[e].o && v[s].p == v[e].p) e++;
                        uint64_t slot = insert_key(make_key(v[s].o, v[s].p, DIR_IN));
                        if (build_failed) return;
                        vertices[slot].ptr = make_ptr(e - s, off);
                        for (uint64_t i = s; i < e; i++) edges[off++] = v[i].s;
                        collect_idx_info(slot);
                        s = e;
                    }
                }
                O_ASSERT(off <= seg.edge_start + seg.num_edges);
            }
        }
        // insert_idx IN then OUT (static_gstore.hpp:217-265, 431-435)
        for (int d : {DIR_IN, DIR_OUT}) {
            auto &pidx = (d == DIR_IN) ? pidx_in_map : pidx_out_map;
            seg_meta_t &seg = seg_map[segid_t{1, d, PREDICATE_ID}];
            uint64_t off = seg.edge_start;
            for (sid_t pid : all_local_preds) {
                auto it = pidx.find(pid);
                if (it == pidx.end()) continue;
                uint64_t slot = insert_key(make_key(0, pid, d));
                if (build_failed) return;
                vertices[slot].ptr = make_ptr(it->second.size(), off);
                for (sid_t v : it->second) edges[off++] = v;
                O_ASSERT(off <= seg.edge_start + seg.num_edges);
            }
            if (d == DIR_IN) {
                for (auto &e : tidx_map) {
                    uint64_t slot = insert_key(make_key(0, e.first, DIR_IN));
                    if (build_failed) return;
                    vertices[slot].ptr = make_ptr(e.second.size(), off);
                    for (sid_t v : e.second) edges[off++] = v;
                    O_ASSERT(off <= seg.edge_start + seg.num_edges);
                }
            }
        }
        all_local_preds.shrink_to_fit();
        pidx_in_map.clear(); pidx_out_map.clear(); tidx_map.clear();
    }

    // ---- probe: gstore.hpp:341-361 (get_vertex_local), :393-410 (get_edges_local) ---------------
    const sid_t *get_edges_local(sid_t vid, sid_t pid, int d, uint64_t &sz) {
        uint64_t key = make_key(vid, pid, d);
        auto it = seg_map.find(segid_of_key(key));
        O_ASSERT(it != seg_map.end() && it->second.num_buckets > 0);   // ASSERT(seg.num_buckets > 0), :245
        uint64_t bucket_id = it->second.bucket_start + hash_u64(key) % it->second.num_buckets;
        while (true) {
            for (int i = 0; i < ASSOCIATIVITY; i++) {
                uint64_t slot_id = bucket_id * ASSOCIATIVITY + i;
                if (i < ASSOCIATIVITY - 1) {
                    if (vertices[slot_id].key == key) {
                        sz = ptr_size(vertices[slot_id].ptr);
                        return &edges[ptr_off(vertices[slot_id].ptr)];
                    }
                } else {
                    if (vertices[slot_id].key == 0) { sz = 0; return nullptr; }
                    bucket_id = key_vid(vertices[slot_id].key);
                    break;
                }
            }
        }
    }
};

// =============================================================================================
// Query data model: core/query.hpp:71-116 (Pattern), :251-557 (Result), :560-682 (SPARQLQuery)
// =============================================================================================
enum { KNOWN_VAR = 0, UNKNOWN_VAR, CONST_VAR };        // query.hpp:51
static const int NO_RESULT = (1 << 16) - 1;            // query.hpp:61
static inline int const_pair(int a, int b) { return (a << 4) | b; }  // query.hpp:49

struct Pattern { ssid_t subject, predicate; int direction; ssid_t object; };

struct Result {
    int col_num = 0, row_num = 0, status_code = SUCCESS;
    bool blind = false;
    int nvars = 0;
    std::vector<ssid_t> required_vars;
    std::vector<int> v2c_map;
    std::vector<sid_t> result_table;

    int var2col(ssid_t vid) {  // query.hpp:359-375
        O_ASSERT_CODE(vid < 0, VERTEX_INVALID);
        O_ASSERT(nvars > 0);
        if (v2c_map.size() == 0) v2c_map.resize(nvars, NO_RESULT);
        int idx = -(vid + 1);
        O_ASSERT_CODE(idx < nvars && idx >= 0, VERTEX_INVALID);
        return v2c_map[idx] & 0xFFFF;   // ext2col
    }
    int var_stat(ssid_t vid) {  // query.hpp:343-350
        if (vid >= 0) return CONST_VAR;
        else if (var2col(vid) == NO_RESULT) return UNKNOWN_VAR;
        else return KNOWN_VAR;
    }
    void add_var2col(ssid_t vid, int col) {  // query.hpp:378-395 (type SID_t=0)
        O_ASSERT(vid < 0 && col >= 0);
        if (v2c_map.size() == 0) v2c_map.resize(nvars, NO_RESULT);
        int idx = -(vid + 1);
        O_ASSERT(idx < nvars && idx >= 0);
        O_ASSERT(v2c_map[idx] == NO_RESULT);
        v2c_map[idx] = col;
    }
    int get_row_num() const { return col_num == 0 ? 0 : (int)(result_table.size() / col_num); }  // :425-428
    void update_nrows() { row_num = get_row_num(); }                                               // :430-433
    sid_t get_row_col(int r, int c) const { return result_table[(size_t)col_num * r + c]; }        // :435-438
    void append_row_to(int r, std::vector<sid_t> &u) const {                                       // :440-443
        for (int c = 0; c < col_num; c++) u.push_back(get_row_col(r, c));
    }
    void append_result(Result &r) {  // query.hpp:536-557
        v2c_map = r.v2c_map;
        col_num = r.col_num;
        row_num += r.row_num;
        if (r.blind) return;
        result_table.insert(result_table.end(), r.result_table.begin(), r.result_table.end());
    }
};

struct Query {
    std::vector<Pattern> patterns;
    int pattern_step = 0;
    int mt_factor = 1, mt_tid = 0;
    ssid_t local_var = 0;
    Result result;
    bool from_proxy = true;
    Pattern &get_pattern() { O_ASSERT(pattern_step < (int)patterns.size()); return patterns[pattern_step]; }
    bool done() const { return pattern_step >= (int)patterns.size(); }   // query.hpp:627-628
    bool start_from_index() {  // query.hpp:660-682
        if (patterns.empty()) return false;
        if (is_tpid(patterns[0].subject)) {
            O_ASSERT_CODE(patterns[0].predicate == PREDICATE_ID || patterns[0].predicate == TYPE_ID, OBJ_ERROR);
            return true;
        }
        return false;
    }
};

// =============================================================================================
// Engine: core/engine/sparql.hpp
// =============================================================================================
struct Cluster {   // one simulated server per store; fork-join done in-process
    std::vector<Store *> stores;
    int num_servers() const { return (int)stores.size(); }
    // DGraph::get_triples / get_index -> GStore::get_edges (dgraph.hpp:106-112, gstore.hpp:1043-1054).
    // The oracle never performs the RDMA remote read: like the reference with use_rdma=false it
    // always fork-joins so that every probed normal vertex is local (sparql.hpp:802-807).
    const sid_t *get_edges(int sid, sid_t vid, sid_t pid, int d, uint64_t &sz) {
        if (vid != 0) O_ASSERT((int)(vid % num_servers()) == sid);
        return stores[sid]->get_edges_local(vid, pid, d, sz);
    }
};

struct Engine {
    Cluster *cl;
    int sid;
    const sid_t *get_triples(sid_t vid, sid_t pid, int d, uint64_t &sz) { return cl->get_edges(sid, vid, pid, d, sz); }
    const sid_t *get_index(sid_t pid, int d, uint64_t &sz) { return cl->get_edges(sid, 0, pid, d, sz); }

    void index_to_known(Query &req) {  // sparql.hpp:80-141 (BASIC group only)
        Pattern &pt = req.get_pattern();
        ssid_t tpid = pt.subject, id01 = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        int col = res.var2col(end);
        O_ASSERT_CODE(col != NO_RESULT, VERTEX_INVALID);
        O_ASSERT_CODE(id01 == PREDICATE_ID || id01 == TYPE_ID, OBJ_ERROR);
        std::vector<sid_t> updated;
        uint64_t sz = 0;
        const sid_t *edges = get_index(tpid, d, sz);
        int start = req.mt_tid % req.mt_factor;
        int length = sz / req.mt_factor;
        std::vector<sid_t> uniq;
        for (uint64_t k = (uint64_t)start * length; k < (uint64_t)(start + 1) * length; k++) uniq.push_back(edges[k]);
        if (start == req.mt_factor - 1)
            for (uint64_t k = (uint64_t)(start + 1) * length; k < sz; k++) uniq.push_back(edges[k]);
        std::sort(uniq.begin(), uniq.end());
        int nrows = res.get_row_num();
        for (int i = 0; i < nrows; i++)
            if (std::binary_search(uniq.begin(), uniq.end(), res.get_row_col(i, col))) res.append_row_to(i, updated);
        res.result_table.swap(updated);
        res.update_nrows();
        req.pattern_step++;
    }

    void const_to_known(Query &req) {  // sparql.hpp:144-186 (BASIC group only)
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, pid = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        int col = res.var2col(end);
        O_ASSERT_CODE(col != NO_RESULT, VERTEX_INVALID);
        uint64_t sz = 0;
        const sid_t *vids = get_triples(start, pid, d, sz);
        std::vector<sid_t> uniq(vids, vids + sz);
        std::sort(uniq.begin(), uniq.end());
        std::vector<sid_t> updated;
        int nrows = res.get_row_num();
        for (int i = 0; i < nrows; i++)
            if (std::binary_search(uniq.begin(), uniq.end(), res.get_row_col(i, col))) res.append_row_to(i, updated);
        res.result_table.swap(updated);
        res.update_nrows();
        req.pattern_step++;
    }

    void index_to_unknown(Query &req) {  // sparql.hpp:194-231
        Pattern &pt = req.get_pattern();
        ssid_t tpid = pt.subject, id01 = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        O_ASSERT_CODE(id01 == PREDICATE_ID || id01 == TYPE_ID, OBJ_ERROR);
        O_ASSERT_CODE(res.col_num == 0, FIRST_PATTERN_ERROR);
        std::vector<sid_t> updated;
        uint64_t sz = 0;
        const sid_t *edges = get_index(tpid, d, sz);
        int start = req.mt_tid % req.mt_factor;
        int length = sz / req.mt_factor;
        for (uint64_t k = (uint64_t)start * length; k < (uint64_t)(start + 1) * length; k++) updated.push_back(edges[k]);
        if (start == req.mt_factor - 1)
            for (uint64_t k = (uint64_t)(start + 1) * length; k < sz; k++) updated.push_back(edges[k]);
        res.result_table.swap(updated);
        res.col_num = 1;
        res.add_var2col(end, 0);
        res.update_nrows();
        req.pattern_step++;
        req.local_var = end;
    }

    void const_to_unknown(Query &req) {  // sparql.hpp:238-285 (SID_t branch)
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, pid = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        O_ASSERT_CODE(res.col_num == 0, FIRST_PATTERN_ERROR);
        uint64_t sz = 0;
        const sid_t *vids = get_triples(start, pid, d, sz);
        std::vector<sid_t> updated;
        for (uint64_t k = 0; k < sz; k++) updated.push_back(vids[k]);
        res.result_table.swap(updated);
        res.add_var2col(end, res.col_num);
        res.col_num = res.col_num + 1;
        res.update_nrows();
        req.pattern_step++;
    }

    void known_to_unknown(Query &req) {  // sparql.hpp:295-407 (SID_t, non-OPTIONAL branch :316-380)
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, pid = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        std::vector<sid_t> updated;
        updated.reserve(res.result_table.size());
        sid_t cached = BLANK_ID;
        const sid_t *vids = nullptr;
        uint64_t sz = 0;
        int nrows = res.get_row_num();
        int scol = res.var2col(start);
        for (int i = 0; i < nrows; i++) {
            sid_t cur = res.get_row_col(i, scol);
            if (cur != cached) {
                cached = cur;
                if (pid == TYPE_ID && d == DIR_IN) vids = get_index(cur, d, sz);
                else vids = get_triples(cur, pid, d, sz);
            }
            for (uint64_t k = 0; k < sz; k++) {
                res.append_row_to(i, updated);
                updated.push_back(vids[k]);
            }
        }
        res.result_table.swap(updated);
        res.add_var2col(end, res.col_num);
        res.col_num = res.col_num + 1;
        res.update_nrows();
        req.pattern_step++;
    }

    void known_to_known(Query &req) {  // sparql.hpp:416-476
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, pid = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        std::vector<sid_t> updated;
        sid_t cached = BLANK_ID;
        const sid_t *vids = nullptr;
        uint64_t sz = 0;
        int nrows = res.get_row_num();
        int scol = res.var2col(start), ecol = res.var2col(end);
        for (int i = 0; i < nrows; i++) {
            sid_t cur = res.get_row_col(i, scol);
            if (cur != cached) { cached = cur; vids = get_triples(cur, pid, d, sz); }
            sid_t known = res.get_row_col(i, ecol);
            for (uint64_t k = 0; k < sz; k++)
                if (vids[k] == known) { res.append_row_to(i, updated); break; }
        }
        res.result_table.swap(updated);
        res.update_nrows();
        req.pattern_step++;
    }

    void known_to_const(Query &req) {  // sparql.hpp:484-549
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, pid = pt.predicate, end = pt.object; int d = pt.direction;
        Result &res = req.result;
        std::vector<sid_t> updated;
        sid_t cached = BLANK_ID;
        const sid_t *vids = nullptr;
        uint64_t sz = 0;
        bool exist = false;
        int nrows = res.get_row_num();
        int scol = res.var2col(start);
        for (int i = 0; i < nrows; i++) {
            sid_t cur = res.get_row_col(i, scol);
            if (cur != cached) {
                exist = false;
                cached = cur;
                vids = get_triples(cur, pid, d, sz);
                for (uint64_t k = 0; k < sz; k++)
                    if (vids[k] == (sid_t)end) { exist = true; res.append_row_to(i, updated); break; }
            } else if (exist) {
                res.append_row_to(i, updated);
            }
        }
        res.result_table.swap(updated);
        res.update_nrows();
        req.pattern_step++;
    }

    bool execute_one_pattern(Query &req) {  // sparql.hpp:938-1061 (non-VERSATILE build)
        O_ASSERT(!req.done());
        Pattern &pt = req.get_pattern();
        ssid_t start = pt.subject, predicate = pt.predicate, end = pt.object;
        if (req.pattern_step == 0 && req.start_from_index()) {
            if (req.result.var2col(end) != NO_RESULT) index_to_known(req);
            else index_to_unknown(req);
            return true;
        }
        if (req.result.var_stat(predicate) != CONST_VAR) O_ASSERT_CODE(false, UNKNOWN_PATTERN);
        switch (const_pair(req.result.var_stat(start), req.result.var_stat(end))) {
        case (CONST_VAR << 4) | CONST_VAR: O_ASSERT_CODE(false, UNKNOWN_PATTERN);
        case (CONST_VAR << 4) | KNOWN_VAR: const_to_known(req); break;
        case (CONST_VAR << 4) | UNKNOWN_VAR: const_to_unknown(req); break;
        case (KNOWN_VAR << 4) | CONST_VAR: known_to_const(req); break;
        case (KNOWN_VAR << 4) | KNOWN_VAR: known_to_known(req); break;
        case (KNOWN_VAR << 4) | UNKNOWN_VAR: known_to_unknown(req); break;
        case (UNKNOWN_VAR << 4) | CONST_VAR:
        case (UNKNOWN_VAR << 4) | KNOWN_VAR:
        case (UNKNOWN_VAR << 4) | UNKNOWN_VAR: O_ASSERT_CODE(false, UNKNOWN_SUB);
        default: O_ASSERT_CODE(false, UNKNOWN_PATTERN);
        }
        return true;
    }
};

// generate_sub_query, sparql.hpp:746-799
static std::vector<Query> generate_sub_query(Query &req, int num_servers, bool need_split) {
    ssid_t start = req.get_pattern().subject;
    std::vector<Query> subs(num_servers);
    for (int i = 0; i < num_servers; i++) {
        subs[i].patterns = req.patterns;
        subs[i].pattern_step = req.pattern_step;
        subs[i].local_var = start;
        subs[i].from_proxy = false;
        subs[i].result.col_num = req.result.col_num;
        subs[i].result.blind = req.result.blind;
        subs[i].result.v2c_map = req.result.v2c_map;
        subs[i].result.nvars = req.result.nvars;
    }
    int nrows = req.result.get_row_num();
    if (!need_split) {
        for (int i = 0; i < num_servers; i++) { subs[i].result.result_table = req.result.result_table; subs[i].result.update_nrows(); }
    } else {
        int scol = req.result.var2col(start);
        for (int i = 0; i < nrows; i++) {
            int dst = req.result.get_row_col(i, scol) % num_servers;   // math::hash_mod, utils/math.hpp:51-55
            req.result.append_row_to(i, subs[dst].result.result_table);
        }
        for (int i = 0; i < num_servers; i++) subs[i].result.update_nrows();
    }
    return subs;
}

// execute_patterns on server `sid` + fork-join; the replies of a fork are merged with
// Result::append_result in server order (rmap.hpp:44-110; arrival order is unspecified there).
// Runs with Global::use_rdma == false semantics: need_fork_join() is true whenever
// num_servers > 1 (sparql.hpp:802-807).
static void run_patterns(Cluster &cl, int sid, Query &r, Result &out) {
    Engine eng{&cl, sid};
    const int S = cl.num_servers();
    while (true) {
        eng.execute_one_pattern(r);
        if (r.done()) { r.result.update_nrows(); out.append_result(r.result); return; }
        // dispatch(r, false): type-index expansion must visit every server (sparql.hpp:1091-1110)
        Pattern &pt = r.get_pattern();
        bool dup_all = (S != 1 && pt.predicate == TYPE_ID && pt.direction == DIR_IN);
        if (dup_all || S > 1) {
            std::vector<Query> subs = generate_sub_query(r, S, !dup_all);
            for (int i = 0; i < S; i++) run_patterns(cl, i, subs[i], out);
            return;
        }
    }
}

// final_process, sparql.hpp:1424-1551: DISTINCT (:1428-1472, rows ordered by ReduceCmp :1406-1421 = all columns compared
// as signed ints, then the p/q walk that keeps a row iff it differs from the last kept row on the required columns),
// OFFSET (:1487-1492), LIMIT (:1494-1499), projection (:1507-1550).  ORDER BY needs the string server: not in scope.
struct Modifiers { bool distinct = false; int64_t offset = 0, limit = -1; };
static void final_process(Result &res, const Modifiers &md = Modifiers()) {
    if (res.blind || res.result_table.size() == 0) return;
    if (md.distinct) {
        const int C = res.col_num, size = res.get_row_num();
        std::vector<std::vector<int>> table(size, std::vector<int>(C));
        for (int i = 0; i < size; i++)
            for (int j = 0; j < C; j++) table[i][j] = (int)res.get_row_col(i, j);
        std::sort(table.begin(), table.end(), [C](const std::vector<int> &a, const std::vector<int> &b) {
            for (int i = 0; i < C; i++) {
                if (a[i] == b[i]) continue;
                return a[i] < b[i];
            }
            return false;
        });
        std::vector<int> cols;
        for (size_t i = 0; i < res.required_vars.size(); i++) cols.push_back(res.var2col(res.required_vars[i]));
        auto equal = [&cols](const std::vector<int> &a, const std::vector<int> &b) {
            for (int c : cols)
                if (a[c] != b[c]) return false;
            return true;
        };
        int p = 0, q = 1;
        bool out = false;
        while (q < size && !out) {
            while (equal(table[p], table[q])) {
                q++;
                if (q >= size) { out = true; break; }
            }
            if (out) break;
            p++;
            std::swap(table[p], table[q]);
            q++;
        }
        const int new_size = p + 1;
        res.result_table.resize((size_t)new_size * C);
        for (int i = 0; i < new_size; i++)
            for (int j = 0; j < C; j++) res.result_table[(size_t)C * i + j] = (sid_t)table[i][j];
    }
    if (md.offset > 0) {
        const size_t drop = std::min<size_t>((size_t)md.offset * res.col_num, res.result_table.size());
        res.result_table.erase(res.result_table.begin(), res.result_table.begin() + drop);
    }
    if (md.limit >= 0) {
        const size_t keep = std::min<size_t>((size_t)md.limit * res.col_num, res.result_table.size());
        res.result_table.erase(res.result_table.begin() + keep, res.result_table.end());
    }
    O_ASSERT_CODE(res.required_vars.size() != 0, NO_REQUIRED_VAR);
    int new_row_num = res.get_row_num();
    int new_col_num = (int)res.required_vars.size();
    std::vector<sid_t> nt((size_t)new_row_num * new_col_num);
    for (int i = 0; i < new_row_num; i++)
        for (int j = 0; j < new_col_num; j++)
            nt[(size_t)i * new_col_num + j] = res.get_row_col(i, res.var2col(res.required_vars[j]));
    res.result_table.swap(nt);
    res.col_num = new_col_num;
    res.update_nrows();
}

// execute_sparql_query pattern phase, sparql.hpp:1564-1673, with dispatch() (sparql.hpp:1064-1089):
// an index-start query from a proxy is replicated to num_servers x mt_factor engines, each
// taking slice mt_tid of its server's local index list; replies are concatenated.
struct QueryOut { Result result; double usec = 0; };

static void run_query(Cluster &cl, const std::vector<Pattern> &patterns, int nvars,
                      const std::vector<ssid_t> &required_vars, int mt_factor, bool blind,
                      bool threaded, QueryOut &qo, const Modifiers &md = Modifiers()) {
    const int S = cl.num_servers();
    Query proto;
    proto.patterns = patterns;
    proto.result.nvars = nvars;
    proto.result.required_vars = required_vars;
    proto.result.v2c_map.assign(nvars, NO_RESULT);
    proto.result.blind = blind;
    Result &fin = qo.result;
    fin.nvars = nvars;
    fin.required_vars = required_vars;
    fin.blind = blind;
    auto t0 = std::chrono::steady_clock::now();
    try {
        if (patterns.empty()) throw OracleError{SYNTAX_ERROR};
        if (proto.start_from_index() && S * mt_factor > 1) {
            proto.mt_factor = mt_factor;
            const int njobs = S * mt_factor;
            std::vector<Result> parts(njobs);
            std::vector<int> codes(njobs, SUCCESS);
            auto job = [&](int j) {
                Query q = proto;
                q.mt_tid = j % mt_factor;
                q.from_proxy = false;
                parts[j].nvars = nvars;
                parts[j].blind = false;
                try { run_patterns(cl, j / mt_factor, q, parts[j]); }
                catch (OracleError &e) { codes[j] = e.code; }
            };
            if (threaded) {
                std::vector<std::thread> th;
                for (int j = 0; j < njobs; j++) th.emplace_back(job, j);
                for (auto &t : th) t.join();
            } else {
                for (int j = 0; j < njobs; j++) job(j);
            }
            for (int j = 0; j < njobs; j++) {
                if (codes[j] != SUCCESS) throw OracleError{codes[j]};
                parts[j].blind = false;
                fin.append_result(parts[j]);
            }
        } else {
            // const-start: runs on the owner of the constant (proxy.hpp:201-219 picks a server;
            // get_edges would go remote otherwise).  Index-start with S*mt==1 runs on server 0.
            int sid0 = 0;
            if (!proto.start_from_index() && patterns[0].subject >= 0) sid0 = patterns[0].subject % S;
            Result acc;
            acc.nvars = nvars;
            run_patterns(cl, sid0, proto, acc);
            acc.blind = false;
            fin.append_result(acc);
        }
        fin.blind = blind;
        // blind replies carry only row_num (accumulated by append_result, query.hpp:536-545); the
        // table itself is dropped by shrink() (query.hpp:619-630) and final_process is skipped
        if (!blind) { fin.update_nrows(); final_process(fin, md); }
        else fin.result_table.clear();
    } catch (OracleError &e) {
        fin.status_code = e.code;   // sparql.hpp:1663-1667
        fin.result_table.clear();
        fin.row_num = 0;
    }
    qo.usec = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
}

// =============================================================================================
// Plan application: core/planner.hpp:1647-1754 (set_plan + set_direction)
// =============================================================================================
static bool set_plan(std::vector<Pattern> &patterns, const std::string &fmt) {
    std::vector<int> orders;
    std::vector<std::string> dirs;
    std::istringstream in(fmt);
    std::string line;
    while (std::getline(in, line)) {
        size_t a = line.find_first_not_of(" \t\r\n");
        if (a == std::string::npos) continue;
        size_t b = line.find_last_not_of(" \t\r\n");
        line = line.substr(a, b - a + 1);
        if (line[0] == '#') continue;
        if (line == "{") continue;
        if (line == "}") break;
        std::istringstream iss(line);
        int order = 0;
        std::string dir = ">";
        iss >> order >> dir;
        orders.push_back(order);
        dirs.push_back(dir);
    }
    if (orders.size() < patterns.size()) return false;   // "wrong format file content!"
    std::vector<Pattern> out;
    for (size_t i = 0; i < orders.size(); i++) {
        if (orders[i] < 1 || orders[i] > (int)patterns.size()) return false;
        Pattern p = patterns[orders[i] - 1];
        if (dirs[i] == "<") { p.direction = DIR_IN; std::swap(p.subject, p.object); }
        else if (dirs[i] == ">") { p.direction = DIR_OUT; }
        else if (dirs[i] == "<<") { p.direction = DIR_IN; p.object = p.subject; p.subject = p.predicate; p.predicate = PREDICATE_ID; }
        else if (dirs[i] == ">>") { p.direction = DIR_OUT; p.subject = p.predicate; p.predicate = PREDICATE_ID; }
        out.push_back(p);
    }
    patterns.swap(out);
    return true;
}

// =============================================================================================
// gsck invariants: store/gchecker.hpp:132-360 (check_idx_in/out, check_type, check_normal)
// =============================================================================================
static uint64_t store_check(Store &st) {
    uint64_t errors = 0;
    const uint64_t total_buckets = st.num_slots / ASSOCIATIVITY;
    auto contains_once = [&](sid_t vid, sid_t pid, int d, sid_t want) {
        uint64_t sz = 0;
        const sid_t *l = st.get_edges_local(vid, pid, d, sz);
        uint64_t c = 0;
        for (uint64_t i = 0; i < sz; i++) c += (l[i] == want);
        return c == 1;
    };
    for (uint64_t b = 0; b < total_buckets; b++) {
        for (int i = 0; i < ASSOCIATIVITY - 1; i++) {
            vertex_t &v = st.vertices[b * ASSOCIATIVITY + i];
            if (v.key == 0) continue;
            sid_t vid = (sid_t)key_vid(v.key), pid = (sid_t)key_pid(v.key);
            int d = (int)key_dir(v.key);
            uint64_t sz = ptr_size(v.ptr), off = ptr_off(v.ptr);
            // the key must be reachable by a probe and return this very slot's edges
            uint64_t psz = 0;
            const sid_t *pl = st.get_edges_local(vid, pid, d, psz);
            if (pl != &st.edges[off] || psz != sz) errors++;
            if (vid == 0) {
                // index vertex: every member must own the matching normal key
                for (uint64_t e = 0; e < sz; e++) {
                    sid_t m = st.edges[off + e];
                    uint64_t s2 = 0;
                    if (d == DIR_IN) {
                        // [0|p|IN] lists subjects of p; [0|t|IN] lists instances of type t
                        st.get_edges_local(m, pid, DIR_OUT, s2);
                        bool as_pred = s2 > 0;
                        bool as_type = contains_once(m, TYPE_ID, DIR_OUT, pid);
                        if (!as_pred && !as_type) errors++;
                    } else {
                        st.get_edges_local(m, pid, DIR_IN, s2);
                        if (s2 == 0) errors++;
                    }
                }
            } else {
                // sorted, duplicate-free edge run (base_loader.hpp:365-373)
                for (uint64_t e = 1; e < sz; e++)
                    if (st.edges[off + e - 1] >= st.edges[off + e]) errors++;
                if (pid == TYPE_ID) {
                    if (d != DIR_OUT) errors++;
                    for (uint64_t e = 0; e < sz; e++)
                        if (!contains_once(0, st.edges[off + e], DIR_IN, vid)) errors++;   // check_type
                } else {
                    if (!contains_once(0, pid, d == DIR_OUT ? DIR_IN : DIR_OUT, vid)) errors++;   // check_idx_in/out
                }
            }
        }
    }
    return errors;
}

}  // namespace wko

// =============================================================================================
// C API (ctypes)
// =============================================================================================
using namespace wko;

struct wko_segmeta {   // flat view of one segment, same fields as include/wukong_b200.h wk_segmeta
    int32_t index, dir;
    uint32_t pid, _pad;
    uint64_t num_keys, num_buckets, bucket_start, num_edges, edge_start, ext_start, ext_num;
};

struct wko_result { QueryOut qo; };

extern "C" {

void *wko_store_build(const uint32_t *triples, uint64_t n, int num_servers, int sid, int num_engines,
                      uint64_t kvstore_bytes, int num_normal_preds, int gpu_ext_mode) {
    Store *st = new Store();
    st->sid = sid;
    st->num_servers = num_servers;
    st->num_engines = num_engines;
    st->gpu_ext_mode = gpu_ext_mode != 0;
    st->num_normal_preds = num_normal_preds;
    st->size_regions(kvstore_bytes);
    st->build(triples, n);
    return st;
}

// Wrap foreign store arrays (e.g. built by the product builder) so the oracle ENGINE can probe
// them; used by bench.py's cpu_baseline leg at scales where the serial oracle build is too slow.
void *wko_store_wrap(int num_servers, int sid, const void *vertices, uint64_t num_slots, const uint32_t *edges,
                     uint64_t num_entries, const wko_segmeta *segs, int nsegs) {
    Store *st = new Store();
    st->sid = sid;
    st->num_servers = num_servers;
    st->vertices = (vertex_t *)vertices;
    st->edges = (sid_t *)edges;
    st->num_slots = num_slots;
    st->num_entries = num_entries;
    for (int i = 0; i < nsegs; i++) {
        seg_meta_t m;
        m.num_keys = segs[i].num_keys; m.num_buckets = segs[i].num_buckets; m.bucket_start = segs[i].bucket_start;
        m.num_edges = segs[i].num_edges; m.edge_start = segs[i].edge_start;
        if (segs[i].ext_num) m.ext.push_back(ext_extent_t{segs[i].ext_num, 0, segs[i].ext_start});
        st->seg_map[segid_t{segs[i].index, segs[i].dir, segs[i].pid}] = m;
    }
    return st;
}

void wko_store_free(void *s) { delete (Store *)s; }
int wko_store_ok(void *s) { return ((Store *)s)->build_failed ? 0 : 1; }
const char *wko_store_error(void *s) { return ((Store *)s)->fail_msg.c_str(); }
const void *wko_store_vertices(void *s) { return ((Store *)s)->vertices; }
const uint32_t *wko_store_edges(void *s) { return ((Store *)s)->edges; }
uint64_t wko_store_num_slots(void *s) { return ((Store *)s)->num_slots; }
uint64_t wko_store_num_buckets(void *s) { return ((Store *)s)->num_buckets; }
uint64_t wko_store_num_entries(void *s) { return ((Store *)s)->num_entries; }
uint64_t wko_store_used_entries(void *s) { return ((Store *)s)->last_entry; }
uint64_t wko_store_used_ext(void *s) { return ((Store *)s)->last_ext; }
int wko_store_num_segs(void *s) { return (int)((Store *)s)->seg_map.size(); }
void wko_store_segs(void *s, wko_segmeta *out) {
    int i = 0;
    for (auto &kv : ((Store *)s)->seg_map) {
        wko_segmeta &m = out[i++];
        memset(&m, 0, sizeof(m));
        m.index = kv.first.index; m.dir = kv.first.dir; m.pid = kv.first.pid;
        m.num_keys = kv.second.num_keys; m.num_buckets = kv.second.num_buckets; m.bucket_start = kv.second.bucket_start;
        m.num_edges = kv.second.num_edges; m.edge_start = kv.second.edge_start;
        if (!kv.second.ext.empty()) {   // contiguous in gpu_ext_mode (single extent)
            m.ext_start = kv.second.ext[0].start;
            m.ext_num = kv.second.ext[0].num_ext_buckets;
        }
    }
}
uint64_t wko_store_check(void *s) { return store_check(*(Store *)s); }

// probe one key; returns size, *out = pointer to the edge run (or NULL)
uint64_t wko_get_edges(void *s, uint32_t vid, uint32_t pid, int dir, const uint32_t **out) {
    uint64_t sz = 0;
    const sid_t *p = ((Store *)s)->get_edges_local(vid, pid, dir, sz);
    if (out) *out = p;
    return sz;
}
uint64_t wko_hash_u64(uint64_t k) { return hash_u64(k); }
uint64_t wko_hash_prime_u64(uint64_t k) { return hash_prime_u64(k); }
uint64_t wko_make_ptr(uint64_t size, uint64_t off) { return make_ptr(size, off); }
int wko_is_tpid(int64_t id) { return is_tpid(id) ? 1 : 0; }
int wko_less_pso(const uint32_t *a, const uint32_t *b) { return less_pso(triple_t{a[0], a[1], a[2]}, triple_t{b[0], b[1], b[2]}) ? 1 : 0; }
int wko_less_pos(const uint32_t *a, const uint32_t *b) { return less_pos(triple_t{a[0], a[1], a[2]}, triple_t{b[0], b[1], b[2]}) ? 1 : 0; }
uint64_t wko_make_key(uint64_t vid, uint64_t pid, uint64_t dir) { return make_key(vid, pid, dir); }

// apply a .fmt plan text to n patterns (4 int32 each: subject, predicate, direction, object);
// out must hold room for max_out patterns.  Returns the new pattern count, or -1.
int wko_set_plan(const int32_t *pats, int n, const char *fmt, int32_t *out, int max_out) {
    std::vector<Pattern> p(n);
    for (int i = 0; i < n; i++) p[i] = Pattern{pats[4 * i], pats[4 * i + 1], pats[4 * i + 2], pats[4 * i + 3]};
    if (!set_plan(p, fmt)) return -1;
    if ((int)p.size() > max_out) return -1;
    for (size_t i = 0; i < p.size(); i++) {
        out[4 * i] = p[i].subject; out[4 * i + 1] = p[i].predicate; out[4 * i + 2] = p[i].direction; out[4 * i + 3] = p[i].object;
    }
    return (int)p.size();
}

// Run one query over a cluster of `nstores` simulated servers.
wko_result *wko_query_run(void **stores, int nstores, const int32_t *pats, int npat, int nvars,
                          const int32_t *required, int nreq, int mt_factor, int blind, int threaded) {
    Cluster cl;
    for (int i = 0; i < nstores; i++) cl.stores.push_back((Store *)stores[i]);
    std::vector<Pattern> p(npat);
    for (int i = 0; i < npat; i++) p[i] = Pattern{pats[4 * i], pats[4 * i + 1], pats[4 * i + 2], pats[4 * i + 3]};
    std::vector<ssid_t> req(required, required + nreq);
    wko_result *r = new wko_result();
    run_query(cl, p, nvars, req, mt_factor < 1 ? 1 : mt_factor, blind != 0, threaded != 0, r->qo);
    return r;
}
// ... with the query modifiers of final_process (SPARQLQuery::distinct / offset / limit)
wko_result *wko_query_run_ex(void **stores, int nstores, const int32_t *pats, int npat, int nvars,
                             const int32_t *required, int nreq, int mt_factor, int blind, int threaded,
                             int distinct, int64_t offset, int64_t limit) {
    Cluster cl;
    for (int i = 0; i < nstores; i++) cl.stores.push_back((Store *)stores[i]);
    std::vector<Pattern> p(npat);
    for (int i = 0; i < npat; i++) p[i] = Pattern{pats[4 * i], pats[4 * i + 1], pats[4 * i + 2], pats[4 * i + 3]};
    std::vector<ssid_t> req(required, required + nreq);
    wko_result *r = new wko_result();
    Modifiers md;
    md.distinct = distinct != 0; md.offset = offset; md.limit = limit;
    run_query(cl, p, nvars, req, mt_factor < 1 ? 1 : mt_factor, blind != 0, threaded != 0, r->qo, md);
    return r;
}
void wko_result_free(wko_result *r) { delete r; }
int wko_result_status(wko_result *r) { return r->qo.result.status_code; }
uint64_t wko_result_rows(wko_result *r) { return (uint64_t)r->qo.result.row_num; }
int wko_result_cols(wko_result *r) { return r->qo.result.col_num; }
const uint32_t *wko_result_table(wko_result *r) { return r->qo.result.result_table.data(); }
uint64_t wko_result_table_len(wko_result *r) { return r->qo.result.result_table.size(); }
double wko_result_usec(wko_result *r) { return r->qo.usec; }

// Closed-loop "emulator" for the throughput comparison (reference proxy.hpp:391-545 runs an open loop of light
// queries over the engine threads): nq blind queries, split statically over nthreads host threads, each thread
// running execute_patterns back to back.  rows[q] receives each query's row count.  Returns wall seconds.
double wko_emu_run(void *store, const int32_t *pats, const int32_t *pat_off, const int32_t *nvars, int nq, int nthreads,
                   uint64_t *rows) {
    Cluster cl;
    cl.stores.push_back((Store *)store);
    if (nthreads < 1) nthreads = 1;
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) {
        th.emplace_back([&, t]() {
            std::vector<ssid_t> req;
            for (int q = t; q < nq; q += nthreads) {
                std::vector<Pattern> p;
                for (int i = pat_off[q]; i < pat_off[q + 1]; i++) p.push_back(Pattern{pats[4 * i], pats[4 * i + 1], pats[4 * i + 2], pats[4 * i + 3]});
                QueryOut qo;
                run_query(cl, p, nvars[q], req, 1, true, false, qo);
                rows[q] = (uint64_t)qo.result.row_num;
            }
        });
    }
    for (auto &x : th) x.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// Single-primitive entry points for kernel-level parity tests: run exactly one pattern function
// on a given input table.  kind: 0 i2u, 1 c2u, 2 k2u, 3 k2k, 4 k2c, 6 c2k, 7 i2k.  Returns rows; fills out.
// For k2u `pid/dir` select the segment, col_start the probed column; k2k uses col_end, k2c end_const.
int64_t wko_run_primitive(void *store, int kind, const uint32_t *table, uint64_t nrows, int ncols,
                          int32_t a_start, int32_t pid, int dir, int32_t a_end, int mt_tid, int mt_factor,
                          uint32_t *out, uint64_t out_cap_words, int *out_cols) {
    Cluster cl;
    cl.stores.push_back((Store *)store);
    Engine eng{&cl, 0};
    Query q;
    // synthetic variable binding: column c holds variable -(c+1); the new variable is -(ncols+1)
    q.result.nvars = ncols + 1;
    q.result.v2c_map.assign(ncols + 1, NO_RESULT);
    q.result.col_num = ncols;
    for (int c = 0; c < ncols; c++) q.result.v2c_map[c] = c;
    if (table) q.result.result_table.assign(table, table + nrows * ncols);
    q.mt_tid = mt_tid;
    q.mt_factor = mt_factor < 1 ? 1 : mt_factor;
    ssid_t newvar = -(ncols + 1);
    try {
        switch (kind) {
        case 0: q.patterns.push_back(Pattern{a_start, pid, dir, newvar}); eng.index_to_unknown(q); break;
        case 1: q.patterns.push_back(Pattern{a_start, pid, dir, newvar}); eng.const_to_unknown(q); break;
        case 2: q.patterns.push_back(Pattern{-(a_start + 1), pid, dir, newvar}); eng.known_to_unknown(q); break;
        case 3: q.patterns.push_back(Pattern{-(a_start + 1), pid, dir, -(a_end + 1)}); eng.known_to_known(q); break;
        case 4: q.patterns.push_back(Pattern{-(a_start + 1), pid, dir, a_end}); eng.known_to_const(q); break;
        case 6: q.patterns.push_back(Pattern{a_start, pid, dir, -(a_end + 1)}); eng.const_to_known(q); break;
        case 7: q.patterns.push_back(Pattern{a_start, pid, dir, -(a_end + 1)}); eng.index_to_known(q); break;
        default: return -1;
        }
    } catch (OracleError &e) { return -(int64_t)e.code - 1000; }
    if (out_cols) *out_cols = q.result.col_num;
    uint64_t len = q.result.result_table.size();
    if (out && len <= out_cap_words) memcpy(out, q.result.result_table.data(), len * sizeof(uint32_t));
    return q.result.col_num ? (int64_t)(len / q.result.col_num) : 0;
}

}  // extern "C"
