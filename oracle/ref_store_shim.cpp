// TEST INFRASTRUCTURE ONLY.  The reference's OWN graph store -- core/store/static_gstore.hpp + gstore.hpp + meta.hpp
// + vertex.hpp + mem.hpp, read in place from a Wukong checkout, never copied -- compiled against the std-based
// stand-ins for Boost / TBB / ZeroMQ in oracle/ref_stubs/ (those libraries are not in this image; see
// ref_stubs/README.md), behind a small C interface: build a store from id triples exactly as the loader hands
// them to StaticGStore::init (base_loader.hpp:308-378: partition by owner and engine, PSO / POS sort with the
// reference's comparators, dedup), read the raw arrays and segment table back, and probe with GStore::get_edges.
// What this pins: segment sizing, insert_key / ext-bucket chaining, edge layout, index lists and the probe --
// i.e. SURVEY.md §8 rows a3-a5 -- of the oracle (and through it the product builders) against compiled
// reference code.  What it does not exercise: the loader's file reading, RDMA / TCP paths, attributes.
// Built by `make -C oracle ref` into oracle/_ref/ (git-ignored).
#include "ref_shim.h"

TCP_Adaptor *con_adaptor = nullptr;   // gstore.hpp:1057 (metadata sync between servers; never reached with one server)

namespace {
void dedup(std::vector<triple_t> &t) {   // base_loader.hpp:81-95
    if (t.size() <= 1) return;
    uint64_t n = 1;
    for (uint64_t i = 1; i < t.size(); i++) {
        if (t[i].s == t[i - 1].s && t[i].p == t[i - 1].p && t[i].o == t[i - 1].o) continue;
        t[n++] = t[i];
    }
    t.resize(n);
}
}  // namespace

extern "C" {

// one server `sid` of `num_servers`; memstore_gb whole GiB (Global::memstore_size_gb is an int)
void *refs_build(const uint32_t *tr, uint64_t n, int num_servers, int sid, int num_engines, int memstore_gb, int num_normal_preds) {
    // One engine: the build then runs single-threaded, which keeps the std-based container stand-ins out of the reference's
    // OpenMP loops (TBB's element locks are only approximated there).  What a probe can observe does not depend on the engine
    // count; only the per-engine partition of the sorted triple lists does.
    num_engines = 1;
    Global::num_servers = num_servers;
    Global::num_engines = num_engines;
    Global::num_threads = num_engines + 1;
    Global::memstore_size_gb = memstore_gb;
    Global::use_rdma = false;
    Global::enable_vattr = false;
    RefStore *r = new RefStore();
    r->mem = new Mem(num_servers, Global::num_threads);
    // The object is created as "server 0 of 1": StaticGStore::init ends by exchanging segment metadata with every OTHER
    // server over TCP (gstore.hpp:905-941), and there is no transport here.  Which triples this shard holds is decided
    // below, by the loader's owner rule with the real (num_servers, sid); the store's content does not depend on its id.
    r->g = new StaticGStore(0, r->mem);
    r->g->num_normal_preds = num_normal_preds;   // base_loader.hpp:424
    r->g->num_attr_preds = 0;
    std::vector<std::vector<triple_t>> pso(num_engines), pos(num_engines);
    std::vector<std::vector<triple_attr_t>> sav(num_engines);
    for (uint64_t i = 0; i < n; i++) {           // aggregate_data, base_loader.hpp:343-361
        const sid_t s = tr[3 * i], p = tr[3 * i + 1], o = tr[3 * i + 2];
        if (wukong::math::hash_mod(s, num_servers) == sid) pso[s % num_engines].push_back(triple_t(s, p, o));
        if (wukong::math::hash_mod(o, num_servers) == sid) pos[o % num_engines].push_back(triple_t(s, p, o));
    }
    for (int t = 0; t < num_engines; t++) {      // base_loader.hpp:363-373
        std::sort(pso[t].begin(), pso[t].end(), triple_sort_by_pso());
        std::sort(pos[t].begin(), pos[t].end(), triple_sort_by_pos());
        dedup(pos[t]);
        dedup(pso[t]);
    }
    Global::num_servers = 1;   // init() ends with a metadata exchange over TCP with the other servers: none here
    r->g->refresh();           // base_loader.hpp:468 (also the only place last_ext / last_entry get their initial value)
    r->g->init(pso, pos, sav);
    for (auto &kv : r->g->rdf_seg_meta_map) {
        const segid_t &id = kv.first;
        const rdf_seg_meta_t &m = kv.second;
        uint64_t e0s = 0, e0n = 0;
        // get_ext_bucket_list_size(): the list is a vector in the CPU build and a fixed array under -DUSE_GPU (meta.hpp:86-111)
        if (m.get_ext_bucket_list_size() > 0) { e0s = m.ext_bucket_list[0].start; e0n = m.ext_bucket_list[0].num_ext_buckets; }
        const uint64_t row[11] = {(uint64_t)id.index, (uint64_t)id.dir, (uint64_t)id.pid, m.num_keys, m.num_buckets, m.bucket_start,
                                  m.num_edges, m.edge_start, (uint64_t)m.get_ext_bucket_list_size(), e0s, e0n};
        r->segs.insert(r->segs.end(), row, row + 11);
    }
    return r;
}
// releases the 1 GiB store memory; the small GStore object itself is leaked on purpose (its destructor chain is not
// exercised by the reference either: a server never tears its store down)
// A reference GStore over EXISTING arrays (the product host builder's, which are bit-identical to what StaticGStore::init
// lays out, see tests/test_reference_pin.py): used to time the reference's own engine on stores that would take its
// single-threaded build here many minutes (LUBM-2560).  segs: nsegs rows of (index, dir, pid, num_keys, num_buckets,
// bucket_start, num_edges, edge_start, ext_start, ext_num).  The arrays must outlive the handle.
void *refs_adopt(const void *vertices, uint64_t num_slots, uint64_t num_main_buckets, const void *edges, uint64_t num_edges,
                 const uint64_t *segs, int nsegs, int num_normal_preds) {
    Global::num_servers = 1;
    Global::num_engines = 1;
    Global::num_threads = 2;
    Global::memstore_size_gb = 1;   // Mem insists on whole GiB; its own buffer stays unused
    Global::use_rdma = false;
    RefStore *r = new RefStore();
    r->mem = new Mem(1, Global::num_threads);
    r->g = new StaticGStore(0, r->mem);
    r->g->num_normal_preds = num_normal_preds;
    r->g->num_attr_preds = 0;
    r->g->vertices = (vertex_t *)vertices;
    r->g->edges = (edge_t *)edges;
    r->g->num_slots = num_slots;
    r->g->num_buckets = num_main_buckets;
    r->g->num_buckets_ext = num_slots / GStore::ASSOCIATIVITY - num_main_buckets;
    r->g->num_entries = num_edges;
    r->g->last_ext = 0;
    r->g->last_entry = num_edges;
    for (int i = 0; i < nsegs; i++) {
        const uint64_t *x = segs + 10 * i;
        rdf_seg_meta_t m;
        m.num_keys = x[3]; m.num_buckets = x[4]; m.bucket_start = x[5]; m.num_edges = x[6]; m.edge_start = x[7];
        if (x[9]) m.add_ext_buckets(ext_bucket_extent_t(x[9], x[8]));
        r->g->rdf_seg_meta_map[segid_t((int)x[0], (sid_t)x[2], (int)x[1])] = m;
        r->segs.insert(r->segs.end(), x, x + 8);
        r->segs.push_back(x[9] ? 1 : 0); r->segs.push_back(x[8]); r->segs.push_back(x[9]);
    }
    return r;
}

void refs_free(void *h) { RefStore *r = (RefStore *)h; delete r->mem; delete r; }
uint64_t refs_num_slots(void *h) { return ((RefStore *)h)->g->num_slots; }
uint64_t refs_num_buckets(void *h) { return ((RefStore *)h)->g->num_buckets; }
uint64_t refs_num_entries(void *h) { return ((RefStore *)h)->g->num_entries; }
uint64_t refs_last_ext(void *h) { return ((RefStore *)h)->g->last_ext; }
uint64_t refs_last_entry(void *h) { return ((RefStore *)h)->g->last_entry; }
const void *refs_vertices(void *h) { return ((RefStore *)h)->g->vertices; }
const void *refs_edges(void *h) { return ((RefStore *)h)->g->edges; }
int refs_num_segs(void *h) { return (int)(((RefStore *)h)->segs.size() / 11); }
const uint64_t *refs_segs(void *h) { return ((RefStore *)h)->segs.data(); }
// the reference's probe: GStore::get_edges_local (gstore.hpp:393-410; bucket_local :242-248, get_vertex_local :341-361).
// GStore::get_edges (:1043-1054) only adds the owner test hash_mod(vid, num_servers) == sid in front of it and sends
// foreign keys to the RDMA path; a shard store is probed for its own keys here.
uint64_t refs_get_edges(void *h, uint32_t vid, uint32_t pid, int dir, const uint32_t **out) {
    uint64_t sz = 0;
    int type = 0;   // the default argument is a reference bound to *(int *)NULL (gstore.hpp:394): give it a real object
    edge_t *e = ((RefStore *)h)->g->get_edges_local(0, vid, pid, (dir_t)dir, sz, type);
    *out = (const uint32_t *)e;
    return e ? sz : 0;
}


}  // extern "C"
