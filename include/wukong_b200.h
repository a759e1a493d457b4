/*
 * wukong_b200 — C ABI of the H100-native (sm_90a) graph-exploration engine.
 *
 * This is the drop-in boundary for ONE path of SJTU-IPADS/wukong: per-triple-pattern frontier
 * expansion over the predicate-indexed cluster-hash graph store.  The reference has no plugin
 * API; its one host->device seam is core/gpu/gpu_hash.hpp (GPUEngineParam + free functions,
 * gpu_hash.hpp:43-150) consumed by the GPUEngineCuda method set (gpu_engine_cuda.hpp:45-409).
 * Every entry point below names the reference interface it replaces (file:line relative to the
 * reference tree).  Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * Conventions
 *  - every function returns an int status: 0 = SUCCESS, 1..12 = the reference's error codes
 *    (utils/errors.hpp:28-43), >= 100 = engine errors (CUDA failure, buffer overflow, bad args).
 *    No exception crosses the ABI; the reference-side wrapper rethrows WukongException(code).
 *  - one caller thread per wk_engine_t (like the single GPUAgent thread, gpu_agent.hpp:245-290);
 *    several engines may share one wk_store_t.
 *  - the binding table lives on the device between calls (engine-owned double buffer, like
 *    GPUMem::res_inbuf/res_outbuf, gpu_mem.hpp:116-124) in the reference's layout: row-major
 *    uint32 sid_t, nrows x ncols (query.hpp:425-443).
 *  - `out_rows` may be NULL: the call is then only enqueued (no host synchronisation), which is
 *    how a whole plan is chained without a sync per pattern.
 */
#ifndef WUKONG_B200_H
#define WUKONG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint32_t wk_sid_t;  /* core/type.hpp:34-38 (sid_t, DTYPE_64BIT off) */

enum { WK_DIR_IN = 0, WK_DIR_OUT = 1 };            /* core/type.hpp:127 dir_t */
enum { WK_PREDICATE_ID = 0, WK_TYPE_ID = 1 };      /* store/vertex.hpp:38 */
#define WK_NBITS_IDX 17                            /* store/vertex.hpp:34 */
#define WK_ASSOCIATIVITY 8                         /* store/gstore.hpp:967 */

/* status codes: utils/errors.hpp:28-43, then engine-specific */
enum {
    WK_SUCCESS = 0, WK_UNKNOWN_ERROR, WK_SYNTAX_ERROR, WK_UNKNOWN_PATTERN, WK_ATTR_DISABLE,
    WK_NO_REQUIRED_VAR, WK_UNSUPPORT_UNION, WK_OBJ_ERROR, WK_VERTEX_INVALID, WK_UNKNOWN_SUB,
    WK_SETTING_ERROR, WK_FIRST_PATTERN_ERROR, WK_UNKNOWN_FILTER,
    WK_ERR_CUDA = 100,        /* a CUDA runtime call failed (reference: CUDA_ASSERT aborts, utils/gpu.hpp:26-37) */
    WK_ERR_BAD_ARG = 101,
    WK_ERR_RBUF_OVERFLOW = 102, /* result does not fit the result buffer (reference: ASSERT, gpu_engine_cuda.hpp:185) */
    WK_ERR_NO_SEGMENT = 103,  /* pattern names a (pid,dir) segment that is not in the store */
    WK_ERR_NO_DEVICE = 104,
    WK_ERR_COMM = 105,
    WK_ERR_STORE_FULL = 106   /* store build: header / ext extent / entry region too small (reference: ASSERT in
                                 gstore.hpp:414-426, 789-856) or a key with >= 2^28 edges */
};

/* 128-bit slot of the cluster-hash header region: store/vertex.hpp:152-155 (vertex_t).
 *   key = ikey_t raw bits:  dir:1 | pid:17 | vid:46   (vertex.hpp:47-50)
 *   ptr = iptr_t raw bits:  size:28 | off:34 | type:2 (vertex.hpp:116-119)               */
typedef struct { uint64_t key; uint64_t ptr; } wk_vertex_t;

/* one (index, pid, dir) segment: segid_t + rdf_seg_meta_t, store/meta.hpp:53-204.
 * ext_start/ext_num describe the segment's indirect-header extent (informational: probes follow
 * the chain pointers stored in the slots, so any number of extents works). */
typedef struct {
    int32_t index;   /* 0 normal segment, 1 index segment (vid == 0 keys)  */
    int32_t dir;
    uint32_t pid;
    uint32_t _pad;
    uint64_t num_keys, num_buckets, bucket_start, num_edges, edge_start, ext_start, ext_num;
} wk_segmeta_t;

/* one triple pattern after planning: SPARQLQuery::Pattern, core/query.hpp:95-116.
 * ids < 0 are variables (-1, -2, ...), ids >= 0 constants. */
typedef struct { int32_t subject, predicate, direction, object; } wk_pattern_t;

typedef struct wk_store wk_store_t;
typedef struct wk_engine wk_engine_t;

/* per-step execution record of the last wk_query_execute (profiling mode only for device_us) */
typedef struct {
    int32_t kind;            /* 0 i2u, 1 c2u, 2 k2u, 3 k2k, 4 k2c, 5 project, 6 c2k, 7 i2k, 8 distinct, 9 slice,
                                10 peer-memory exchange: buckets_visited = rows pushed to peers, edges_touched = rows received,
                                algo_bytes = bytes sent over NVLink; 11 fused filter chain (wk_query_execute, WK_OPT_FUSE_FILTERS) */
    int32_t in_cols;
    uint64_t in_rows, out_rows;
    uint64_t buckets_visited;   /* sum over rows of L_i  (SURVEY.md §8d)                    */
    uint64_t edges_touched;     /* sum d_i (k2u) / sum s_i (k2k,k2c) / d (i2u,c2u)          */
    uint64_t algo_bytes;        /* algorithmic bytes of the step, SURVEY.md §8d formula      */
    float device_us;            /* CUDA-event time of the step's kernel(s); 0 if not profiled */
    int32_t launches;
} wk_step_stats_t;

const char *wk_strerror(int code);
int wk_version(void);
int wk_device_count(int *count);

/* ---- store ------------------------------------------------------------------------------------
 * Replaces GPUCache(gmem, vertex_t*, edge_t*, map<segid_t, rdf_seg_meta_t>) (gpu_cache.hpp:425-467)
 * and its segment paging: the whole store is uploaded once into flat HBM arrays. The host arrays
 * stay owned by the caller (GStore::vertices / GStore::edges, gstore.hpp:962-963). */
int wk_store_create(int device, const wk_vertex_t *vertices, uint64_t num_slots,
                    const wk_sid_t *edges, uint64_t num_edges,
                    const wk_segmeta_t *segs, int nsegs, wk_store_t **out);
/* Adopt arrays that already live on `device` (e.g. produced by a device-side builder). */
int wk_store_adopt(int device, wk_vertex_t *d_vertices, uint64_t num_slots, wk_sid_t *d_edges,
                   uint64_t num_edges, const wk_segmeta_t *segs, int nsegs, int take_ownership,
                   wk_store_t **out);
/* Build the store on the device from raw id triples: replaces the loader's sort/dedup/partition
 * (loader/base_loader.hpp:308-378) + StaticGStore::init (store/static_gstore.hpp:383-454) for server `sid`
 * of `num_servers`.  Same segment table and edge array as the CPU build; slot placement inside a bucket
 * chain is free.  kvstore_bytes == 0 sizes the regions from the data (est_load_factor, global.hpp:99-104). */
typedef struct {
    int32_t num_servers, sid;
    int32_t num_normal_preds;     /* (#lines of str_index) - 1, base_loader.hpp:409-424 */
    int32_t est_load_factor;      /* 0 = 55 */
    uint64_t kvstore_bytes;
    int32_t triples_on_device;    /* `triples` is a device pointer on `device` */
    int32_t _pad;
} wk_build_opts_t;
typedef struct {
    uint64_t num_keys, num_triples_out, num_triples_in, num_buckets, num_buckets_ext, used_ext, num_slots, num_edges;
    float ms_upload, ms_sort, ms_insert, ms_total;
} wk_build_stats_t;
int wk_store_build(int device, const wk_sid_t *triples, uint64_t n, const wk_build_opts_t *opts, wk_store_t **out,
                   wk_build_stats_t *stats);
/* shape of a store, its segment table, and a copy of its arrays back to the host (checks, CPU baseline) */
int wk_store_info(wk_store_t *store, uint64_t *num_slots, uint64_t *num_edges, int *nsegs);
int wk_store_segs(wk_store_t *store, wk_segmeta_t *dst, int cap);
int wk_store_download(wk_store_t *store, wk_vertex_t *vertices, uint64_t num_slots, wk_sid_t *edges, uint64_t num_edges);
int wk_store_destroy(wk_store_t *store);
/* host-side probe of one key through the device arrays (debug / gsck-style checks) */
int wk_store_get_edges(wk_store_t *store, wk_sid_t vid, wk_sid_t pid, int dir,
                       wk_sid_t *dst, uint64_t cap, uint64_t *size);

/* ---- engine -----------------------------------------------------------------------------------
 * Replaces GPUEngineCuda(sid, GPUCache*, GPUMem*, GPUStreamPool*) (gpu_engine_cuda.hpp:80-85).
 * rbuf_bytes is the size of EACH of the two result buffers (Global::gpu_rbuf_size_mb). */
int wk_engine_create(wk_store_t *store, uint64_t rbuf_bytes, wk_engine_t **out);
int wk_engine_destroy(wk_engine_t *engine);
/* 0 off; 1 = CUDA events around each wk_query_execute (device time of the whole pattern phase);
 * 2 = additionally one event pair per step (wk_step_stats_t.device_us);
 * 3 = additionally SM-clock stamps at the phase boundaries of the fused light-query kernel */
int wk_engine_set_profiling(wk_engine_t *engine, int level);
/* Engine options.
 *  WK_OPT_RESIDENT_LIGHT (default 1; environment WK_RESIDENT=0 turns it off for a whole process, e.g. under a profiler):
 *    const-start ("light") plans are answered by a resident single-CTA server kernel that polls a doorbell in mapped pinned
 *    memory -- no kernel launch and no stream round trip per query, like the reference's resident engine threads
 *    (core/engine/engine.hpp:120-221, core/proxy.hpp:298-385).  The server leaves the device when a grid-filling kernel of
 *    this engine is about to run, when it has been idle for WK_OPT_RESIDENT_IDLE_US (default 10 000), and in
 *    wk_engine_destroy; it is relaunched on demand.  0 = one kernel launch per light query.
 *  WK_INFO_* are read-only (wk_engine_get_option). */
enum { WK_OPT_RESIDENT_LIGHT = 1, WK_OPT_RESIDENT_IDLE_US = 2,
       WK_OPT_DIRECT_OUT = 4,             /* default 0 (pays only for results of a few thousand rows): when `table` of wk_query_execute is pinned host memory the device can address
                                             (wk_host_alloc), the last step of the plan writes the projected rows straight into it
                                             (final_process fused into the step, zero-copy over PCIe) */
       WK_OPT_RESIDENT_VARIANT = 5,       /* shape of the server CTA, for A/B runs: 0 (default) / 1 / 2 / 3, see engine.cu */
       WK_OPT_FUSE_FILTERS = 3,           /* default 1: a run of consecutive known_to_known / known_to_const steps of a plan is ONE
                                             launch (rows staged once, no intermediate tables); the steps are reported as kind 11 */
       WK_INFO_RESIDENT_LAUNCHES = 100,   /* server instances launched so far */
       WK_INFO_RESIDENT_REQUESTS = 101,   /* queries answered through the doorbell */
       WK_INFO_LAST_RESIDENT = 102,       /* 1 if the last wk_query_execute was answered by the server */
       WK_INFO_LAST_RESIDENT_NS = 103,    /* its in-kernel span: request acquired -> record stored (%globaltimer) */
       WK_INFO_RESIDENT_RUNNING = 104,
       WK_INFO_COMM_BYTES_PUSHED = 110 };  /* bytes this rank has stored into peers' buffers (peer-memory exchange) */
int wk_engine_set_option(wk_engine_t *engine, int option, int64_t value);
int wk_engine_get_option(wk_engine_t *engine, int option, int64_t *value);
/* level 3 diagnostics: dst[0] entry, [1] control block cleared, [2+s] step s done, [26] table written, [27] record stored */
int wk_engine_light_trace(wk_engine_t *engine, int64_t *dst, int cap);
int wk_engine_sync(wk_engine_t *engine);                     /* CUDA_STREAM_SYNC */
int wk_engine_reset(wk_engine_t *engine);                    /* empty table, 0 columns */

/* load_result_buf(const Result&) / (const char*, size), gpu_engine_cuda.hpp:89-105 */
int wk_table_upload(wk_engine_t *engine, const wk_sid_t *table, uint64_t nrows, int ncols);
/* last-pattern device->host copy (thrust::copy into new_table), gpu_engine_cuda.hpp:189-196 */
int wk_table_download(wk_engine_t *engine, wk_sid_t *dst, uint64_t cap_words,
                      uint64_t *nrows, int *ncols);
int wk_table_info(wk_engine_t *engine, uint64_t *nrows, int *ncols);

/* ---- pattern primitives: GPUEngineCuda methods (gpu_engine_cuda.hpp:107-362) and the two seeds
 * the reference keeps on the CPU (gpu_engine.hpp:63-123); semantics = core/engine/sparql.hpp ---- */
/* index_to_unknown, sparql.hpp:194-231 (mt slicing :211-221) */
int wk_index_to_unknown(wk_engine_t *engine, wk_sid_t tpid, int dir, int mt_tid, int mt_factor,
                        uint64_t *out_rows);
/* const_to_unknown, sparql.hpp:238-285 */
int wk_const_to_unknown(wk_engine_t *engine, wk_sid_t vid, wk_sid_t pid, int dir, uint64_t *out_rows);
/* known_to_unknown, sparql.hpp:295-407 / gpu_engine_cuda.hpp:112-197 */
int wk_known_to_unknown(wk_engine_t *engine, int col_start, wk_sid_t pid, int dir, uint64_t *out_rows);
/* known_to_known, sparql.hpp:416-476 / gpu_engine_cuda.hpp:199-281 */
int wk_known_to_known(wk_engine_t *engine, int col_start, wk_sid_t pid, int dir, int col_end,
                      uint64_t *out_rows);
/* known_to_const, sparql.hpp:484-549 / gpu_engine_cuda.hpp:283-362 */
int wk_known_to_const(wk_engine_t *engine, int col_start, wk_sid_t pid, int dir, wk_sid_t end_const,
                      uint64_t *out_rows);
/* const_to_known, sparql.hpp:144-186: keep the rows whose column col_end occurs in edges(vid, pid, dir) */
int wk_const_to_known(wk_engine_t *engine, wk_sid_t vid, wk_sid_t pid, int dir, int col_end, uint64_t *out_rows);
/* index_to_known, sparql.hpp:80-141: keep the rows whose column col_end occurs in (this mt slice of) the index list */
int wk_index_to_known(wk_engine_t *engine, wk_sid_t tpid, int dir, int col_end, int mt_tid, int mt_factor,
                      uint64_t *out_rows);
/* final_process DISTINCT, sparql.hpp:1428-1472: rows ordered by all columns (compared as signed ints, ReduceCmp :1406-1421),
 * then adjacent rows that agree on `cols` (the columns of the required variables) collapse to the first */
int wk_table_distinct(wk_engine_t *engine, const int32_t *cols, int n, uint64_t *out_rows);
/* final_process OFFSET / LIMIT, sparql.hpp:1487-1499 (limit < 0: none) */
int wk_table_slice(wk_engine_t *engine, uint64_t offset, int64_t limit, uint64_t *out_rows);
/* final_process projection, sparql.hpp:1507-1550: out[i][j] = in[i][cols[j]] */
int wk_project(wk_engine_t *engine, const int32_t *cols, int ncols_out, uint64_t *out_rows);

/* ---- whole pattern phase: SPARQLEngine::execute_patterns + final_process for one engine
 * (sparql.hpp:1113-1154, 1424-1551), i.e. what GPUAgent::execute_sparql_query drives
 * (gpu_agent.hpp:170-243).  Dispatches each step by (var_stat(subject), var_stat(object)) exactly
 * like execute_one_pattern (sparql.hpp:938-1061) and runs the plan without a host sync per step.
 * blind != 0 mirrors Result::blind / Global::silent: only the row count comes back.
 * If table != NULL (non-blind) the projected table is copied into it (cap in words). */
int wk_query_execute(wk_engine_t *engine, const wk_pattern_t *patterns, int npatterns, int nvars,
                     const int32_t *required_vars, int nrequired, int mt_tid, int mt_factor,
                     int blind, wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols);
/* The same with the query modifiers final_process applies before the projection (SPARQLQuery::distinct / offset / limit,
 * query.hpp:560-682; sparql.hpp:1428-1499): DISTINCT, then OFFSET, then LIMIT.  A blind query skips them like the reference.
 * ORDER BY compares string-server strings and is left to the host. */
typedef struct {
    int32_t mt_tid, mt_factor;
    int32_t blind;
    int32_t distinct;
    int64_t offset;      /* rows to drop, <= 0: none */
    int64_t limit;       /* rows to keep, < 0: no limit */
} wk_query_opts_t;
int wk_query_execute_ex(wk_engine_t *engine, const wk_pattern_t *patterns, int npatterns, int nvars,
                        const int32_t *required_vars, int nrequired, const wk_query_opts_t *opts,
                        wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols);
/* Throughput path for light queries (the reference's emulator, Proxy::run_query_emu, proxy.hpp:391-545, keeps many
 * light queries in flight): nqueries independent const-start plans are answered by ONE launch, one CTA per
 * query; blind replies.  patterns holds all plans back to back, pat_off[q]..pat_off[q+1] delimit plan q.
 * out_status[q] is the per-query status code (a malformed plan does not fail the batch). */
int wk_query_execute_batch(wk_engine_t *engine, const wk_pattern_t *patterns, const int32_t *pat_off,
                           const int32_t *nvars, int nqueries, uint64_t *out_rows, int32_t *out_status);
/* stats of the last wk_query_execute / primitive calls since the last reset */
int wk_engine_num_steps(wk_engine_t *engine);
int wk_engine_step_stats(wk_engine_t *engine, int step, wk_step_stats_t *out);
uint64_t wk_engine_launch_count(wk_engine_t *engine);   /* kernels launched by this engine so far */
/* device time (CUDA events on the engine's stream) of the last wk_query_execute; profiling >= 1 */
int wk_engine_last_query_device_us(wk_engine_t *engine, float *us);
/* measurement helpers: evict the L2 (overwrite a scratch buffer larger than L2, then sync) and
 * page-locked host buffers for the host<->device copies of the end-to-end path */
int wk_engine_flush_l2(wk_engine_t *engine);
int wk_host_alloc(uint64_t bytes, void **out);
int wk_host_free(void *ptr);

/* ---- sharded execution (one process per GPU): generate_sub_query / gpu_shuffle_result_buf +
 * gpu_split_result_buf (sparql.hpp:746-799; gpu_hash.cu:599-760; gpu_engine_cuda.hpp:364-407) --- */
/* Bucketise the current table by row[col_start] % nparts into contiguous per-destination runs.
 * part_rows[nparts] receives the run lengths (synchronises). */
int wk_partition(wk_engine_t *engine, int col_start, int nparts, uint64_t *part_rows);
/* Device pointer + rows of partition `part` after wk_partition (borrowed; valid until next call) */
int wk_partition_ptr(wk_engine_t *engine, int part, const wk_sid_t **d_ptr, uint64_t *rows);
/* Join a communicator: nccl_unique_id is the 128-byte ncclUniqueId created by rank 0. */
int wk_comm_unique_id(void *id128);
int wk_comm_init(wk_engine_t *engine, int nranks, int rank, const void *id128);
/* wk_partition + all-to-all(v) of the partitions over NCCL; afterwards the table holds exactly the
 * rows whose row[col_start] % nranks == rank. */
int wk_exchange(wk_engine_t *engine, int col_start, uint64_t *out_rows);
int wk_comm_stats(wk_engine_t *engine, uint64_t *exchanges, uint64_t *rows_sent, uint64_t *rows_recv);
/* Peer-memory exchange over NVLink / NVSwitch instead of NCCL (one process per GPU, CUDA IPC): every rank exports a
 * 192-byte record (handles of its two result buffers and of its exchange control block), the records of all ranks
 * are gathered by the caller (rank order) and imported.  Afterwards wk_query_execute_sharded bucketises rows by owner
 * and stores them straight into the owners' next-table buffers from the kernel, ONE pass over the table: space in an
 * owner's buffer is reserved with one (remote) atomic per tile and owner, "ready" / "pushed" flags travel through peer
 * memory too, so an exchange needs no host synchronisation at all.  Up to 16 ranks, all with the same rbuf_bytes.
 * A barrier that times out (dead peer) returns WK_ERR_COMM and poisons the group: re-import to use it again. */
int wk_comm_p2p_export(wk_engine_t *engine, int nranks, int rank, void *out192);
int wk_comm_p2p_import(wk_engine_t *engine, const void *all_handles);
int wk_exchange_p2p(wk_engine_t *engine, int col_start, uint64_t *out_rows);
/* The same group for engines of ONE process (one caller thread per engine; several shards may share a GPU): buffers, control
 * blocks and store arrays of the peers are wired directly, engines[r] becomes rank r.  In-place light queries are enabled too.
 * All engines must have the same rbuf_bytes. */
int wk_comm_local_group(wk_engine_t **engines, int n);
/* In-place light queries on a sharded store -- the reference answers small tables with one-sided RDMA reads of the remote
 * header / edge regions instead of a fork-join (sparql.hpp:802-814, Global::rdma_threshold): here every rank also maps its
 * peers' store arrays.  export_store writes [IPC handles of the header and edge arrays][segment table] (size in *size; call
 * with blob == NULL to learn it); import_store takes all ranks' blobs back to back, offsets[r] .. offsets[r + 1] = rank r.
 * Afterwards wk_query_execute_sharded runs a const-start plan of <= 12 steps on the constant's owner alone, probing the
 * other shards with loads over NVLink; a table that outgrows shared memory is redone through the exchange path. <= 8 ranks. */
int wk_comm_p2p_export_store(wk_engine_t *engine, void *blob, uint64_t cap, uint64_t *size);
int wk_comm_p2p_import_store(wk_engine_t *engine, const void *blobs, const uint64_t *offsets, int nranks);
/* Host-only planning helper: out[i] = -1 no exchange before step i, -2 replicate the table to every
 * shard (type-index lookup of a known variable, sparql.hpp:1091-1110), c >= 0 re-shard by column c
 * (need_fork_join with local_var, sparql.hpp:802-814).  Needs no GPU. */
int wk_plan_exchanges(const wk_pattern_t *patterns, int npatterns, int nvars, int32_t *out);
/* Sharded whole-query execution: like wk_query_execute, with the store sharded by vid % nranks
 * and an exchange before every step whose start variable is not local (need_fork_join,
 * sparql.hpp:802-814).  out_rows is this rank's share of the result. */
int wk_query_execute_sharded(wk_engine_t *engine, const wk_pattern_t *patterns, int npatterns, int nvars,
                             const int32_t *required_vars, int nrequired, int mt_tid, int mt_factor,
                             int blind, wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols);

#ifdef __cplusplus
}
#endif
#endif /* WUKONG_B200_H */
