// Sharded execution: the store is partitioned by vid % nranks (reference utils/math.hpp:51-55,
// base_loader.hpp:343-351); before a step whose start variable is not the current sharding column
// the binding table is bucketised by row[col] % nranks and exchanged all-to-all(v) over NCCL
// (replaces generate_sub_query + the Bundle/RDMA hop: sparql.hpp:746-814, gpu_hash.cu:599-760,
// gpu_engine_cuda.hpp:364-407).  Included by engine.cu (needs wk_engine internals).
#pragma once
#include <dlfcn.h>
#include <nccl.h>

// ---- bucketise-by-owner kernels -----------------------------------------------------------------
enum { MAX_PARTS = 64 };

// counts[MAX_PARTS - 1] carries this rank's overflow verdict to the other ranks (nparts < MAX_PARTS): after an overflow the
// row count of the table is a claim, not a fill level, and the table must not be walked
__global__ void __launch_bounds__(CTA_THREADS) part_count_kernel(const uint32_t *in, const uint64_t *in_count, int C, int col,
                                                                 uint32_t nparts, uint64_t *counts, const uint32_t *status) {
    __shared__ uint32_t hist[MAX_PARTS];
    if (threadIdx.x < MAX_PARTS) hist[threadIdx.x] = 0;
    __syncthreads();
    if (__ldcg(status) != 0) {
        if (blockIdx.x == 0 && threadIdx.x == 0) counts[MAX_PARTS - 1] = 1;
        return;
    }
    const uint64_t N = ld_count(in_count);
    for (uint64_t r = (uint64_t)blockIdx.x * CTA_THREADS + threadIdx.x; r < N; r += (uint64_t)gridDim.x * CTA_THREADS)
        atomicAdd(&hist[ld_table(in + r * (uint64_t)C + col) % nparts], 1u);
    __syncthreads();
    if (threadIdx.x < nparts && hist[threadIdx.x]) atomicAdd((unsigned long long *)&counts[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
}

// replicate mode of the NCCL path: every destination receives the whole table
__global__ void dup_counts_kernel(uint64_t *counts, const uint64_t *in_count, int n, const uint32_t *status) {
    const int d = threadIdx.x;
    const bool bad = __ldcg(status) != 0;
    if (d < MAX_PARTS) counts[d] = (d < n && !bad) ? ld_count(in_count) : 0;
    if (d == MAX_PARTS - 1 && bad) counts[d] = 1;
}

__global__ void part_scan_kernel(const uint64_t *counts, uint64_t *cursor, uint32_t nparts) {
    uint64_t acc = 0;
    for (uint32_t d = 0; d < nparts; d++) { cursor[d] = acc; acc += counts[d]; }
}

// each tile reserves a run per destination, then places its rows (order inside a run is free)
__global__ void __launch_bounds__(CTA_THREADS) part_scatter_kernel(const uint32_t *in, const uint64_t *in_count, int C, int col,
                                                                   uint32_t nparts, uint64_t *cursor, uint32_t *out, const uint32_t *status) {
    __shared__ uint32_t hist[MAX_PARTS];
    __shared__ uint64_t base[MAX_PARTS];
    if (__ldcg(status) != 0) return;
    const uint64_t N = ld_count(in_count);
    for (uint64_t t0 = (uint64_t)blockIdx.x * CTA_THREADS; t0 < N; t0 += (uint64_t)gridDim.x * CTA_THREADS) {
        if (threadIdx.x < MAX_PARTS) hist[threadIdx.x] = 0;
        __syncthreads();
        const uint64_t r = t0 + threadIdx.x;
        uint32_t d = 0, local = 0;
        if (r < N) {
            d = ld_table(in + r * (uint64_t)C + col) % nparts;
            local = atomicAdd(&hist[d], 1u);
        }
        __syncthreads();
        if (threadIdx.x < nparts && hist[threadIdx.x])
            base[threadIdx.x] = atomicAdd((unsigned long long *)&cursor[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
        __syncthreads();
        if (r < N) {
            const uint32_t *src = in + r * (uint64_t)C;
            uint32_t *dst = out + (base[d] + local) * (uint64_t)C;
            for (int c = 0; c < C; c++) dst[c] = ld_table(src + c);
        }
        __syncthreads();
    }
}

// ---- NCCL through dlopen (no link-time dependency; shares the copy torch may already have loaded) ----
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

static NcclApi &nccl_api() {
    static NcclApi api;
    if (api.h) return api;
    api.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.h) api.h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!api.h) { fprintf(stderr, "[wukong_b200] cannot load libnccl: %s\n", dlerror()); return api; }
#define WK_NCCL_SYM(field, name) *(void **)(&api.field) = dlsym(api.h, name)
    WK_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
    WK_NCCL_SYM(CommInitRank, "ncclCommInitRank");
    WK_NCCL_SYM(CommDestroy, "ncclCommDestroy");
    WK_NCCL_SYM(GroupStart, "ncclGroupStart");
    WK_NCCL_SYM(GroupEnd, "ncclGroupEnd");
    WK_NCCL_SYM(Send, "ncclSend");
    WK_NCCL_SYM(Recv, "ncclRecv");
    WK_NCCL_SYM(AllGather, "ncclAllGather");
    WK_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef WK_NCCL_SYM
    api.ok = api.GetUniqueId && api.CommInitRank && api.GroupStart && api.GroupEnd && api.Send && api.Recv && api.AllGather;
    return api;
}

#define NCCL_TRY(x)                                                                                        \
    do {                                                                                                   \
        ncclResult_t _r = (x);                                                                             \
        if (_r != ncclSuccess) {                                                                           \
            fprintf(stderr, "[wukong_b200] NCCL error at %s:%d: %s\n", __FILE__, __LINE__,                 \
                    nccl_api().GetErrorString ? nccl_api().GetErrorString(_r) : "?");                      \
            return WK_ERR_COMM;                                                                            \
        }                                                                                                  \
    } while (0)

struct wk_comm {
    ncclComm_t comm = nullptr;
    int nranks = 1, rank = 0;
    uint64_t *d_counts = nullptr;    // [MAX_PARTS] rows per destination
    uint64_t *d_cursor = nullptr;    // [MAX_PARTS] running offsets
    uint64_t *d_matrix = nullptr;    // [nranks][MAX_PARTS] all-gathered counts
    uint64_t *h_matrix = nullptr;    // pinned copy
    uint64_t part_rows[MAX_PARTS] = {0}, part_off[MAX_PARTS] = {0};
    bool partitioned = false;
    uint64_t exchanges = 0, rows_sent = 0, rows_recv = 0, bytes_pushed = 0;
    // peer-memory path (CUDA IPC)
    bool p2p_ready = false;
    struct XchCtl *d_xctl = nullptr;
    struct P2PLocal *d_p2p_local = nullptr;
    struct P2PTable *p2p = nullptr;     // host copy of the peer pointer table (passed to kernels by value)
    uint64_t epoch = 0;
    bool poisoned = false;              // a barrier timed out (WK_ERR_COMM): the epochs of the ranks may be skewed, rebuild the group
    bool local_group = false;           // peers are engines of this process (wk_comm_local_group): pointers wired directly
    std::vector<void *> ipc_opened;
    // peers' stores mapped through CUDA IPC (in-place light queries): header / edge arrays and segment tables per rank
    bool peer_stores = false;
    const uint4 *peer_v[8] = {nullptr};
    const uint32_t *peer_e[8] = {nullptr};
    std::vector<std::map<std::tuple<int, uint32_t, int>, wk_segmeta_t>> peer_segs;
    SegLite *d_segr_tab = nullptr;      // [segment slot of my store][LIGHT_PEERS]: the sharded light-query server's segment directory
};

// Which steps need an exchange: out[i] = -1 none, -2 replicate to every rank, c >= 0 re-shard by column c.
// Mirrors need_fork_join()/local_var (sparql.hpp:802-814) and dispatch(r,false) for type-index
// lookups of a known variable (sparql.hpp:1091-1110).
static void plan_exchanges(const std::vector<PlannedStep> &steps, std::vector<int> &out) {
    out.assign(steps.size(), -1);
    int shard_col = -1;
    for (size_t i = 0; i < steps.size(); i++) {
        const PlannedStep &ps = steps[i];
        if (ps.kind == KIND_I2U) { shard_col = 0; continue; }     // local index slice: the new column is local
        if (ps.kind == KIND_C2U) { shard_col = -1; continue; }    // rows only on the owner of the constant
        if (ps.kind == KIND_C2K) continue;                        // refused by the sharded executor (OBJ_ERROR, sparql.hpp:808)
        if (ps.kind == KIND_K2U && ps.pid == WK_TYPE_ID && ps.dir == WK_DIR_IN) {
            out[i] = -2;
            shard_col = ps.in_cols;   // the appended instances are local to the rank that found them
            continue;
        }
        if (ps.col_start != shard_col) { out[i] = ps.col_start; shard_col = ps.col_start; }
    }
}

// =============================================================================================
// Peer-memory exchange (NVLink / NVSwitch, no NCCL, no host synchronisation), ONE pass over the table:
//   ready   (1 CTA)  every rank tells every peer "all my earlier kernels are done" and waits for the same from them:
//                    the peers' next-table buffers and receive counters may now be written;
//   push    (grid)   tiles of rows are fetched with cp.async into a double buffer, grouped by owner in shared memory, space
//                    for the owners' runs is reserved with ONE atomic per (chunk of up to 8 tiles, owner) on the owner's
//                    receive counter -- a remote atomic over NVLink for the peers -- and the runs are stored STRAIGHT INTO
//                    the owners' next-table buffers as 16-byte stores; the last CTA fences system-wide and raises the
//                    "pushed" flags (multi-device groups take barrier "ready" inside this kernel);
//   wait    (1 CTA)  every peer has pushed: the receive counter is the new row count.
// No count pass, no count matrix, no second pass over the table (round 1: count -> publish -> scatter -> wait).
// Buffers and control blocks of the peers are mapped with CUDA IPC (one process per GPU) or wired directly for engines
// of one process (wk_comm_local_group).
// =============================================================================================
struct XchCtl {
    uint64_t flagA[MAX_PARTS];               // epoch of the last "ready" seen from each rank
    uint64_t flagB[MAX_PARTS];               // epoch of the last completed push seen from each rank
    uint64_t flagL[MAX_PARTS];               // light query answered in place by rank r: 2 * epoch (+ 1: redo it collectively)
    uint64_t ovf[MAX_PARTS];                 // epoch at which rank r met a full buffer (its own or an owner's)
    uint64_t recv_count;                     // rows reserved in my next-table buffer during the running exchange (all ranks add)
    uint64_t poison;                         // a rank gave up waiting: nobody pushes any more until the group is rebuilt
};

struct P2PTable {
    uint32_t *buf[2][MAX_PARTS / 4];         // peers' result buffers (up to 16 ranks per box)
    XchCtl *ctl[MAX_PARTS / 4];
    int nranks, rank;
};
enum { P2P_MAX_RANKS = MAX_PARTS / 4 };
enum { P2P_CHUNK_TILES = 8 };    // tiles per reservation of the push kernel (see p2p_push_kernel): the chunks of all CTAs together must stay in L2

struct P2PLocal {                            // device scratch of one rank
    uint32_t done_ctas;
    uint32_t ovf;                            // some CTA of the running push met a full buffer
    uint64_t rows_sent, rows_landed, rows_kept;   // running totals over all exchanges (wk_comm_stats): pushed to peers, arrived here (own included), own
    uint64_t bytes_pushed;                   // bytes stored into peers' buffers (NVLink traffic of the data path)
    uint64_t sent_mark;                      // rows_sent when the running exchange began
};

// st_sys_u64 / ld_sys_u64 / wait_flag (bounded spin on a peer-written flag): wk_light.cuh

// barrier A.  A rank that gives up poisons the whole group: a late peer must not push into a buffer that may already
// hold another query's table.
__global__ void p2p_ready_kernel(P2PTable t, XchCtl *my, P2PLocal *loc, uint64_t epoch, uint32_t *status) {
    const int p = threadIdx.x;
    __shared__ int ok;
    if (p == 0) { ok = 1; loc->done_ctas = 0; loc->ovf = 0; loc->sent_mark = loc->rows_sent; }
    __syncthreads();
    if (p < t.nranks) {
        __threadfence_system();
        st_sys_u64(&t.ctl[p]->flagA[t.rank], epoch);
        if (!wait_flag(&my->flagA[p], epoch)) atomicExch(&ok, 0);
    }
    __syncthreads();
    if (!ok) {
        if (p < t.nranks) st_sys_u64(&t.ctl[p]->poison, 1);
        if (p == 0) atomicOr(status, 2u);
    }
}

// x % n for n <= 2^16 without a division: magic = ceil(2^32 / n) (host side; n = 1 is handled by the caller)
__host__ __device__ __forceinline__ uint32_t mod_small(uint32_t x, uint32_t n, uint32_t magic) {
#ifdef __CUDA_ARCH__
    const uint32_t q = __umulhi(x, magic);       // floor(x / n) or one more
#else
    const uint32_t q = (uint32_t)(((uint64_t)x * magic) >> 32);
#endif
    int32_t r = (int32_t)(x - q * n);
    if (r < 0) r += (int32_t)n;
    return (uint32_t)r;
}

// L words of shared memory -> global words dst[0 .. L): the head up to the first 16-byte boundary of dst and the tail as
// 4-byte stores, the body as 16-byte stores (one 512-byte request per warp instead of four 128-byte ones: what crosses NVLink
// is full-width).  All threads of the CTA take part.
__device__ __forceinline__ void push_run(uint32_t *dst, const uint32_t *src, uint32_t L, uint32_t tid) {
    const uint32_t mis = (uint32_t)((reinterpret_cast<uintptr_t>(dst) >> 2) & 3u);
    uint32_t head = (4u - mis) & 3u;
    if (head > L) head = L;
    const uint32_t nvec = (L - head) >> 2, tail = L - head - (nvec << 2);
    if (tid < head) dst[tid] = src[tid];
    uint4 *dv = reinterpret_cast<uint4 *>(dst + head);
    const uint32_t *sv = src + head;
    for (uint32_t v = tid; v < nvec; v += CTA_THREADS) {
        uint4 x;
        x.x = sv[4 * v]; x.y = sv[4 * v + 1]; x.z = sv[4 * v + 2]; x.w = sv[4 * v + 3];
        dv[v] = x;
    }
    if (tid < tail) dst[head + (nvec << 2) + tid] = src[head + (nvec << 2) + tid];
}

// one pass: tile -> group by owner -> reserve -> push.  RPT rows per thread: tile = 256 * RPT rows.
// ready_inside: barrier A is taken inside this kernel (one launch less per exchange): CTA 0 tells every peer that this rank's
// earlier kernels are done, and every CTA waits for all peers' word before its first store into a peer's buffer.  Only for
// ranks on different devices: on a shared device a grid of waiting CTAs could keep a peer's kernel from becoming resident.
//
// Pipeline of a CTA (scripts/exchange_bench.py --variants: with the reservations and the remote stores switched off the
// first version of this kernel still took most of its time -- it was bound by its own load -> sync -> rank -> sync ->
// reserve -> sync -> stage -> sync -> store -> sync chain, not by NVLink):
//   * tiles are fetched with 16-byte cp.async into a double buffer: tile i + 1 is in flight while tile i is grouped;
//   * three barriers per tile: rows landed | ranks known | staged; every warp derives the run offsets it needs from the
//     tile's histogram by a shuffle scan, only warp 0 publishes them (and reserves) for the store phase;
//   * the reservation of a tile's space is either free (chunk mode: G > 1 consecutive tiles were counted and reserved at
//     once) or a remote atomic issued by warp 0 while the other warps stage;
//   * runs leave as 16-byte stores (push_run).
// gmax: most tiles per reservation (P2P_CHUNK_TILES; WK_P2P_G overrides it for experiments).  dbg (WK_P2P_DEBUG, timing
// experiments of scripts/exchange_bench.py only -- the received tables are garbage): 1 = rows owned by peers are not stored,
// 2 = no reservations (every tile writes at its own row index).
template <int RPT>
__global__ void __launch_bounds__(CTA_THREADS, 5) p2p_push_kernel(P2PTable t, XchCtl *my, P2PLocal *loc, const uint32_t *in, const uint64_t *in_count,
                                                                  int C, int col, int dup, int dst_buf, uint64_t epoch, uint64_t cap_rows,
                                                                  uint32_t *status, int ready_inside, int gmax, int dbg, uint32_t nmagic) {
    extern __shared__ __align__(16) uint32_t p2p_dyn[];
    constexpr uint32_t TILE = CTA_THREADS * RPT;
    const uint32_t tile_words = TILE * (uint32_t)C;
    uint32_t *stage = p2p_dyn + 2 * (size_t)tile_words;
    __shared__ uint32_t hist[2][P2P_MAX_RANKS], off[P2P_MAX_RANKS + 1], chist[P2P_MAX_RANKS];
    __shared__ uint64_t base[P2P_MAX_RANKS];
    __shared__ uint32_t last, s_ovf;
    __shared__ int s_ok;
    const uint32_t n = (uint32_t)t.nranks;
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    if (ready_inside) {
        if (tid == 0) s_ok = 1;
        __syncthreads();
        if (tid < n) {
            if (blockIdx.x == 0) {
                __threadfence_system();
                st_sys_u64(&t.ctl[tid]->flagA[t.rank], epoch);
            }
            if (!wait_flag(&my->flagA[tid], epoch)) atomicExch(&s_ok, 0);
        }
        __syncthreads();
        if (!s_ok) {   // a peer never showed up: poison the group, push nothing (the flags below still go out)
            if (tid < n) st_sys_u64(&t.ctl[tid]->poison, 1);
            if (tid == 0) atomicOr(status, 2u);
            __syncthreads();
        }
    }
    // an earlier step of this rank overflowed (its table is not usable), or the group is poisoned: push nothing, but
    // still take part in the barriers so that the ranks stay in step
    const bool bad = __ldcg(status) != 0 || ld_sys_u64(&my->poison) != 0;
    const uint64_t N = bad ? 0 : ld_count(in_count);
    if (tid == 0) s_ovf = (__ldcg(status) & 1u) ? 1u : 0u;
    if (tid < P2P_MAX_RANKS) { hist[0][tid] = 0; hist[1][tid] = 0; }
    uint64_t sent = 0, kept = 0;      // threads tid < n: rows reserved at owner tid
    uint64_t cbase = 0;               // threads tid < n: start of the running chunk's reservation at owner tid (~0: refused)
    uint32_t crun = 0;                //                  rows of the chunk already placed there
    // Space in the owners' buffers is reserved per CHUNK of G consecutive tiles when the table is long enough: the reservation
    // is an atomic on ONE word per owner that every CTA of every rank hits (measured on 2 GPUs, 64 M rows: one reservation per
    // tile costs 0.34 ms of 1.10 ms).  The chunk is counted first (key column only: that pass also pulls the chunk into L2),
    // its tiles then come from L2.  G grows with the table: a table of up to one tile per CTA keeps per-tile reservations.
    const uint64_t tiles_total = (N + TILE - 1) / TILE;
    uint32_t G = (uint32_t)(tiles_total / (uint64_t)gridDim.x);
    G = G < 1 ? 1 : (G > (uint32_t)gmax ? (uint32_t)gmax : G);
    const uint64_t CH = (uint64_t)G * TILE, stride = (uint64_t)gridDim.x * CH;
    const bool chunked = dup || G > 1;

    // fetch rows [t0, t0 + nrows) into buffer b; one cp.async group per tile (empty groups keep the count regular)
    auto fetch = [&](uint32_t b, uint64_t t0, uint32_t nrows) {
        const uint32_t words = nrows * (uint32_t)C;
        const uint32_t *src = in + t0 * (uint64_t)C;
        if (nrows == TILE && (tile_words & 3u) == 0) {
            const uint32_t d0 = (uint32_t)__cvta_generic_to_shared(p2p_dyn + (size_t)b * tile_words);
            for (uint32_t v = tid; v < (words >> 2); v += CTA_THREADS) cp_async16(d0 + v * 16, src + v * 4);
        } else {
            uint32_t *dstw = p2p_dyn + (size_t)b * tile_words;
            for (uint32_t w = tid; w < words; w += CTA_THREADS) dstw[w] = ld_table(src + w);
        }
        cp_async_commit();
    };
    uint64_t c0 = (uint64_t)blockIdx.x * CH;     // start of the running chunk
    uint32_t q0 = 0, p = 0;                      // running tile's offset inside the chunk; its buffer
    if (c0 < N) fetch(0, c0, (uint32_t)((N - c0 < TILE) ? (N - c0) : TILE));
    __syncthreads();
    while (c0 < N) {
        const uint32_t crows = (uint32_t)((N - c0 < CH) ? (N - c0) : CH);
        // ---- chunk prologue: count and reserve ----------------------------------------------------------------------------
        if (q0 == 0 && chunked) {
            if (!dup) {
                if (tid < P2P_MAX_RANKS) chist[tid] = 0;
                __syncthreads();
                const uint32_t *key = in + c0 * (uint64_t)C + col;
                for (uint32_t r0 = 0; r0 < crows; r0 += 16 * CTA_THREADS) {      // 16 independent loads in flight per thread
                    uint32_t d[16];
#pragma unroll
                    for (int j = 0; j < 16; j++) {
                        const uint32_t r = r0 + (uint32_t)j * CTA_THREADS + tid;
                        d[j] = r < crows ? ld_table(key + (uint64_t)r * C) : 0xFFFFFFFFu;
                    }
#pragma unroll
                    for (int j = 0; j < 16; j++) {
                        // lanes with the same owner elect one of them to add their number (rows past the end share owner ~0)
                        const uint32_t dj = d[j] == 0xFFFFFFFFu ? 0xFFFFFFFFu : (n == 1 ? 0u : mod_small(d[j], n, nmagic));
                        const uint32_t m = __match_any_sync(0xFFFFFFFFu, dj);
                        if (lane == (uint32_t)__ffs(m) - 1u && dj != 0xFFFFFFFFu) atomicAdd(&chist[dj], __popc(m));
                    }
                }
                __syncthreads();
            }
            if (tid < n) {
                const uint32_t want = dup ? crows : chist[tid];
                uint64_t b = 0;
                if (dbg & 2) {
                    b = c0;
                } else if (want) {
                    b = atomicAdd_system((unsigned long long *)&t.ctl[tid]->recv_count, (unsigned long long)want);
                    if (b + want > cap_rows) { b = ~0ull; s_ovf = 1; }   // the owner's buffer is full: drop the run, flag it
                    else if (tid != (uint32_t)t.rank) sent += want;
                    else kept += want;
                }
                cbase = b;
                crun = 0;
            }
        }
        // ---- the running tile; the next one (same chunk, or the first of this CTA's next chunk) is fetched meanwhile -------
        const uint64_t t0 = c0 + q0;
        const uint32_t nrows = (crows - q0 < TILE) ? (crows - q0) : TILE;
        const uint32_t words = nrows * (uint32_t)C;
        uint64_t nc0 = c0;
        uint32_t nq0 = q0 + TILE;
        if (nq0 >= crows) { nc0 = c0 + stride; nq0 = 0; }
        if (nc0 < N) {
            const uint64_t left = N - (nc0 + nq0);
            const uint64_t cleft = ((N - nc0 < CH) ? (N - nc0) : CH) - nq0;
            const uint64_t m = left < cleft ? left : cleft;
            fetch(p ^ 1u, nc0 + nq0, (uint32_t)(m < TILE ? m : TILE));
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();                                            // (A) the tile's rows are in shared memory
        const uint32_t *rows = p2p_dyn + (size_t)p * tile_words;
        if (!dup) {
            if (tid < P2P_MAX_RANKS) hist[p ^ 1u][tid] = 0;       // the next tile's histogram
            uint32_t d[RPT], local[RPT];
#pragma unroll
            for (int j = 0; j < RPT; j++) {
                const uint32_t r = tid + (uint32_t)j * CTA_THREADS;
                d[j] = r < nrows ? (n == 1 ? 0u : mod_small(rows[r * C + col], n, nmagic)) : 0xFFFFFFFFu;
                // rank of the row among the tile's rows of the same owner: the lanes of a warp that share an owner elect a leader,
                // which takes their places with one shared-memory atomic
                const uint32_t m = __match_any_sync(0xFFFFFFFFu, d[j]);
                const uint32_t leader = (uint32_t)__ffs(m) - 1u;
                uint32_t wb = 0;
                if (lane == leader && d[j] != 0xFFFFFFFFu) wb = atomicAdd(&hist[p][d[j]], __popc(m));
                wb = __shfl_sync(0xFFFFFFFFu, wb, leader);
                local[j] = wb + __popc(m & ((1u << lane) - 1u));
            }
            __syncthreads();                                        // (B) the histogram is complete
            // exclusive prefix of the histogram (rows), by every warp for itself: lane dd holds owner dd's run start
            const uint32_t hv = lane < n ? hist[p][lane] : 0;
            uint32_t incl = hv;
#pragma unroll
            for (int o = 1; o < P2P_MAX_RANKS; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if ((int)lane >= o) incl += y;
            }
            const uint32_t excl = incl - hv;
            if (tid < n) {                                          // warp 0 publishes run offsets and destinations
                off[tid] = excl * (uint32_t)C;
                if (tid == n - 1) off[n] = incl * (uint32_t)C;
                uint64_t b = 0;
                if (chunked) {
                    b = cbase == ~0ull ? ~0ull : cbase + crun;
                    crun += hv;
                } else if (dbg & 2) {
                    b = t0;
                } else if (hv) {
                    b = atomicAdd_system((unsigned long long *)&t.ctl[tid]->recv_count, (unsigned long long)hv);
                    if (b + hv > cap_rows) { b = ~0ull; s_ovf = 1; }
                    else if (tid != (uint32_t)t.rank) sent += hv;
                    else kept += hv;
                }
                base[tid] = b;
            }
#pragma unroll
            for (int j = 0; j < RPT; j++) {
                const uint32_t r = tid + (uint32_t)j * CTA_THREADS;
                const uint32_t o = __shfl_sync(0xFFFFFFFFu, excl, d[j] & 31u);
                if (r < nrows) {
                    uint32_t *q = stage + (o + local[j]) * (uint32_t)C;
                    for (int c = 0; c < C; c++) q[c] = rows[r * C + c];
                }
            }
            __syncthreads();                                        // (C) staged, destinations known
            for (uint32_t dd = 0; dd < n; dd++) {
                const uint64_t b = base[dd];
                const uint32_t L = off[dd + 1] - off[dd];
                if (b == ~0ull || L == 0 || ((dbg & 1) && dd != (uint32_t)t.rank)) continue;
                push_run(t.buf[dst_buf][dd] + b * (uint64_t)C, stage + off[dd], L, tid);
            }
        } else {
            if (tid < n) base[tid] = cbase == ~0ull ? ~0ull : cbase + q0;
            __syncthreads();
            for (uint32_t dd = 0; dd < n; dd++) {
                if (base[dd] == ~0ull || ((dbg & 1) && dd != (uint32_t)t.rank)) continue;
                push_run(t.buf[dst_buf][dd] + base[dd] * (uint64_t)C, rows, words, tid);
            }
            __syncthreads();   // base[] is rewritten by the next tile before its first barrier
        }
        c0 = nc0;
        q0 = nq0;
        p ^= 1u;
    }
    cp_async_wait<0>();
    if (sent) {
        atomicAdd((unsigned long long *)&loc->rows_sent, (unsigned long long)sent);
        atomicAdd((unsigned long long *)&loc->bytes_pushed, (unsigned long long)(sent * (uint64_t)C * 4ull));
    }
    if (kept) atomicAdd((unsigned long long *)&loc->rows_kept, (unsigned long long)kept);
    // completion: fence my stores system-wide, count CTAs, the last one raises the flags
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        if (s_ovf) atomicOr(&loc->ovf, 1u);
        __threadfence();
        last = (atomicAdd(&loc->done_ctas, 1u) == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (last && tid < n) {
        __threadfence_system();
        if (__ldcg(&loc->ovf)) st_sys_u64(&t.ctl[tid]->ovf[t.rank], epoch);
        __threadfence_system();
        st_sys_u64(&t.ctl[tid]->flagB[t.rank], epoch);
    }
}

// a peer of an in-place light query: wait for the owner's verdict; bit 2 of the status word asks for the collective redo
__global__ void p2p_light_wait_kernel(XchCtl *my, int owner, uint64_t epoch, uint32_t *status) {
    if (!wait_flag(&my->flagL[owner], 2 * epoch)) { atomicOr(status, 2u); return; }
    if (ld_sys_u64(&my->flagL[owner]) == 2 * epoch + 1) atomicOr(status, 4u);
}

// the owner of an in-place light query could not run it (its shard lacks a segment, ...): tell the peers anyway,
// or they would wait for a verdict that never comes
__global__ void p2p_light_verdict_kernel(P2PTable t, uint64_t value) {
    const int p = threadIdx.x;
    if (p < t.nranks && p != t.rank) st_sys_u64(&t.ctl[p]->flagL[t.rank], value);
}

// barrier B: every peer has finished pushing into my buffer; the receive counter is my new row count
__global__ void p2p_wait_kernel(P2PTable t, XchCtl *my, P2PLocal *loc, uint64_t epoch, uint64_t cap_rows, uint64_t *out_count,
                                uint32_t *status, uint64_t *stats) {
    const int p = threadIdx.x;
    __shared__ int ok, ovf;
    if (p == 0) { ok = 1; ovf = 0; }
    __syncthreads();
    if (p < t.nranks) {
        if (!wait_flag(&my->flagB[p], epoch)) atomicExch(&ok, 0);
        else if (ld_sys_u64(&my->ovf[p]) == epoch) atomicExch(&ovf, 1);
    }
    __threadfence_system();
    __syncthreads();
    if (!ok && p < t.nranks) st_sys_u64(&t.ctl[p]->poison, 1);
    if (p == 0) {
        const uint64_t cnt = ld_sys_u64(&my->recv_count);
        st_sys_u64(&my->recv_count, 0);   // nobody adds again before my next "ready"
        const uint64_t sent = loc->rows_sent - loc->sent_mark;
        loc->done_ctas = 0;               // scratch of the next exchange's push kernel (my push of this one is over: stream order)
        loc->ovf = 0;
        loc->sent_mark = loc->rows_sent;
        if (!ok) { atomicOr(status, 2u); *out_count = 0; return; }
        if (ovf || cnt > cap_rows) { atomicOr(status, 1u); *out_count = 0; return; }   // the same verdict on every rank
        *out_count = cnt;
        loc->rows_landed += cnt;
        stats[0] = sent;                  // per-exchange figures for wk_engine_step_stats (kind 10)
        stats[1] = cnt;
    }
}
