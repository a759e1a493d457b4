// wukong_b200 GPU engine: kernels + C-ABI (include/wukong_b200.h).  sm_90a (H100) only.
//
// Design (H100-first, not a port of the reference's core/gpu):
//   * the whole cluster-hash store lives in flat HBM arrays (no segment paging / block maps);
//   * one fused kernel per pattern step: probe -> multiplicity -> tile scan -> materialise,
//     persistent grid sized from the SM count, row counts stay on the device between steps
//     so a plan runs without a host synchronisation per pattern (the reference does 5 launches,
//     a D2H copy and 2 stream syncs per pattern: gpu_engine_cuda.hpp:112-197);
//   * const-start ("light") plans run as ONE single-CTA kernel that interprets the plan and
//     reports through mapped pinned memory (launch-latency bound, not bandwidth bound);
//   * completion/row counts come back through a mapped pinned record, not a cudaMemcpy.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "wukong_b200.h"
#include "wk_device.cuh"
#include "wk_light.cuh"
#include "wk_server.cuh"
#include "wk_internal.h"

using namespace wk;

// =============================================================================================
// device-side control block and kernels
// =============================================================================================
enum { MAX_STEPS = 60 };
enum { KIND_I2U = 0, KIND_C2U = 1, KIND_K2U = 2, KIND_K2K = 3, KIND_K2C = 4, KIND_PROJECT = 5, KIND_C2K = 6, KIND_I2K = 7, KIND_DISTINCT = 8, KIND_SLICE = 9, KIND_EXCHANGE = 10, KIND_FILTER = 11 };

struct CtlBlock {
    uint64_t counts[MAX_STEPS + 4];       // counts[s] = rows of the table that step s reads
    uint64_t stats[2 * (MAX_STEPS + 4)];  // per step: buckets visited, edges touched
    uint64_t hq_packed[MAX_STEPS + 4];    // per step: heavy-tile queue (entries:24 | chunks:40)
    uint64_t hq_ticket[MAX_STEPS + 4];    // per step: chunk ticket dispenser
    uint32_t status;                      // sticky: bit0 = result buffer overflow
    uint32_t _pad;
};

static_assert(sizeof(CtlBlock) % sizeof(uint64_t) == 0, "CtlBlock is cleared in 8-byte words");

// Programmatic dependent launch (sm_90+): the kernels of a plan are launched with the programmatic-stream-serialization
// attribute, so the launch of step s+1 is set up while step s still runs and only its body waits -- here, before the first
// read of anything the previous kernel wrote.  Without the attribute the instruction is a no-op.
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// completion record in mapped pinned host memory: wk::LightRecord (32 bytes, two 16-byte stores,
// validated on the host by record_check instead of a system-scope fence on the device)
typedef LightRecord HostRec;

struct SeedParam {
    const uint4 *vertices;
    const uint32_t *edges;
    uint32_t *out;
    uint64_t *out_count;
    uint64_t out_cap_rows;
    uint64_t *stats;
    uint32_t *status;
    uint64_t key;
    uint64_t bucket_start;
    FastMod fm;
    int32_t mt_tid, mt_factor;
};

struct ProjParam {
    const uint32_t *in;
    uint32_t *out;
    const uint64_t *in_count;
    uint64_t *out_count;
    uint64_t out_cap_rows;
    uint32_t *status;
    int32_t C, Cn;
    int8_t cols[MAX_COLS];
};

// ---- known_to_{unknown,known,const}: one persistent fused kernel ---------------------------------
// BATCH / MINB: probe batch size and minimum resident CTAs per SM (register budget); see DESIGN.md
// CT: compile-time column count (1..4), 0 = read it from the parameters
template <int MODE, int BATCH, int MINB, int CT>
__global__ void __launch_bounds__(CTA_THREADS, MINB) step_kernel(const StepParam p) {
    extern __shared__ uint32_t dyn_rows[];
    __shared__ TileSmem sm;
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;   // an earlier step overflowed: its output is not usable
    const uint64_t N = ld_count(p.in_count);
    uint64_t acc_visited = 0, acc_edges = 0;
    for (uint64_t tile = blockIdx.x; tile * TILE_ROWS < N; tile += gridDim.x) {
        const uint64_t row0 = tile * TILE_ROWS;
        const uint32_t nrows = (uint32_t)((N - row0 < (uint64_t)TILE_ROWS) ? (N - row0) : (uint64_t)TILE_ROWS);
        process_tile<MODE, BATCH, CT>(p, row0, nrows, sm, dyn_rows, acc_visited, acc_edges);
    }
    flush_stats(p.stats, acc_visited, acc_edges);
}

// v5: warp-autonomous pipeline (see wk_device.cuh).  Dynamic smem: [bucket staging 32 KB][8 warps x 3 x rows]
template <int MODE, int MINB, int CT, bool PROJ = false>
__global__ void __launch_bounds__(CTA_THREADS, MINB) step_kernel_v5(const StepParam p) {
    extern __shared__ __align__(16) unsigned char dyn5[];
    __shared__ TileSmem4 sm;
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;
    step_body_v5<MODE, CT, PROJ>(p, ld_count(p.in_count), sm, dyn5);
}

template <int CT>
__global__ void __launch_bounds__(CTA_THREADS, 8) expand_heavy_kernel(const StepParam p) {
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;
    expand_heavy_body<CT>(p);
}

// ---- probe of ONE key by the first 8 lanes of a warp (seeds) ---------------------------------------
__device__ __forceinline__ uint64_t probe_single(const uint4 *__restrict__ vertices, uint64_t key, uint64_t bucket,
                                                 int lane, uint32_t &visited) {
    uint64_t result = 0;
    visited = 0;
    while (true) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (lane < 8) v = ld_slot(vertices + (bucket * 8 + lane));
        const uint64_t kk = (uint64_t)v.x | ((uint64_t)v.y << 32);
        const uint64_t pp = (uint64_t)v.z | ((uint64_t)v.w << 32);
        const uint32_t hit = __ballot_sync(0xFFFFFFFFu, lane < 7 && kk == key && kk != 0);
        const uint64_t chain = __shfl_sync(0xFFFFFFFFu, kk, 7);
        visited++;
        if (hit) {
            result = __shfl_sync(0xFFFFFFFFu, pp, __ffs(hit) - 1);
            break;
        }
        if (chain == 0) break;
        bucket = chain >> WK_KEY_VID_SHIFT;
    }
    return result;
}

// body shared by seed_kernel and the fused light kernel.  nblocks/bid describe the cooperating CTAs.
__device__ __forceinline__ void seed_body(const SeedParam &p, uint64_t *s_ptr, uint32_t bid, uint32_t nblocks) {
    const int tid = threadIdx.x;
    if (tid < 32) {
        uint32_t visited;
        const uint64_t bucket = p.bucket_start + fastmod(hash_u64(p.key), p.fm);
        const uint64_t ptr = probe_single(p.vertices, p.key, bucket, tid, visited);
        if (tid == 0) {
            *s_ptr = ptr;
            if (bid == 0) atomicAdd((unsigned long long *)&p.stats[0], (unsigned long long)visited);
        }
    }
    __syncthreads();
    const uint64_t ptr = *s_ptr;
    const uint64_t size = ptr_size(ptr), off = ptr_off(ptr);
    // mt slicing exactly as sparql.hpp:211-221: length = sz / mt_factor, the last one takes the tail
    const uint64_t start = (uint64_t)(p.mt_tid % p.mt_factor);
    const uint64_t length = size / (uint64_t)p.mt_factor;
    const uint64_t begin = start * length;
    const uint64_t len = (start == (uint64_t)p.mt_factor - 1) ? (size - begin) : length;
    if (len > p.out_cap_rows) {
        if (bid == 0 && tid == 0) { atomicOr(p.status, 1u); *p.out_count = len; }
        return;
    }
    const uint32_t *src = p.edges + off + begin;
    const uint64_t stride = (uint64_t)nblocks * CTA_THREADS;
    uint64_t k = (uint64_t)bid * CTA_THREADS + tid;
    for (; k + 3 * stride < len; k += 4 * stride) {   // 4 independent loads in flight per thread
        const uint32_t a0 = ld_edge(src + k), a1 = ld_edge(src + k + stride), a2 = ld_edge(src + k + 2 * stride),
                       a3 = ld_edge(src + k + 3 * stride);
        p.out[k] = a0; p.out[k + stride] = a1; p.out[k + 2 * stride] = a2; p.out[k + 3 * stride] = a3;
    }
    for (; k < len; k += stride) p.out[k] = ld_edge(src + k);
    if (bid == 0 && tid == 0) {
        *p.out_count = len;
        atomicAdd((unsigned long long *)&p.stats[1], (unsigned long long)len);
    }
}

__global__ void __launch_bounds__(CTA_THREADS) seed_kernel(const SeedParam p) {
    __shared__ uint64_t s_ptr;
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;
    seed_body(p, &s_ptr, blockIdx.x, gridDim.x);
}

// ---- index_to_unknown / const_to_unknown with the copy engine (sm_90+ bulk asynchronous copies) ----------------------
// The seed of a heavy query is a plain copy of millions of ids.  Instead of every thread issuing loads and waiting for
// them, one elected thread per CTA asks the TMA unit for a whole 16 KB chunk (cp.async.bulk global -> shared, completion on
// an mbarrier), three chunks in flight per CTA; the chunk leaves again as ONE bulk store (shared -> global) when source and
// destination agree modulo 16 bytes, otherwise through 16-byte vector stores of the re-aligned words.  No registers are
// held while the data is in flight and the SM issues two instructions per 16 KB instead of thousands.
namespace bulk {
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void load(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void store(void *gdst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void store_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
}  // namespace bulk

enum { SEED_STAGES = 3, SEED_CHUNK_WORDS = 4096, SEED_STAGE_BYTES = SEED_CHUNK_WORDS * 4 + 128 };

__global__ void __launch_bounds__(CTA_THREADS) seed_bulk_kernel(const SeedParam p) {
    extern __shared__ __align__(128) unsigned char seed_dyn[];
    __shared__ __align__(8) uint64_t bar[SEED_STAGES];
    __shared__ uint64_t s_ptr;
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < SEED_STAGES; i++) bulk::mbar_init(&bar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < 32) {
        uint32_t visited;
        const uint64_t bucket = p.bucket_start + fastmod(hash_u64(p.key), p.fm);
        const uint64_t ptr = probe_single(p.vertices, p.key, bucket, tid, visited);
        if (tid == 0) {
            s_ptr = ptr;
            if (blockIdx.x == 0) atomicAdd((unsigned long long *)&p.stats[0], (unsigned long long)visited);
        }
    }
    __syncthreads();
    const uint64_t ptr = s_ptr;
    const uint64_t size = ptr_size(ptr), off = ptr_off(ptr);
    // mt slicing exactly as sparql.hpp:211-221: length = sz / mt_factor, the last one takes the tail
    const uint64_t start = (uint64_t)(p.mt_tid % p.mt_factor);
    const uint64_t length = size / (uint64_t)p.mt_factor;
    const uint64_t begin = start * length;
    const uint64_t len = (start == (uint64_t)p.mt_factor - 1) ? (size - begin) : length;
    if (len > p.out_cap_rows) {
        if (blockIdx.x == 0 && tid == 0) { atomicOr(p.status, 1u); *p.out_count = len; }
        return;
    }
    const uint32_t *src = p.edges + off + begin;
    const uint32_t shw = (uint32_t)(((uintptr_t)src >> 2) & 3u);          // words by which the source is off a 16-byte boundary
    const uint64_t nchunks = (len + SEED_CHUNK_WORDS - 1) / SEED_CHUNK_WORDS;
    // chunk k of this CTA is chunk blockIdx.x + k * gridDim.x of the list
    auto chunk_words = [&](uint64_t c) -> uint32_t {
        const uint64_t w0 = c * SEED_CHUNK_WORDS;
        return (uint32_t)((len - w0 < (uint64_t)SEED_CHUNK_WORDS) ? (len - w0) : (uint64_t)SEED_CHUNK_WORDS);
    };
    // bytes the copy engine moves for a chunk: whole 16-byte units inside [aligned start, end of the chunk's words)
    auto bulk_bytes = [&](uint32_t n) -> uint32_t { return ((shw + n) * 4u) & ~15u; };
    auto issue = [&](uint64_t c, int stage) {
        const uint32_t n = chunk_words(c);
        const uint32_t bytes = bulk_bytes(n);
        if (bytes) {
            const uint32_t *a0 = src + c * SEED_CHUNK_WORDS - shw;          // 16-byte aligned, never before the edge array
            bulk::mbar_expect_tx(&bar[stage], bytes);
            bulk::load(seed_dyn + (size_t)stage * SEED_STAGE_BYTES, a0, bytes, &bar[stage]);
        }
    };
    uint64_t c = blockIdx.x;
    if (tid == 0) {
        uint64_t cc = c;
        for (int s = 0; s < SEED_STAGES - 1 && cc < nchunks; s++, cc += gridDim.x) issue(cc, s);
    }
    uint32_t it = 0;
    for (; c < nchunks; c += gridDim.x, it++) {
        const int stage = (int)(it % SEED_STAGES);
        if (tid == 0) {
            // the stage this load goes to was drained by every thread (and by its bulk store) in the previous iteration
            const uint64_t cn = c + (uint64_t)(SEED_STAGES - 1) * gridDim.x;
            if (cn < nchunks) issue(cn, (int)((it + SEED_STAGES - 1) % SEED_STAGES));
        }
        const uint32_t n = chunk_words(c);
        const uint32_t bytes = bulk_bytes(n);
        uint32_t *dst = p.out + c * SEED_CHUNK_WORDS;
        const uint32_t *sm = reinterpret_cast<const uint32_t *>(seed_dyn + (size_t)stage * SEED_STAGE_BYTES);
        const uint32_t avail = bytes ? bytes / 4u - shw : 0u;    // words of this chunk that arrive through shared memory
        if (bytes) bulk::mbar_wait(&bar[stage], (it / SEED_STAGES) & 1u);
        if (shw == 0 && bytes) {
            // same alignment on both sides: the chunk leaves as one bulk store
            if (tid == 0) {
                bulk::store(dst, sm, bytes);
                bulk::store_commit();
            }
        } else {
            const uint32_t nvec = avail >> 2;
            for (uint32_t v = tid; v < nvec; v += CTA_THREADS) {
                const uint32_t *q = sm + shw + 4 * v;
                *reinterpret_cast<uint4 *>(dst + 4 * v) = make_uint4(q[0], q[1], q[2], q[3]);
            }
            for (uint32_t w = nvec * 4 + tid; w < avail; w += CTA_THREADS) dst[w] = sm[shw + w];
        }
        for (uint32_t w = avail + tid; w < n; w += CTA_THREADS) dst[w] = ld_edge(src + c * SEED_CHUNK_WORDS + w);   // ragged tail (< 4 words)
        if (tid == 0 && shw == 0 && bytes) bulk::store_wait_read_all();   // the stage may be refilled once the store has read it
        __syncthreads();
    }
    if (tid == 0) bulk::store_wait_all();
    if (blockIdx.x == 0 && tid == 0) {
        *p.out_count = len;
        atomicAdd((unsigned long long *)&p.stats[1], (unsigned long long)len);
    }
}

// ---- final_process projection -------------------------------------------------------------------
__device__ __forceinline__ void project_body(const ProjParam &p, uint64_t N, uint32_t bid, uint32_t nblocks) {
    if (N > p.out_cap_rows) {
        if (bid == 0 && threadIdx.x == 0) atomicOr(p.status, 1u);
        return;
    }
    const uint64_t nwords = N * (uint64_t)p.Cn;
    for (uint64_t w = (uint64_t)bid * CTA_THREADS + threadIdx.x; w < nwords; w += (uint64_t)nblocks * CTA_THREADS) {
        const uint64_t r = w / (uint32_t)p.Cn;
        const uint32_t j = (uint32_t)(w - r * (uint32_t)p.Cn);
        p.out[w] = ld_table(p.in + r * (uint64_t)p.C + p.cols[j]);
    }
    if (bid == 0 && threadIdx.x == 0) *p.out_count = N;
}

__global__ void __launch_bounds__(CTA_THREADS) project_kernel(const ProjParam p) {
    grid_dependency_wait();
    if (__ldcg(p.status) != 0) return;
    project_body(p, ld_count(p.in_count), blockIdx.x, gridDim.x);
}

// ---- index_to_known / const_to_known (sparql.hpp:80-186): keep the rows whose column value occurs in ONE edge list --
// The list is hashed into an engine-owned open-addressing table (lists from a reference-built store are not
// guaranteed to be sorted), then every row does one lookup.
struct ListSetCtl {
    uint64_t off, len;     // slice of the edge array that forms the set
    uint32_t mask;         // table size - 1 (power of two >= 2 * len)
    uint32_t visited;
};
static constexpr uint32_t SET_EMPTY = 0xFFFFFFFFu;   // BLANK_ID is never a vertex id (type.hpp:37)
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

struct ListParam {
    const uint4 *vertices;
    const uint32_t *edges;
    uint32_t *table;
    uint64_t table_cap;          // words available in `table`
    ListSetCtl *ctl;
    uint32_t *status;
    uint64_t key, bucket_start;
    FastMod fm;
    int32_t mt_tid, mt_factor;
};

__global__ void list_probe_kernel(const ListParam p) {
    uint32_t visited;
    const uint64_t bucket = p.bucket_start + fastmod(hash_u64(p.key), p.fm);
    const uint64_t ptr = probe_single(p.vertices, p.key, bucket, threadIdx.x, visited);
    if (threadIdx.x == 0) {
        const uint64_t size = ptr_size(ptr);
        const uint64_t mtf = (uint64_t)(p.mt_factor < 1 ? 1 : p.mt_factor), start = (uint64_t)p.mt_tid % mtf, length = size / mtf;
        const uint64_t begin = start * length;
        const uint64_t len = (start == mtf - 1) ? (size - begin) : length;   // same slicing as index_to_unknown
        uint64_t ts = 16;
        while (ts < 2 * len) ts <<= 1;
        if (ts > p.table_cap) { atomicOr(p.status, 1u); ts = 16; p.ctl->len = 0; }
        else p.ctl->len = len;
        p.ctl->off = ptr_off(ptr) + begin;
        p.ctl->mask = (uint32_t)(ts - 1);
        p.ctl->visited = visited;
    }
}

__global__ void __launch_bounds__(CTA_THREADS) list_clear_kernel(const ListParam p) {
    const uint64_t n = (uint64_t)__ldcg(&p.ctl->mask) + 1;
    for (uint64_t i = (uint64_t)blockIdx.x * CTA_THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * CTA_THREADS) p.table[i] = SET_EMPTY;
}

__global__ void __launch_bounds__(CTA_THREADS) list_insert_kernel(const ListParam p) {
    const uint64_t len = ld_count(&p.ctl->len), off = ld_count(&p.ctl->off);
    const uint32_t mask = __ldcg(&p.ctl->mask);
    for (uint64_t i = (uint64_t)blockIdx.x * CTA_THREADS + threadIdx.x; i < len; i += (uint64_t)gridDim.x * CTA_THREADS) {
        const uint32_t v = ld_edge(p.edges + off + i);
        uint32_t h = mix32(v) & mask;
        while (true) {
            const uint32_t old = atomicCAS(&p.table[h], SET_EMPTY, v);
            if (old == SET_EMPTY || old == v) break;
            h = (h + 1) & mask;
        }
    }
}

__global__ void __launch_bounds__(CTA_THREADS) list_filter_kernel(const StepParam p, const uint32_t *table, const ListSetCtl *ctl) {
    extern __shared__ uint32_t dyn_rows[];
    __shared__ TileSmem sm;
    if (__ldcg(p.status) != 0) return;
    const uint64_t N = ld_count(p.in_count);
    const uint32_t mask = __ldcg(&ctl->mask);
    const int C = p.C, tid = threadIdx.x;
    for (uint64_t tile = blockIdx.x; tile * TILE_ROWS < N; tile += gridDim.x) {
        const uint64_t row0 = tile * TILE_ROWS;
        const uint32_t nrows = (uint32_t)((N - row0 < (uint64_t)TILE_ROWS) ? (N - row0) : (uint64_t)TILE_ROWS);
        const bool active = (uint32_t)tid < nrows;
        uint32_t mult = 0;
        if (active) {
            const uint32_t *src = p.in + (row0 + tid) * (uint64_t)C;
            for (int c = 0; c < C; c++) dyn_rows[tid * C + c] = ld_table(src + c);
            const uint32_t v = dyn_rows[tid * C + p.col_end];
            uint32_t h = mix32(v) & mask;
            while (true) {
                const uint32_t x = __ldcg(table + h);
                if (x == v) { mult = 1; break; }
                if (x == SET_EMPTY) break;
                h = (h + 1) & mask;
            }
        }
        const uint64_t excl = tile_scan_and_claim(mult, sm, tid, p);
        const uint64_t base = sm.base;
        if (base != ~0ull && mult) copy_row<0>(p.out + (base + excl) * (uint64_t)C, dyn_rows + tid * C, C);
        __syncthreads();
    }
}

// ---- largest edge list per segment (one pass at store creation) ------------------------------------------
// A known_to_unknown step can only produce a "heavy" tile (>= HEAVY_TILE_MIN output rows from 256 input rows) when some
// key of its segment has at least HEAVY_TILE_MIN / TILE_ROWS edges; for all other segments the heavy-queue pass
// (one more launch per step) is skipped.  Every warp walks contiguous chunks, so it meets few segment changes and
// issues few atomics.
__global__ void __launch_bounds__(CTA_THREADS) seg_maxdeg_kernel(const uint4 *__restrict__ V, uint64_t num_slots, uint32_t P,
                                                                 uint32_t *__restrict__ tab) {
    constexpr uint64_t CHUNK = 8192;
    const uint64_t warps = (uint64_t)gridDim.x * (CTA_THREADS / 32);
    const uint64_t w = (uint64_t)blockIdx.x * (CTA_THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    for (uint64_t base = w * CHUNK; base < num_slots; base += warps * CHUNK) {
        uint32_t cur_seg = ~0u, cur_max = 0;
        const uint64_t end = base + CHUNK < num_slots ? base + CHUNK : num_slots;
        for (uint64_t i = base + lane; i < end; i += 32) {
            if ((i & 7) == 7) continue;   // chain pointer slot
            const uint4 v = __ldcs(V + i);
            const uint64_t key = (uint64_t)v.x | ((uint64_t)v.y << 32);
            if (key == 0) continue;
            const uint32_t pid = (uint32_t)(key >> 1) & ((1u << WK_NBITS_IDX) - 1);
            if (pid >= P) continue;
            const uint32_t seg = (((key >> WK_KEY_VID_SHIFT) == 0 ? 1u : 0u) * 2 + (uint32_t)(key & 1)) * P + pid;
            const uint32_t size = ptr_size((uint64_t)v.z | ((uint64_t)v.w << 32));
            if (seg != cur_seg) {
                if (cur_seg != ~0u && cur_max) atomicMax(&tab[cur_seg], cur_max);
                cur_seg = seg;
                cur_max = 0;
            }
            cur_max = size > cur_max ? size : cur_max;
        }
        if (cur_seg != ~0u && cur_max) atomicMax(&tab[cur_seg], cur_max);
    }
}

// ---- bookkeeping kernels -------------------------------------------------------------------------
__global__ void set_count_kernel(uint64_t *dst, uint64_t v) { *dst = v; }

__global__ void rebase_kernel(CtlBlock *ctl, int from, int to) {
    const uint64_t v = ctl->counts[from];
    for (int i = 0; i < MAX_STEPS + 4; i++) ctl->counts[i] = 0;
    for (int i = 0; i < 2 * (MAX_STEPS + 4); i++) ctl->stats[i] = 0;
    for (int i = 0; i < MAX_STEPS + 4; i++) { ctl->hq_packed[i] = 0; ctl->hq_ticket[i] = 0; }
    ctl->counts[to] = v;
}

__global__ void finish_kernel(const uint64_t *count, const uint32_t *status, HostRec *rec, uint64_t seq, int resume) {
    grid_dependency_wait();
    const uint64_t rows = ld_count(count);
    const uint64_t sr = (uint64_t)__ldcg(status) | ((uint64_t)(uint32_t)resume << 32);
    uint64_t *r = (uint64_t *)rec;
    st_sys_v2u64(r + 2, sr, record_check(seq, rows, sr, 0));
    st_sys_v2u64(r, seq, rows);
}

// =============================================================================================
// host side
// =============================================================================================
#define CUDA_TRY(x)                                                                                   \
    do {                                                                                              \
        cudaError_t _e = (x);                                                                         \
        if (_e != cudaSuccess) {                                                                      \
            fprintf(stderr, "[wukong_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
                    cudaGetErrorString(_e));                                                          \
            return WK_ERR_CUDA;                                                                       \
        }                                                                                             \
    } while (0)

typedef std::tuple<int, uint32_t, int> SegKey;   // (index, pid, dir)

static bool g_use_pdl = true;   // WK_PDL=0: plain stream-ordered launches
template <class... P, class... A>
static cudaError_t launch_chained(void (*fn)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A... p) {
    if (!g_use_pdl) {
        fn<<<grid, block, smem, st>>>(p...);
        return cudaGetLastError();
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, fn, p...);
}

struct wk_store {
    int device = 0;
    uint4 *d_vertices = nullptr;
    uint32_t *d_edges = nullptr;
    uint64_t num_slots = 0, num_edges = 0;
    bool owns = true;
    std::map<SegKey, wk_segmeta_t> segs;
    std::map<SegKey, uint32_t> maxdeg;   // largest edge list of a key of the segment (index segments: of the predicate's list)
    std::map<SegKey, int> seg_slot;      // slot of every segment in d_segtab (resident light-query server, wk_server.cuh)
    SegLite *d_segtab = nullptr;
    int nsegslots = 0;
};

struct StepRecord {
    int kind = 0, in_cols = 0, launches = 0;
    int s = 0;   // index into CtlBlock::counts / stats
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool timed = false;
};

struct wk_engine {
    wk_store *store = nullptr;
    cudaStream_t stream = nullptr;
    uint32_t *buf[2] = {nullptr, nullptr};
    uint64_t cap_words = 0;
    CtlBlock *d_ctl = nullptr;
    HostRec *h_rec = nullptr, *d_rec = nullptr;
    uint32_t *h_stage = nullptr, *d_stage = nullptr;
    uint64_t stage_words = 0;
    int ncols = 0;
    int step = 0;           // table is in buf[step & 1], its row count in ctl.counts[step]
    uint64_t seq = 0;
    int profiling = 0;   // 0 off, 1 query-level CUDA events, 2 also per-step events
    cudaEvent_t q_ev0 = nullptr, q_ev1 = nullptr;
    bool q_timed = false;
    int num_sms = 132;
    int occ[3] = {1, 1, 1};
    int variant = 1;
    uint64_t launches = 0;
    uint64_t light_escalate_rows = 4096;
    struct wk_comm *comm = nullptr;      // sharded execution (wk_comm_init)
    long long *d_trace = nullptr;        // light-kernel phase clocks (profiling level 3, lazy)
    uint32_t *d_set = nullptr;           // hash set of index_to_known / const_to_known (lazy)
    uint64_t set_cap = 0;
    ListSetCtl *d_setctl = nullptr;
    BatchPlan *h_bplans = nullptr, *d_bplans = nullptr;   // wk_query_execute_batch staging
    BatchResult *h_bres = nullptr, *d_bres = nullptr;
    int batch_cap = 0;
    HeavyTile *d_hq = nullptr;           // heavy-tile queue (skewed fan-out)
    uint32_t hq_cap = 0;
    void *d_flush = nullptr;             // > L2-sized scratch for wk_engine_flush_l2
    size_t flush_bytes = 0;
    int flush_gen = 0;
    // resident light-query server (wk_server.cuh)
    struct {
        bool enabled = true;             // WK_OPT_RESIDENT_LIGHT
        uint64_t idle_ns = 10ull * 1000 * 1000;
        cudaStream_t stream = nullptr;
        SrvMailbox *h_box = nullptr, *d_box = nullptr;   // mapped pinned page
        uint64_t seq = 0;                // sequence number of the last request posted (QUIT included)
        uint64_t launch_id = 0;          // 0: never launched
        bool quitting = false;           // a QUIT is on its way: wait for the exit word before relaunching
        bool sharded = false;            // the last instance launched is the sharded server (peer view, verdict flags)
        uint64_t launches = 0, requests = 0;
        uint64_t last_ns = 0;            // in-kernel span of the last request
        int variant = 0;                 // WK_OPT_RESIDENT_VARIANT (default 0): 0 = 1024 threads + warp mode, 1 = 256 + warp mode, 2 = 256, block steps only, 3 = 512 + warp mode
    } srv;
    bool last_resident = false;          // the last wk_query_execute was answered by the resident server
    // WK_OPT_DIRECT_OUT: last step writes projected rows into the caller's pinned buffer.  Off by default: row-sized
    // stores from the expand kernel cross PCIe far slower than one bulk copy of the projected table; it only pays for
    // results of a few thousand rows.
    bool direct_out = false;
    const void *dout_host = nullptr;     // last caller buffer examined, and its device address (nullptr: not device-accessible)
    uint32_t *dout_dev = nullptr;
    bool seed_bulk = true;               // seeds through cp.async.bulk (WK_SEED_BULK=0: plain loads, for A/B runs)
    bool fuse_filters = true;            // WK_OPT_FUSE_FILTERS: runs of known_to_known / known_to_const steps as one launch
    std::vector<StepRecord> recs;        // one per step since the last reset
    std::vector<cudaEvent_t> event_pool;
    size_t event_next = 0;
    // snapshot of per-step stats taken at the last synchronising call
    std::vector<wk_step_stats_t> stats;
};

extern "C" {   // defined inside the extern "C" block below
static void srv_park(wk_engine *e);   // resident light-query server: leave before a grid-filling kernel
static int srv_fill_peers(wk_engine *e, SrvPeers &Q);   // after wk_sharded.cuh
static void srv_stop(wk_engine *e);
static bool srv_exited(const wk_engine *e);
}
static void comm_free(wk_engine *e);   // wk_sharded.cuh
static uint64_t comm_bytes_pushed(const wk_engine *e);
static int preload_kernels(wk_engine *e);   // end of this file

static const char *k_errs[] = {"success", "unknown error", "syntax error", "unsupported triple pattern",
                               "attribute support disabled", "no required variables", "unsupported UNION",
                               "object should not be an index", "subject or object is not valid",
                               "triple pattern should not start from unknown subject", "setting error",
                               "const_X_X or index_X_X must be the first pattern", "unsupported filter"};

static inline bool is_tpid(int64_t id) { return id > 1 && id < (1 << WK_NBITS_IDX); }

static const wk_segmeta_t *find_seg(const wk_store *st, int index, uint32_t pid, int dir) {
    auto it = st->segs.find(SegKey(index, pid, dir));
    if (it == st->segs.end() || it->second.num_buckets == 0) return nullptr;
    return &it->second;
}
// segment of a key, store/meta.hpp:143-153 (segid_t(const ikey_t&))
static const wk_segmeta_t *seg_of_key(const wk_store *st, uint64_t vid, uint32_t pid, int dir) {
    return vid == 0 ? find_seg(st, 1, WK_PREDICATE_ID, dir) : find_seg(st, 0, pid, dir);
}

static SegParam make_segparam(const wk_segmeta_t *m, uint32_t pid, int dir, bool index_mode) {
    SegParam s;
    s.bucket_start = m->bucket_start;
    s.fm = make_fastmod(m->num_buckets);
    s.pid = pid;
    s.dir = (uint32_t)dir;
    s.index_mode = index_mode ? 1u : 0u;
    s._pad = 0;
    return s;
}

static cudaEvent_t get_event(wk_engine *e) {
    if (e->event_next == e->event_pool.size()) {
        cudaEvent_t ev;
        if (cudaEventCreate(&ev) != cudaSuccess) return nullptr;
        e->event_pool.push_back(ev);
    }
    return e->event_pool[e->event_next++];
}

static StepRecord &begin_step(wk_engine *e, int kind, int in_cols) {
    e->recs.emplace_back();
    StepRecord &r = e->recs.back();
    r.kind = kind;
    r.in_cols = in_cols;
    r.s = e->step;
    if (e->profiling >= 2) {
        r.ev0 = get_event(e);
        r.ev1 = get_event(e);
        if (r.ev0 && r.ev1) { cudaEventRecord(r.ev0, e->stream); r.timed = true; }
    }
    return r;
}
static void end_step(wk_engine *e, StepRecord &r, int launches) {
    r.launches = launches;
    e->launches += launches;
    if (r.timed) cudaEventRecord(r.ev1, e->stream);
}

static int reset_ctl(wk_engine *e) {
    CUDA_TRY(cudaMemsetAsync(e->d_ctl, 0, sizeof(CtlBlock), e->stream));
    e->step = 0;
    e->recs.clear();
    e->event_next = 0;
    return WK_SUCCESS;
}

// make room for one more step in the control block (keeps buffer parity)
static int ensure_step_room(wk_engine *e) {
    if (e->step < MAX_STEPS) return WK_SUCCESS;
    const int to = e->step & 1;
    rebase_kernel<<<1, 1, 0, e->stream>>>(e->d_ctl, e->step, to);
    CUDA_TRY(cudaGetLastError());
    e->launches++;
    e->step = to;
    e->recs.clear();
    e->event_next = 0;
    return WK_SUCCESS;
}

// Wait for the mapped completion record of sequence number `seq` (spin; falls back to the stream
// status to catch faults).  The record and an optional zero-copy result table are written without
// a device-side system fence, so they are accepted only once the record's checksum matches what
// the host reads (table_cols > 0: the table in h_stage is rows x table_cols words).
struct RecView { uint64_t rows; uint32_t status; int resume; };

static bool record_valid_at(const volatile uint64_t *r, wk_engine *e, uint64_t seq, int nsteps_full, int table_cols, RecView &out) {
    if (r[0] != seq) return false;
    const uint64_t rows = r[1], sr = r[2], check = r[3];
    uint64_t tsum = 0;
    const int resume = (int)(uint32_t)(sr >> 32);
    if (table_cols > 0 && resume == nsteps_full && (uint32_t)sr == 0 && rows > 0) {
        const uint64_t words = rows * (uint64_t)table_cols;
        if (words > e->stage_words) return false;
        const volatile uint32_t *t = (const volatile uint32_t *)e->h_stage;
        for (uint64_t i = 0; i < words; i++) tsum += table_word_mix(t[i], i);
    }
    if (record_check(seq, rows, sr, tsum) != check) return false;
    out.rows = rows;
    out.status = (uint32_t)sr;
    out.resume = resume;
    return true;
}
static bool record_valid(wk_engine *e, uint64_t seq, int nsteps_full, int table_cols, RecView &out) {
    return record_valid_at((const volatile uint64_t *)e->h_rec, e, seq, nsteps_full, table_cols, out);
}

static int wait_record(wk_engine *e, uint64_t seq, int nsteps_full, int table_cols, RecView &out) {
    uint32_t spins = 0;
    while (!record_valid(e, seq, nsteps_full, table_cols, out)) {
        if ((++spins & 0x3FF) == 0) {
            cudaError_t q = cudaStreamQuery(e->stream);
            if (q == cudaSuccess) {
                if (record_valid(e, seq, nsteps_full, table_cols, out)) break;
                CUDA_TRY(cudaStreamSynchronize(e->stream));
                if (record_valid(e, seq, nsteps_full, table_cols, out)) break;
                fprintf(stderr, "[wukong_b200] completion record missing or corrupt (seq %llu)\n", (unsigned long long)seq);
                return WK_ERR_CUDA;
            } else if (q != cudaErrorNotReady) {
                CUDA_TRY(q);
            }
        }
    }
    return WK_SUCCESS;
}

// enqueue the completion record for the current table and wait for it
static int sync_rows(wk_engine *e, uint64_t *rows, cudaEvent_t after = nullptr) {
    const uint64_t seq = ++e->seq;
    CUDA_TRY(launch_chained(finish_kernel, dim3(1), dim3(1), 0, e->stream, (const uint64_t *)&e->d_ctl->counts[e->step],
                            (const uint32_t *)&e->d_ctl->status, e->d_rec, seq, e->step));
    if (after) cudaEventRecord(after, e->stream);   // device-side end of the query, before the host waits
    e->launches++;
    RecView rv;
    int rc = wait_record(e, seq, -1, 0, rv);
    if (rc) return rc;
    if (rows) *rows = rv.rows;
    if (rv.status & 2u) return WK_ERR_COMM;          // a peer did not show up at an exchange barrier
    if (rv.status & 1u) return WK_ERR_RBUF_OVERFLOW;
    return WK_SUCCESS;
}

static size_t rows_smem(int C) { return (size_t)TILE_ROWS * (size_t)(C | 1) * sizeof(uint32_t); }
static size_t step_smem(const wk_engine *e, int C);

// kernel variants for A/B runs (WK_VARIANT): 0-3 register-staged probe with batch 8/4/4/2 and 1/4/5/6 CTAs per SM,
// 6 (default) / 7 = asynchronously staged, software-pipelined v5 with 4 / 5 CTAs per SM
#define WK_NUM_VARIANTS 8
#define WK_DEFAULT_VARIANT 6
typedef void (*StepKernelFn)(const StepParam);
template <int MODE, int CT>
static StepKernelFn step_kernel_variant(int v) {
    switch (v) {
    case 0: return step_kernel<MODE, 8, 1, CT>;
    case 1: return step_kernel<MODE, 4, 4, CT>;
    case 3: return step_kernel<MODE, 2, 6, CT>;
    case 7: return step_kernel_v5<MODE, 5, CT>;
    case 2: return step_kernel<MODE, 4, 5, CT>;
    default: return step_kernel_v5<MODE, 4, CT>;
    }
}
template <int MODE>
static StepKernelFn step_kernel_cols(int v, int C) {
    switch (C) {
    case 1: return step_kernel_variant<MODE, 1>(v);
    case 2: return step_kernel_variant<MODE, 2>(v);
    case 3: return step_kernel_variant<MODE, 3>(v);
    case 4: return step_kernel_variant<MODE, 4>(v);
    default: return step_kernel_variant<MODE, 0>(v);
    }
}
template <int MODE>
static StepKernelFn step_kernel_proj(int C) {   // last step of a non-blind plan: projected rows straight to the caller's buffer
    switch (C) {
    case 1: return step_kernel_v5<MODE, 4, 1, true>;
    case 2: return step_kernel_v5<MODE, 4, 2, true>;
    case 3: return step_kernel_v5<MODE, 4, 3, true>;
    case 4: return step_kernel_v5<MODE, 4, 4, true>;
    default: return step_kernel_v5<MODE, 4, 0, true>;
    }
}
static StepKernelFn step_kernel_fn(int mode, int v, int C) {
    return mode == MODE_K2U ? step_kernel_cols<MODE_K2U>(v, C)
         : mode == MODE_K2K ? step_kernel_cols<MODE_K2K>(v, C) : step_kernel_cols<MODE_K2C>(v, C);
}

static size_t rows_smem_v5(int C) { return (size_t)BKT_BYTES + (size_t)(CTA_THREADS / 32) * 3 * 128 * (size_t)C; }
static size_t step_smem(const wk_engine *e, int C) { return e->variant >= 4 ? rows_smem_v5(C) : rows_smem(C); }

template <int MODE>
static int launch_step(wk_engine *e, const StepParam &p) {
    const int grid = e->num_sms * e->occ[MODE];
    StepKernelFn fn = p.proj_n > 0 ? step_kernel_proj<MODE>(p.C) : step_kernel_fn(MODE, e->variant, p.C);
    const size_t smem = step_smem(e, p.C);
    if (smem > 40 * 1024) CUDA_TRY(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(launch_chained(fn, dim3(grid), dim3(CTA_THREADS), smem, e->stream, p));
    if (MODE == MODE_K2U && p.hq_cap) {   // spreads queued heavy tiles over the grid; returns at once when there are none
        const int g2 = e->num_sms * 8;
        switch (p.C) {
        case 1: CUDA_TRY(launch_chained(expand_heavy_kernel<1>, dim3(g2), dim3(CTA_THREADS), 0, e->stream, p)); break;
        case 2: CUDA_TRY(launch_chained(expand_heavy_kernel<2>, dim3(g2), dim3(CTA_THREADS), 0, e->stream, p)); break;
        case 3: CUDA_TRY(launch_chained(expand_heavy_kernel<3>, dim3(g2), dim3(CTA_THREADS), 0, e->stream, p)); break;
        default: CUDA_TRY(launch_chained(expand_heavy_kernel<0>, dim3(g2), dim3(CTA_THREADS), 0, e->stream, p)); break;
        }
    }
    return WK_SUCCESS;
}

// ---- enqueue one known_to_* step on the multi-CTA path ------------------------------------------
// extra: further known_to_known / known_to_const filters fused into the same launch (StepParam::extra); record_kind is what
// the step is reported as (KIND_FILTER for a fused chain)
struct ChainFilter { int kind, col_start, col_end, dir; uint32_t pid, end_const; };
// direct: the step is the last one of a non-blind plan and writes the projected rows straight into the caller's (pinned,
// device-accessible) buffer
struct DirectOut { uint32_t *dev_ptr; uint64_t cap_words; int n; const int32_t *cols; };
static int enqueue_known(wk_engine *e, int kind, int col_start, uint32_t pid, int dir, int col_end, uint32_t end_const,
                         const ChainFilter *extra = nullptr, int nextra = 0, const DirectOut *direct = nullptr) {
    srv_park(e);
    if (kind != KIND_K2U && kind != KIND_K2K && kind != KIND_K2C) return WK_UNKNOWN_PATTERN;
    if (e->ncols <= 0 || e->ncols > MAX_COLS - 1) return e->ncols <= 0 ? WK_FIRST_PATTERN_ERROR : WK_ERR_BAD_ARG;
    if (col_start < 0 || col_start >= e->ncols) return WK_VERTEX_INVALID;
    if (kind == KIND_K2K && (col_end < 0 || col_end >= e->ncols)) return WK_VERTEX_INVALID;
    if (dir != WK_DIR_IN && dir != WK_DIR_OUT) return WK_ERR_BAD_ARG;
    const bool index_mode = (kind == KIND_K2U && pid == WK_TYPE_ID && dir == WK_DIR_IN);   // sparql.hpp:339-340
    const wk_segmeta_t *m = index_mode ? find_seg(e->store, 1, WK_PREDICATE_ID, dir) : find_seg(e->store, 0, pid, dir);
    if (!m) return WK_ERR_NO_SEGMENT;
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    StepParam p;
    memset(&p, 0, sizeof(p));
    p.vertices = e->store->d_vertices;
    p.edges = e->store->d_edges;
    p.in = e->buf[s & 1];
    p.out = e->buf[(s + 1) & 1];
    p.in_count = &e->d_ctl->counts[s];
    p.out_count = &e->d_ctl->counts[s + 1];
    const int Cout = (kind == KIND_K2U) ? e->ncols + 1 : e->ncols;
    p.out_cap_rows = e->cap_words / (uint64_t)Cout;
    p.stats = &e->d_ctl->stats[2 * s];
    p.status = &e->d_ctl->status;
    p.seg = make_segparam(m, pid, dir, index_mode);
    p.C = e->ncols;
    p.col_start = col_start;
    p.col_end = col_end;
    p.end_const = end_const;
    p.inv_c = ((1u << 20) + (uint32_t)e->ncols - 1) / (uint32_t)e->ncols;
    if (nextra > 0) {
        if (kind == KIND_K2U || nextra > MAX_CHAIN - 1 || e->variant < 4) return WK_ERR_BAD_ARG;
        for (int f = 0; f < nextra; f++) {
            const ChainFilter &cf = extra[f];
            if (cf.col_start < 0 || cf.col_start >= e->ncols) return WK_VERTEX_INVALID;
            if (cf.kind == KIND_K2K && (cf.col_end < 0 || cf.col_end >= e->ncols)) return WK_VERTEX_INVALID;
            const wk_segmeta_t *mx = find_seg(e->store, 0, cf.pid, cf.dir);
            if (!mx) return WK_ERR_NO_SEGMENT;
            p.extra[f].seg = make_segparam(mx, cf.pid, cf.dir, false);
            p.extra[f].col_start = cf.col_start;
            p.extra[f].col_end = cf.kind == KIND_K2K ? cf.col_end : -1;
            p.extra[f].end_const = cf.end_const;
        }
        p.nextra = nextra;
    }
    // the heavy-tile pass is only needed where a tile of TILE_ROWS rows can reach HEAVY_TILE_MIN output rows
    bool may_be_heavy = true;
    {
        auto it = e->store->maxdeg.find(SegKey(m->index, m->pid, m->dir));
        if (it != e->store->maxdeg.end()) may_be_heavy = (uint64_t)it->second * TILE_ROWS >= HEAVY_TILE_MIN;
    }
    if (direct) {
        if (e->variant < 4 || direct->n <= 0 || direct->n > MAX_COLS) return WK_ERR_BAD_ARG;
        p.out = direct->dev_ptr;
        p.out_cap_rows = direct->cap_words / (uint64_t)direct->n;
        p.proj_n = direct->n;
        for (int j = 0; j < direct->n; j++) {
            if (direct->cols[j] < 0 || direct->cols[j] >= Cout) return WK_VERTEX_INVALID;
            p.proj_cols[j] = (int8_t)direct->cols[j];
        }
    }
    if (kind == KIND_K2U && e->variant >= 4 && e->d_hq && may_be_heavy && !direct) {   // queued tiles are expanded in table layout
        p.hq = e->d_hq;
        p.hq_cap = e->hq_cap;
        p.hq_packed = &e->d_ctl->hq_packed[s];
        p.hq_ticket = &e->d_ctl->hq_ticket[s];
    }
    StepRecord &r = begin_step(e, nextra > 0 ? KIND_FILTER : kind, e->ncols);
    if (kind == KIND_K2U) rc = launch_step<MODE_K2U>(e, p);
    else if (kind == KIND_K2K) rc = launch_step<MODE_K2K>(e, p);
    else rc = launch_step<MODE_K2C>(e, p);
    if (rc) return rc;
    end_step(e, r, p.hq_cap ? 2 : 1);
    e->step = s + 1;
    e->ncols = Cout;
    return WK_SUCCESS;
}

static int enqueue_seed(wk_engine *e, int kind, uint64_t vid, uint32_t pid, int dir, int mt_tid, int mt_factor) {
    srv_park(e);
    if (e->ncols != 0) return WK_FIRST_PATTERN_ERROR;
    if (dir != WK_DIR_IN && dir != WK_DIR_OUT) return WK_ERR_BAD_ARG;
    if (mt_factor < 1) mt_factor = 1;
    const wk_segmeta_t *m = seg_of_key(e->store, vid, pid, dir);
    if (!m) return WK_ERR_NO_SEGMENT;
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    SeedParam p;
    memset(&p, 0, sizeof(p));
    p.vertices = e->store->d_vertices;
    p.edges = e->store->d_edges;
    p.out = e->buf[(s + 1) & 1];
    p.out_count = &e->d_ctl->counts[s + 1];
    p.out_cap_rows = e->cap_words;
    p.stats = &e->d_ctl->stats[2 * s];
    p.status = &e->d_ctl->status;
    p.key = make_key(vid, pid, (uint32_t)dir);
    p.bucket_start = m->bucket_start;
    p.fm = make_fastmod(m->num_buckets);
    p.mt_tid = mt_tid;
    p.mt_factor = mt_factor;
    StepRecord &r = begin_step(e, kind, 0);
    if (e->seed_bulk) {
        const size_t smem = (size_t)SEED_STAGES * SEED_STAGE_BYTES;
        static bool attr_set = false;
        if (!attr_set) {
            CUDA_TRY(cudaFuncSetAttribute((const void *)seed_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_set = true;
        }
        CUDA_TRY(launch_chained(seed_bulk_kernel, dim3(e->num_sms * 4), dim3(CTA_THREADS), smem, e->stream, p));
    } else {
        CUDA_TRY(launch_chained(seed_kernel, dim3(e->num_sms * 4), dim3(CTA_THREADS), 0, e->stream, p));
    }
    end_step(e, r, 1);
    e->step = s + 1;
    e->ncols = 1;
    return WK_SUCCESS;
}

static int enqueue_project(wk_engine *e, const int32_t *cols, int n) {
    srv_park(e);
    if (n <= 0 || n > MAX_COLS) return WK_NO_REQUIRED_VAR;
    if (e->ncols <= 0) return WK_ERR_BAD_ARG;
    for (int i = 0; i < n; i++)
        if (cols[i] < 0 || cols[i] >= e->ncols) return WK_VERTEX_INVALID;
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    ProjParam p;
    memset(&p, 0, sizeof(p));
    p.in = e->buf[s & 1];
    p.out = e->buf[(s + 1) & 1];
    p.in_count = &e->d_ctl->counts[s];
    p.out_count = &e->d_ctl->counts[s + 1];
    p.out_cap_rows = e->cap_words / (uint64_t)n;
    p.status = &e->d_ctl->status;
    p.C = e->ncols;
    p.Cn = n;
    for (int i = 0; i < n; i++) p.cols[i] = (int8_t)cols[i];
    StepRecord &r = begin_step(e, KIND_PROJECT, e->ncols);
    CUDA_TRY(launch_chained(project_kernel, dim3(e->num_sms * 4), dim3(CTA_THREADS), 0, e->stream, p));
    end_step(e, r, 1);
    e->step = s + 1;
    e->ncols = n;
    return WK_SUCCESS;
}

// DISTINCT of final_process (sparql.hpp:1428-1472).  `rows` is the current row count, known on the host.
static int enqueue_distinct(wk_engine *e, const int32_t *cols, int n, uint64_t rows) {
    srv_park(e);
    if (n <= 0 || n > MAX_COLS) return WK_NO_REQUIRED_VAR;
    if (e->ncols <= 0) return WK_ERR_BAD_ARG;
    for (int i = 0; i < n; i++)
        if (cols[i] < 0 || cols[i] >= e->ncols) return WK_VERTEX_INVALID;
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    StepRecord &r = begin_step(e, KIND_DISTINCT, e->ncols);
    if (rows == 0) {
        CUDA_TRY(cudaMemsetAsync(&e->d_ctl->counts[s + 1], 0, sizeof(uint64_t), e->stream));
    } else {
        rc = wk_internal_distinct(e->stream, e->num_sms, e->buf[s & 1], e->buf[(s + 1) & 1], rows, e->ncols, cols, n,
                                  &e->d_ctl->counts[s + 1]);
        if (rc) return rc;
    }
    end_step(e, r, 3 + 5 * e->ncols);
    e->step = s + 1;
    return WK_SUCCESS;
}

// OFFSET / LIMIT of final_process (sparql.hpp:1487-1499)
static int enqueue_slice(wk_engine *e, uint64_t offset, int64_t limit, uint64_t rows_upper_bound) {
    srv_park(e);
    if (e->ncols <= 0) return WK_ERR_BAD_ARG;
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    StepRecord &r = begin_step(e, KIND_SLICE, e->ncols);
    rc = wk_internal_slice(e->stream, e->num_sms, e->buf[s & 1], &e->d_ctl->counts[s], e->ncols, offset, limit, e->buf[(s + 1) & 1],
                           &e->d_ctl->counts[s + 1], rows_upper_bound);
    if (rc) return rc;
    end_step(e, r, 1);
    e->step = s + 1;
    return WK_SUCCESS;
}

// index_to_known / const_to_known: rows whose column `col_end` occurs in the edge list of key (vid, pid, dir)
static int enqueue_to_known(wk_engine *e, int kind, uint64_t vid, uint32_t pid, int dir, int col_end, int mt_tid, int mt_factor) {
    srv_park(e);
    if (e->ncols <= 0 || e->ncols >= MAX_COLS) return e->ncols <= 0 ? WK_VERTEX_INVALID : WK_ERR_BAD_ARG;
    if (col_end < 0 || col_end >= e->ncols) return WK_VERTEX_INVALID;
    if (dir != WK_DIR_IN && dir != WK_DIR_OUT) return WK_ERR_BAD_ARG;
    const wk_segmeta_t *m = seg_of_key(e->store, vid, pid, dir);
    if (!m) return WK_ERR_NO_SEGMENT;
    if (!e->d_set) {
        e->set_cap = std::min<uint64_t>(e->cap_words, 1ull << 28);
        CUDA_TRY(cudaMalloc((void **)&e->d_set, e->set_cap * sizeof(uint32_t)));
        CUDA_TRY(cudaMalloc((void **)&e->d_setctl, sizeof(ListSetCtl)));
    }
    int rc = ensure_step_room(e);
    if (rc) return rc;
    const int s = e->step;
    ListParam lp;
    memset(&lp, 0, sizeof(lp));
    lp.vertices = e->store->d_vertices;
    lp.edges = e->store->d_edges;
    lp.table = e->d_set;
    lp.table_cap = e->set_cap;
    lp.ctl = e->d_setctl;
    lp.status = &e->d_ctl->status;
    lp.key = make_key(vid, pid, (uint32_t)dir);
    lp.bucket_start = m->bucket_start;
    lp.fm = make_fastmod(m->num_buckets);
    lp.mt_tid = mt_tid;
    lp.mt_factor = mt_factor < 1 ? 1 : mt_factor;
    StepParam p;
    memset(&p, 0, sizeof(p));
    p.in = e->buf[s & 1];
    p.out = e->buf[(s + 1) & 1];
    p.in_count = &e->d_ctl->counts[s];
    p.out_count = &e->d_ctl->counts[s + 1];
    p.out_cap_rows = e->cap_words / (uint64_t)e->ncols;
    p.stats = &e->d_ctl->stats[2 * s];
    p.status = &e->d_ctl->status;
    p.C = e->ncols;
    p.col_end = col_end;
    StepRecord &r = begin_step(e, kind, e->ncols);
    const int grid = e->num_sms * 4;
    list_probe_kernel<<<1, 32, 0, e->stream>>>(lp);
    list_clear_kernel<<<grid, CTA_THREADS, 0, e->stream>>>(lp);
    list_insert_kernel<<<grid, CTA_THREADS, 0, e->stream>>>(lp);
    list_filter_kernel<<<grid, CTA_THREADS, (size_t)TILE_ROWS * e->ncols * sizeof(uint32_t), e->stream>>>(p, e->d_set, e->d_setctl);
    CUDA_TRY(cudaGetLastError());
    end_step(e, r, 4);
    e->step = s + 1;
    return WK_SUCCESS;
}

// copy per-step counters back and derive the algorithmic bytes (SURVEY.md §8d)
static int snapshot_stats(wk_engine *e) {
    CtlBlock h;
    CUDA_TRY(cudaMemcpyAsync(&h, e->d_ctl, sizeof(CtlBlock), cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->stats.clear();
    for (size_t i = 0; i < e->recs.size(); i++) {
        const StepRecord &r = e->recs[i];
        const int s = r.s;
        wk_step_stats_t st;
        memset(&st, 0, sizeof(st));
        st.kind = r.kind;
        st.in_cols = r.in_cols;
        st.in_rows = (r.kind == KIND_I2U || r.kind == KIND_C2U) ? 0 : h.counts[s];
        st.out_rows = h.counts[s + 1];
        st.buckets_visited = h.stats[2 * s];
        st.edges_touched = h.stats[2 * s + 1];
        st.launches = r.launches;
        const uint64_t C = (uint64_t)r.in_cols, N = st.in_rows, R = st.out_rows;
        switch (r.kind) {
        case KIND_K2U: st.algo_bytes = 4 * C * N + 128 * st.buckets_visited + 4 * st.edges_touched + 4 * (C + 1) * R; break;
        case KIND_FILTER:
        case KIND_K2K:
        case KIND_K2C: st.algo_bytes = 4 * C * N + 128 * st.buckets_visited + 4 * st.edges_touched + 4 * C * R; break;
        case KIND_I2U:
        case KIND_C2U: st.algo_bytes = 128 * st.buckets_visited + 4 * R + 4 * R; break;
        case KIND_EXCHANGE:   // buckets_visited = rows pushed to peers, edges_touched = rows that landed here; NVLink bytes sent
            st.algo_bytes = 4 * C * st.buckets_visited;
            break;
        case KIND_C2K:
        case KIND_I2K:
        case KIND_DISTINCT:
        case KIND_SLICE: st.algo_bytes = 4 * C * N + 4 * C * R; break;
        default: st.algo_bytes = 4 * C * R + 4 * (uint64_t)e->ncols * R; break;
        }
        if (r.timed) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, r.ev0, r.ev1) == cudaSuccess) st.device_us = ms * 1000.0f;
        }
        e->stats.push_back(st);
    }
    return WK_SUCCESS;
}

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

const char *wk_strerror(int code) {
    if (code >= 0 && code <= WK_UNKNOWN_FILTER) return k_errs[code];
    switch (code) {
    case WK_ERR_CUDA: return "CUDA runtime error";
    case WK_ERR_BAD_ARG: return "bad argument";
    case WK_ERR_RBUF_OVERFLOW: return "result buffer overflow (raise rbuf_bytes / global_gpu_rbuf_size_mb)";
    case WK_ERR_NO_SEGMENT: return "no such (pid, dir) segment in the store";
    case WK_ERR_NO_DEVICE: return "no CUDA device";
    case WK_ERR_COMM: return "communicator not initialised";
    case WK_ERR_STORE_FULL: return "store build: header, ext extent or entry region too small (or a key with >= 2^28 edges)";
    default: return "unknown status";
    }
}

int wk_version(void) { return 100; }

int wk_device_count(int *count) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (count) *count = (e == cudaSuccess) ? n : 0;
    return (e == cudaSuccess && n > 0) ? WK_SUCCESS : WK_ERR_NO_DEVICE;
}

static int store_set_segs(wk_store *st, const wk_segmeta_t *segs, int nsegs) {
    for (int i = 0; i < nsegs; i++) {
        if (segs[i].num_buckets >= (1ull << 32)) return WK_ERR_BAD_ARG;
        if (segs[i].num_buckets && segs[i].bucket_start + segs[i].num_buckets > st->num_slots / WK_ASSOCIATIVITY) return WK_ERR_BAD_ARG;
        st->segs[SegKey(segs[i].index, segs[i].pid, segs[i].dir)] = segs[i];
    }
    return WK_SUCCESS;
}

// device copy of {bucket_start, % num_buckets} per segment, addressed by slot: requests to the resident light-query server
// name segments by slot instead of carrying 32 bytes of modulo magic per step (the device must be current)
static int store_upload_segtab(wk_store *st) {
    std::vector<SegLite> tab;
    st->seg_slot.clear();
    for (auto &kv : st->segs) {
        SegLite sl;
        sl.bucket_start = kv.second.bucket_start;
        sl.fm = make_fastmod(kv.second.num_buckets);
        st->seg_slot[kv.first] = (int)tab.size();
        tab.push_back(sl);
    }
    st->nsegslots = (int)tab.size();
    if (st->d_segtab) { cudaFree(st->d_segtab); st->d_segtab = nullptr; }
    if (tab.empty()) return WK_SUCCESS;
    CUDA_TRY(cudaMalloc((void **)&st->d_segtab, tab.size() * sizeof(SegLite)));
    CUDA_TRY(cudaMemcpy(st->d_segtab, tab.data(), tab.size() * sizeof(SegLite), cudaMemcpyHostToDevice));
    return WK_SUCCESS;
}

// one pass over the header: largest edge list per (index, pid, dir)
static int store_scan_degrees(wk_store *st) {
    const uint32_t P = 1u << WK_NBITS_IDX;   // pid field of a key: predicate / type id (2 MB of counters)
    uint32_t *d_tab = nullptr;
    CUDA_TRY(cudaMalloc((void **)&d_tab, 4ull * P * sizeof(uint32_t)));
    CUDA_TRY(cudaMemset(d_tab, 0, 4ull * P * sizeof(uint32_t)));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, st->device));
    seg_maxdeg_kernel<<<prop.multiProcessorCount * 8, CTA_THREADS>>>(st->d_vertices, st->num_slots, P, d_tab);
    std::vector<uint32_t> tab(4ull * P);
    cudaError_t err = cudaMemcpy(tab.data(), d_tab, tab.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    cudaFree(d_tab);
    if (err != cudaSuccess) return WK_ERR_CUDA;
    for (auto &kv : st->segs) {
        const wk_segmeta_t &m = kv.second;
        uint32_t mx = 0;
        if (m.index == 0) {
            if (m.pid < P) mx = tab[(0 * 2 + (uint32_t)m.dir) * P + m.pid];
        } else {
            for (uint32_t p = 0; p < P; p++) mx = std::max(mx, tab[(1 * 2 + (uint32_t)m.dir) * P + p]);
        }
        st->maxdeg[kv.first] = mx;
    }
    return WK_SUCCESS;
}

// error paths of the create functions must not leak the half-built object
#define STORE_TRY(x)                                                                                  \
    do {                                                                                              \
        cudaError_t _e = (x);                                                                         \
        if (_e != cudaSuccess) {                                                                      \
            fprintf(stderr, "[wukong_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
                    cudaGetErrorString(_e));                                                          \
            wk_store_destroy(st);                                                                     \
            return WK_ERR_CUDA;                                                                       \
        }                                                                                             \
    } while (0)

int wk_store_create(int device, const wk_vertex_t *vertices, uint64_t num_slots, const wk_sid_t *edges,
                    uint64_t num_edges, const wk_segmeta_t *segs, int nsegs, wk_store_t **out) {
    if (!vertices || !segs || !out || num_slots == 0 || (num_slots % WK_ASSOCIATIVITY) != 0) return WK_ERR_BAD_ARG;
    if (num_slots / WK_ASSOCIATIVITY >= (1ull << 32)) return WK_ERR_BAD_ARG;   // bucket ids are 32-bit on the device
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return WK_ERR_NO_DEVICE;
    CUDA_TRY(cudaSetDevice(device));
    wk_store *st = new wk_store();
    st->device = device;
    st->num_slots = num_slots;
    st->num_edges = num_edges;
    int rc = store_set_segs(st, segs, nsegs);
    if (rc) { delete st; return rc; }
    STORE_TRY(cudaMalloc((void **)&st->d_vertices, num_slots * sizeof(uint4)));
    STORE_TRY(cudaMalloc((void **)&st->d_edges, (num_edges ? num_edges : 1) * sizeof(uint32_t)));
    STORE_TRY(cudaMemcpy(st->d_vertices, vertices, num_slots * sizeof(uint4), cudaMemcpyHostToDevice));
    if (num_edges) STORE_TRY(cudaMemcpy(st->d_edges, edges, num_edges * sizeof(uint32_t), cudaMemcpyHostToDevice));
    rc = store_scan_degrees(st);
    if (!rc) rc = store_upload_segtab(st);
    if (rc) { wk_store_destroy(st); return rc; }
    *out = st;
    return WK_SUCCESS;
}

int wk_store_adopt(int device, wk_vertex_t *d_vertices, uint64_t num_slots, wk_sid_t *d_edges, uint64_t num_edges,
                   const wk_segmeta_t *segs, int nsegs, int take_ownership, wk_store_t **out) {
    if (!d_vertices || !segs || !out || num_slots == 0 || (num_slots % WK_ASSOCIATIVITY) != 0) return WK_ERR_BAD_ARG;
    if (num_slots / WK_ASSOCIATIVITY >= (1ull << 32)) return WK_ERR_BAD_ARG;
    wk_store *st = new wk_store();
    st->device = device;
    st->num_slots = num_slots;
    st->num_edges = num_edges;
    st->d_vertices = (uint4 *)d_vertices;
    st->d_edges = d_edges;
    st->owns = false;   // until the adoption has succeeded the arrays stay the caller's
    int rc = store_set_segs(st, segs, nsegs);
    if (rc) { delete st; return rc; }
    if (cudaSetDevice(device) != cudaSuccess) { delete st; return WK_ERR_CUDA; }
    rc = store_scan_degrees(st);
    if (!rc) rc = store_upload_segtab(st);
    if (rc) { wk_store_destroy(st); return rc; }
    st->owns = take_ownership != 0;
    *out = st;
    return WK_SUCCESS;
}

int wk_store_info(wk_store_t *st, uint64_t *num_slots, uint64_t *num_edges, int *nsegs) {
    if (!st) return WK_ERR_BAD_ARG;
    if (num_slots) *num_slots = st->num_slots;
    if (num_edges) *num_edges = st->num_edges;
    if (nsegs) *nsegs = (int)st->segs.size();
    return WK_SUCCESS;
}

int wk_store_segs(wk_store_t *st, wk_segmeta_t *dst, int cap) {
    if (!st || !dst || cap < (int)st->segs.size()) return WK_ERR_BAD_ARG;
    // ordered like segid_t::operator< (pid, index, dir), the order of GStore::rdf_seg_meta_map
    std::vector<wk_segmeta_t> v;
    for (auto &kv : st->segs) v.push_back(kv.second);
    std::sort(v.begin(), v.end(), [](const wk_segmeta_t &a, const wk_segmeta_t &b) {
        return std::make_tuple(a.pid, a.index, a.dir) < std::make_tuple(b.pid, b.index, b.dir);
    });
    memcpy(dst, v.data(), v.size() * sizeof(wk_segmeta_t));
    return WK_SUCCESS;
}

int wk_store_download(wk_store_t *st, wk_vertex_t *vertices, uint64_t num_slots, wk_sid_t *edges, uint64_t num_edges) {
    if (!st || (vertices && num_slots != st->num_slots) || (edges && num_edges != st->num_edges)) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(st->device));
    if (vertices) CUDA_TRY(cudaMemcpy(vertices, st->d_vertices, num_slots * sizeof(wk_vertex_t), cudaMemcpyDeviceToHost));
    if (edges) CUDA_TRY(cudaMemcpy(edges, st->d_edges, num_edges * sizeof(wk_sid_t), cudaMemcpyDeviceToHost));
    return WK_SUCCESS;
}

int wk_store_destroy(wk_store_t *st) {
    if (!st) return WK_ERR_BAD_ARG;
    cudaSetDevice(st->device);
    if (st->owns) {
        if (st->d_vertices) cudaFree(st->d_vertices);
        if (st->d_edges) cudaFree(st->d_edges);
    }
    if (st->d_segtab) cudaFree(st->d_segtab);
    delete st;
    return WK_SUCCESS;
}

int wk_store_get_edges(wk_store_t *st, wk_sid_t vid, wk_sid_t pid, int dir, wk_sid_t *dst, uint64_t cap, uint64_t *size) {
    if (!st || !size) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(st->device));
    const wk_segmeta_t *m = seg_of_key(st, vid, pid, dir);
    if (!m) return WK_ERR_NO_SEGMENT;
    const uint64_t key = make_key(vid, pid, (uint32_t)dir);
    uint64_t bucket = m->bucket_start + hash_u64(key) % m->num_buckets;
    *size = 0;
    while (true) {
        wk_vertex_t b[WK_ASSOCIATIVITY];
        CUDA_TRY(cudaMemcpy(b, st->d_vertices + bucket * WK_ASSOCIATIVITY, sizeof(b), cudaMemcpyDeviceToHost));
        for (int i = 0; i < WK_ASSOCIATIVITY - 1; i++) {
            if (b[i].key == key) {
                const uint64_t sz = ptr_size(b[i].ptr), off = ptr_off(b[i].ptr);
                *size = sz;
                if (dst && sz <= cap && sz) CUDA_TRY(cudaMemcpy(dst, st->d_edges + off, sz * sizeof(uint32_t), cudaMemcpyDeviceToHost));
                return WK_SUCCESS;
            }
        }
        if (b[WK_ASSOCIATIVITY - 1].key == 0) return WK_SUCCESS;
        bucket = b[WK_ASSOCIATIVITY - 1].key >> WK_KEY_VID_SHIFT;
        if (bucket >= st->num_slots / WK_ASSOCIATIVITY) return WK_ERR_BAD_ARG;
    }
}

// release everything an engine owns (also the error path of wk_engine_create: nothing half-built is leaked)
static void engine_free(wk_engine *e) {
    cudaSetDevice(e->store->device);
    srv_stop(e);
    if (e->stream) cudaStreamSynchronize(e->stream);
    comm_free(e);
    for (auto ev : e->event_pool) cudaEventDestroy(ev);
    if (e->d_flush) cudaFree(e->d_flush);
    if (e->q_ev0) cudaEventDestroy(e->q_ev0);
    if (e->q_ev1) cudaEventDestroy(e->q_ev1);
    if (e->buf[0]) cudaFree(e->buf[0]);
    if (e->buf[1]) cudaFree(e->buf[1]);
    if (e->d_ctl) cudaFree(e->d_ctl);
    if (e->d_hq) cudaFree(e->d_hq);
    if (e->d_set) cudaFree(e->d_set);
    if (e->d_setctl) cudaFree(e->d_setctl);
    if (e->d_trace) cudaFree(e->d_trace);
    if (e->d_bplans) cudaFree(e->d_bplans);
    if (e->d_bres) cudaFree(e->d_bres);
    if (e->h_bplans) cudaFreeHost(e->h_bplans);
    if (e->h_bres) cudaFreeHost(e->h_bres);
    if (e->h_rec) cudaFreeHost((void *)e->h_rec);
    if (e->h_stage) cudaFreeHost((void *)e->h_stage);
    if (e->srv.h_box) cudaFreeHost((void *)e->srv.h_box);
    if (e->srv.stream) cudaStreamDestroy(e->srv.stream);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

#define ENGINE_TRY(x)                                                                                 \
    do {                                                                                              \
        cudaError_t _e = (x);                                                                         \
        if (_e != cudaSuccess) {                                                                      \
            fprintf(stderr, "[wukong_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
                    cudaGetErrorString(_e));                                                          \
            engine_free(e);                                                                           \
            return WK_ERR_CUDA;                                                                       \
        }                                                                                             \
    } while (0)

int wk_engine_create(wk_store_t *store, uint64_t rbuf_bytes, wk_engine_t **out) {
    if (!store || !out || rbuf_bytes < 4096) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(store->device));
    wk_engine *e = new wk_engine();
    e->store = store;
    e->cap_words = rbuf_bytes / sizeof(uint32_t);
    ENGINE_TRY(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    ENGINE_TRY(cudaMalloc((void **)&e->buf[0], e->cap_words * sizeof(uint32_t)));
    ENGINE_TRY(cudaMalloc((void **)&e->buf[1], e->cap_words * sizeof(uint32_t)));
    ENGINE_TRY(cudaMalloc((void **)&e->d_ctl, sizeof(CtlBlock)));
    // one descriptor (4 KB) per 256-row tile that may turn out heavy: sized for 64 M-row frontiers at most
    e->hq_cap = (uint32_t)std::min<uint64_t>(262144, std::max<uint64_t>(8192, e->cap_words / 16384));
    ENGINE_TRY(cudaMalloc((void **)&e->d_hq, (size_t)e->hq_cap * sizeof(HeavyTile)));
    ENGINE_TRY(cudaHostAlloc((void **)&e->h_rec, sizeof(HostRec), cudaHostAllocMapped));
    memset((void *)e->h_rec, 0, sizeof(HostRec));
    ENGINE_TRY(cudaHostGetDevicePointer((void **)&e->d_rec, (void *)e->h_rec, 0));
    e->stage_words = (1u << 20) / sizeof(uint32_t);   // 1 MiB zero-copy staging for small results
    ENGINE_TRY(cudaHostAlloc((void **)&e->h_stage, e->stage_words * sizeof(uint32_t), cudaHostAllocMapped));
    ENGINE_TRY(cudaHostGetDevicePointer((void **)&e->d_stage, (void *)e->h_stage, 0));
    cudaDeviceProp prop;
    ENGINE_TRY(cudaGetDeviceProperties(&prop, store->device));
    e->num_sms = prop.multiProcessorCount;
    // resident CTAs per SM of each fused kernel (persistent grid = SMs x occupancy)
    e->variant = WK_DEFAULT_VARIANT;
    if (const char *ev = getenv("WK_VARIANT")) {
        const int v = atoi(ev);
        if (v >= 0 && v < WK_NUM_VARIANTS) e->variant = v;
    }
    for (int m = 0; m < 3; m++) {
        StepKernelFn fn = step_kernel_fn(m, e->variant, 3);
        const size_t smem = step_smem(e, 3);
        if (smem > 40 * 1024) ENGINE_TRY(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ENGINE_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&e->occ[m], fn, CTA_THREADS, smem));
    }
    if (getenv("WK_VERBOSE"))
        fprintf(stderr, "[wukong_b200] variant %d: CTAs/SM k2u=%d k2k=%d k2c=%d, %d SMs\n", e->variant, e->occ[0], e->occ[1], e->occ[2], e->num_sms);
    for (int i = 0; i < 3; i++)
        if (e->occ[i] < 1) e->occ[i] = 1;
    // resident light-query server: on unless WK_RESIDENT=0 (profilers and sanitizers serialise kernels; see wk_server.cuh)
    if (const char *ev = getenv("WK_RESIDENT")) e->srv.enabled = atoi(ev) != 0;
    if (const char *ev = getenv("WK_FUSE_FILTERS")) e->fuse_filters = atoi(ev) != 0;
    if (const char *ev = getenv("WK_SEED_BULK")) e->seed_bulk = atoi(ev) != 0;
    if (const char *ev = getenv("WK_PDL")) g_use_pdl = atoi(ev) != 0;
    if (const char *ev = getenv("WK_DIRECT_OUT")) e->direct_out = atoi(ev) != 0;
    if (const char *ev = getenv("WK_SRV_VARIANT")) e->srv.variant = atoi(ev);
    if (const char *ev = getenv("WK_RESIDENT_IDLE_US")) e->srv.idle_ns = (uint64_t)std::max(1, atoi(ev)) * 1000ull;
    if (reset_ctl(e) != WK_SUCCESS) { engine_free(e); return WK_ERR_CUDA; }
    ENGINE_TRY(cudaStreamSynchronize(e->stream));
    if (preload_kernels(e) != WK_SUCCESS) { engine_free(e); return WK_ERR_CUDA; }
    *out = e;
    return WK_SUCCESS;
}

int wk_engine_destroy(wk_engine_t *e) {
    if (!e) return WK_ERR_BAD_ARG;
    engine_free(e);
    return WK_SUCCESS;
}

int wk_engine_set_profiling(wk_engine_t *e, int on) {
    if (!e) return WK_ERR_BAD_ARG;
    e->profiling = on < 0 ? 0 : on;
    if (e->profiling && !e->q_ev0) {
        CUDA_TRY(cudaSetDevice(e->store->device));
        CUDA_TRY(cudaEventCreate(&e->q_ev0));
        CUDA_TRY(cudaEventCreate(&e->q_ev1));
    }
    return WK_SUCCESS;
}

int wk_engine_set_option(wk_engine_t *e, int option, int64_t value) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    switch (option) {
    case WK_OPT_RESIDENT_LIGHT:
        e->srv.enabled = value != 0;
        if (!e->srv.enabled) srv_stop(e);
        return WK_SUCCESS;
    case WK_OPT_FUSE_FILTERS:
        e->fuse_filters = value != 0;
        return WK_SUCCESS;
    case WK_OPT_RESIDENT_VARIANT:
        if (value < 0 || value > 3) return WK_ERR_BAD_ARG;
        srv_stop(e);
        e->srv.variant = (int)value;
        return WK_SUCCESS;
    case WK_OPT_DIRECT_OUT:
        e->direct_out = value != 0;
        return WK_SUCCESS;
    case WK_OPT_RESIDENT_IDLE_US:
        if (value < 1 || value > 10 * 1000 * 1000) return WK_ERR_BAD_ARG;
        srv_stop(e);   // the next instance picks the new value up
        e->srv.idle_ns = (uint64_t)value * 1000ull;
        return WK_SUCCESS;
    default: return WK_ERR_BAD_ARG;
    }
}

int wk_engine_get_option(wk_engine_t *e, int option, int64_t *value) {
    if (!e || !value) return WK_ERR_BAD_ARG;
    switch (option) {
    case WK_OPT_RESIDENT_LIGHT: *value = e->srv.enabled ? 1 : 0; return WK_SUCCESS;
    case WK_OPT_RESIDENT_IDLE_US: *value = (int64_t)(e->srv.idle_ns / 1000ull); return WK_SUCCESS;
    case WK_OPT_FUSE_FILTERS: *value = e->fuse_filters ? 1 : 0; return WK_SUCCESS;
    case WK_OPT_DIRECT_OUT: *value = e->direct_out ? 1 : 0; return WK_SUCCESS;
    case WK_INFO_RESIDENT_LAUNCHES: *value = (int64_t)e->srv.launches; return WK_SUCCESS;
    case WK_INFO_RESIDENT_REQUESTS: *value = (int64_t)e->srv.requests; return WK_SUCCESS;
    case WK_INFO_LAST_RESIDENT: *value = e->last_resident ? 1 : 0; return WK_SUCCESS;
    case WK_INFO_LAST_RESIDENT_NS: *value = (int64_t)e->srv.last_ns; return WK_SUCCESS;
    case WK_INFO_COMM_BYTES_PUSHED: {
        if (!e->comm) return WK_ERR_COMM;
        int rc = wk_comm_stats(e, nullptr, nullptr, nullptr);
        if (rc) return rc;
        *value = (int64_t)comm_bytes_pushed(e);
        return WK_SUCCESS;
    }
    case WK_INFO_RESIDENT_RUNNING: *value = (e->srv.h_box && !e->srv.quitting && !srv_exited(e)) ? 1 : 0; return WK_SUCCESS;
    default: return WK_ERR_BAD_ARG;
    }
}

int wk_engine_sync(wk_engine_t *e) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return WK_SUCCESS;
}

int wk_engine_reset(wk_engine_t *e) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    e->ncols = 0;
    return reset_ctl(e);
}

int wk_table_upload(wk_engine_t *e, const wk_sid_t *table, uint64_t nrows, int ncols) {
    if (!e || ncols < 0 || ncols >= MAX_COLS || (nrows && ncols && !table)) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (nrows * (uint64_t)ncols > e->cap_words) return WK_ERR_RBUF_OVERFLOW;
    int rc = reset_ctl(e);
    if (rc) return rc;
    e->ncols = ncols;
    if (nrows && ncols) {
        CUDA_TRY(cudaMemcpyAsync(e->buf[0], table, nrows * (uint64_t)ncols * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
        set_count_kernel<<<1, 1, 0, e->stream>>>(&e->d_ctl->counts[0], nrows);
        CUDA_TRY(cudaGetLastError());
        e->launches++;
    }
    return WK_SUCCESS;
}

int wk_table_info(wk_engine_t *e, uint64_t *nrows, int *ncols) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    uint64_t rows = 0;
    int rc = sync_rows(e, &rows);
    if (nrows) *nrows = rows;
    if (ncols) *ncols = e->ncols;
    return rc;
}

int wk_table_download(wk_engine_t *e, wk_sid_t *dst, uint64_t cap_words, uint64_t *nrows, int *ncols) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    uint64_t rows = 0;
    int rc = sync_rows(e, &rows);
    if (nrows) *nrows = rows;
    if (ncols) *ncols = e->ncols;
    if (rc) return rc;
    const uint64_t words = rows * (uint64_t)e->ncols;
    if (words > cap_words) return WK_ERR_BAD_ARG;
    if (words && dst) {
        CUDA_TRY(cudaMemcpyAsync(dst, e->buf[e->step & 1], words * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    return WK_SUCCESS;
}

static int finish_call(wk_engine *e, int rc, uint64_t *out_rows) {
    if (rc) return rc;
    if (out_rows) return sync_rows(e, out_rows);
    return WK_SUCCESS;
}

int wk_index_to_unknown(wk_engine_t *e, wk_sid_t tpid, int dir, int mt_tid, int mt_factor, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_seed(e, KIND_I2U, 0, tpid, dir, mt_tid, mt_factor), out_rows);
}

int wk_const_to_unknown(wk_engine_t *e, wk_sid_t vid, wk_sid_t pid, int dir, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_seed(e, KIND_C2U, vid, pid, dir, 0, 1), out_rows);
}

int wk_known_to_unknown(wk_engine_t *e, int col_start, wk_sid_t pid, int dir, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_known(e, KIND_K2U, col_start, pid, dir, 0, 0), out_rows);
}

int wk_known_to_known(wk_engine_t *e, int col_start, wk_sid_t pid, int dir, int col_end, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_known(e, KIND_K2K, col_start, pid, dir, col_end, 0), out_rows);
}

int wk_known_to_const(wk_engine_t *e, int col_start, wk_sid_t pid, int dir, wk_sid_t end_const, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_known(e, KIND_K2C, col_start, pid, dir, 0, end_const), out_rows);
}

int wk_const_to_known(wk_engine_t *e, wk_sid_t vid, wk_sid_t pid, int dir, int col_end, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_to_known(e, KIND_C2K, vid, pid, dir, col_end, 0, 1), out_rows);
}

int wk_index_to_known(wk_engine_t *e, wk_sid_t tpid, int dir, int col_end, int mt_tid, int mt_factor, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_to_known(e, KIND_I2K, 0, tpid, dir, col_end, mt_tid, mt_factor), out_rows);
}

// diagnostics: SM clocks of the fused light kernel's phase boundaries (profiling level 3):
// [0] entry, [1] control block cleared, [2 + s] step s done, [2 + 24] table / projection written, [3 + 24] record stored
int wk_engine_light_trace(wk_engine_t *e, int64_t *dst, int cap) {
    if (!e || !dst || cap < MAX_LIGHT_STEPS + 4) return WK_ERR_BAD_ARG;
    if (!e->d_trace) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    // a blocking copy on the legacy stream does not wait for the resident server (its stream is non-blocking)
    const int n = cap < (int)LIGHT_TRACE_WORDS ? cap : (int)LIGHT_TRACE_WORDS;
    CUDA_TRY(cudaMemcpy(dst, e->d_trace, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost));
    return WK_SUCCESS;
}

int wk_table_distinct(wk_engine_t *e, const int32_t *cols, int n, uint64_t *out_rows) {
    if (!e || !cols) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    uint64_t rows = 0;
    int rc = sync_rows(e, &rows);
    if (rc) return rc;
    return finish_call(e, enqueue_distinct(e, cols, n, rows), out_rows);
}

int wk_table_slice(wk_engine_t *e, uint64_t offset, int64_t limit, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_slice(e, offset, limit, e->cap_words / (uint64_t)std::max(1, e->ncols)), out_rows);
}

int wk_project(wk_engine_t *e, const int32_t *cols, int n, uint64_t *out_rows) {
    if (!e || !cols) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    return finish_call(e, enqueue_project(e, cols, n), out_rows);
}

// ---- whole pattern phase ---------------------------------------------------------------------------
struct PlannedStep {
    int kind;
    int col_start, col_end;
    uint32_t pid, end_const;
    int dir;
    uint64_t vid;   // seeds
    int in_cols;
};

// Resolve each pattern to a primitive exactly like execute_one_pattern (sparql.hpp:938-1061),
// tracking var -> column like Result::add_var2col (query.hpp:378-395).
static int plan_steps(const wk_pattern_t *pats, int npat, int nvars, std::vector<int> &v2c, std::vector<PlannedStep> &steps) {
    const int NO_RESULT = 0xFFFF;
    if (npat <= 0 || nvars <= 0 || nvars > 4096) return npat <= 0 ? WK_SYNTAX_ERROR : WK_ERR_BAD_ARG;
    v2c.assign(nvars, NO_RESULT);
    int ncols = 0;
    auto var2col = [&](int32_t vid, int &col) -> int {
        if (vid >= 0) return WK_VERTEX_INVALID;
        const int idx = -(vid + 1);
        if (idx < 0 || idx >= nvars) return WK_VERTEX_INVALID;
        col = v2c[idx];
        return WK_SUCCESS;
    };
    enum { KNOWN = 0, UNKNOWN = 1, CONST = 2 };
    auto var_stat = [&](int32_t vid, int &st) -> int {
        if (vid >= 0) { st = CONST; return WK_SUCCESS; }
        int col;
        int rc = var2col(vid, col);
        if (rc) return rc;
        st = (col == NO_RESULT) ? UNKNOWN : KNOWN;
        return WK_SUCCESS;
    };
    for (int i = 0; i < npat; i++) {
        const wk_pattern_t &pt = pats[i];
        PlannedStep ps;
        memset(&ps, 0, sizeof(ps));
        ps.dir = pt.direction;
        ps.in_cols = ncols;
        if (pt.direction != WK_DIR_IN && pt.direction != WK_DIR_OUT) return WK_ERR_BAD_ARG;
        if (i == 0 && is_tpid(pt.subject)) {   // start_from_index(), query.hpp:660-682
            if (pt.predicate != WK_PREDICATE_ID && pt.predicate != WK_TYPE_ID) return WK_OBJ_ERROR;
            int col;
            int rc = var2col(pt.object, col);
            if (rc) return rc;
            if (col != NO_RESULT) return WK_UNKNOWN_PATTERN;   // index_to_known: not on the device path
            if (ncols != 0) return WK_FIRST_PATTERN_ERROR;
            ps.kind = KIND_I2U;
            ps.vid = 0;
            ps.pid = (uint32_t)pt.subject;
            v2c[-(pt.object + 1)] = 0;
            ncols = 1;
            steps.push_back(ps);
            continue;
        }
        int sp, ss, so;
        int rc = var_stat(pt.predicate, sp);
        if (rc) return rc;
        if (sp != CONST) return WK_UNKNOWN_PATTERN;   // variable predicates need VERSATILE
        if ((rc = var_stat(pt.subject, ss)) || (rc = var_stat(pt.object, so))) return rc;
        ps.pid = (uint32_t)pt.predicate;
        if (ss == CONST && so == UNKNOWN) {
            if (ncols != 0) return WK_FIRST_PATTERN_ERROR;
            ps.kind = KIND_C2U;
            ps.vid = (uint64_t)pt.subject;
            v2c[-(pt.object + 1)] = ncols;
            ncols += 1;
        } else if (ss == KNOWN && so == CONST) {
            ps.kind = KIND_K2C;
            ps.col_start = v2c[-(pt.subject + 1)];
            ps.end_const = (uint32_t)pt.object;
        } else if (ss == KNOWN && so == KNOWN) {
            ps.kind = KIND_K2K;
            ps.col_start = v2c[-(pt.subject + 1)];
            ps.col_end = v2c[-(pt.object + 1)];
        } else if (ss == KNOWN && so == UNKNOWN) {
            ps.kind = KIND_K2U;
            ps.col_start = v2c[-(pt.subject + 1)];
            v2c[-(pt.object + 1)] = ncols;
            ncols += 1;
        } else if (ss == CONST && so == KNOWN) {
            ps.kind = KIND_C2K;          // const_to_known (sparql.hpp:144-186)
            ps.vid = (uint64_t)pt.subject;
            ps.col_end = v2c[-(pt.object + 1)];
        } else if (ss == UNKNOWN) {
            return WK_UNKNOWN_SUB;
        } else {
            return WK_UNKNOWN_PATTERN;   // CONST/CONST
        }
        if (ncols >= MAX_COLS) return WK_ERR_BAD_ARG;
        steps.push_back(ps);
    }
    return WK_SUCCESS;
}

// translate planned steps into the light interpreter's step descriptors
static int fill_light_steps(wk_engine *e, const std::vector<PlannedStep> &steps, int mt_tid, int mt_factor, LightStep *out) {
    for (size_t i = 0; i < steps.size(); i++) {
        const PlannedStep &ps = steps[i];
        LightStep &ls = out[i];
        memset(&ls, 0, sizeof(ls));
        ls.kind = ps.kind;
        ls.C = ps.in_cols;
        ls.col_start = ps.col_start;
        ls.col_end = ps.col_end;
        ls.end_const = ps.end_const;
        ls.mt_tid = ps.kind == KIND_I2U ? mt_tid : 0;   // only index_to_unknown is sliced (sparql.hpp:211-221)
        ls.mt_factor = (ps.kind != KIND_I2U || mt_factor < 1) ? 1 : mt_factor;
        if (ps.kind == KIND_I2U || ps.kind == KIND_C2U) {
            const wk_segmeta_t *m = seg_of_key(e->store, ps.vid, ps.pid, ps.dir);
            if (!m) return WK_ERR_NO_SEGMENT;
            ls.seg = make_segparam(m, ps.pid, ps.dir, false);
            ls.key = make_key(ps.vid, ps.pid, (uint32_t)ps.dir);
        } else {
            const bool index_mode = (ps.kind == KIND_K2U && ps.pid == WK_TYPE_ID && ps.dir == WK_DIR_IN);
            const wk_segmeta_t *m = index_mode ? find_seg(e->store, 1, WK_PREDICATE_ID, ps.dir) : find_seg(e->store, 0, ps.pid, ps.dir);
            if (!m) return WK_ERR_NO_SEGMENT;
            ls.seg = make_segparam(m, ps.pid, ps.dir, index_mode);
        }
    }
    return WK_SUCCESS;
}

// =============================================================================================
// resident light-query server (wk_server.cuh): host side
// =============================================================================================
static int srv_init(wk_engine *e) {
    if (e->srv.h_box) return WK_SUCCESS;
    if (!e->srv.stream) CUDA_TRY(cudaStreamCreateWithFlags(&e->srv.stream, cudaStreamNonBlocking));
    SrvMailbox *box = nullptr;
    CUDA_TRY(cudaHostAlloc((void **)&box, sizeof(SrvMailbox), cudaHostAllocMapped));
    memset((void *)box, 0, sizeof(SrvMailbox));
    e->srv.h_box = box;
    CUDA_TRY(cudaHostGetDevicePointer((void **)&e->srv.d_box, (void *)box, 0));
    CUDA_TRY(cudaFuncSetAttribute((const void *)light_server_kernel<LIGHT_SRV_THREADS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SrvSmem)));
    CUDA_TRY(cudaFuncSetAttribute((const void *)light_server_kernel<256, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SrvSmem)));
    CUDA_TRY(cudaFuncSetAttribute((const void *)light_server_kernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SrvSmem)));
    CUDA_TRY(cudaFuncSetAttribute((const void *)light_server_kernel<512, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SrvSmem)));
    CUDA_TRY(cudaFuncSetAttribute((const void *)light_server_sharded_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SrvSmemSharded)));
    if (!e->d_trace) {
        CUDA_TRY(cudaMalloc((void **)&e->d_trace, LIGHT_TRACE_WORDS * sizeof(long long)));
        CUDA_TRY(cudaMemset(e->d_trace, 0, LIGHT_TRACE_WORDS * sizeof(long long)));
    }
    return WK_SUCCESS;
}

// no server instance is (or will stay) on the device: never launched, or the last instance has stored its exit word
static bool srv_exited(const wk_engine *e) {
    if (e->srv.launch_id == 0) return true;
    return *(const volatile uint64_t *)&e->srv.h_box->exit_word == e->srv.launch_id;
}

static int srv_launch(wk_engine *e, uint64_t first_seq, bool sharded = false) {
    SrvParams P;
    memset(&P, 0, sizeof(P));
    P.vertices = e->store->d_vertices;
    P.edges = e->store->d_edges;
    P.segtab = e->store->d_segtab;
    P.nsegs = e->store->nsegslots;
    P.ctl_nwords = (int)(sizeof(CtlBlock) / sizeof(uint64_t));
    P.req = e->srv.d_box->req;
    P.rec = &e->srv.d_box->rec;
    P.times = e->srv.d_box->times;
    P.exit_word = &e->srv.d_box->exit_word;
    P.host_table = e->d_stage;
    P.host_table_words = e->stage_words;
    P.buf[0] = e->buf[0];
    P.buf[1] = e->buf[1];
    P.cap_words = e->cap_words;
    P.counts = e->d_ctl->counts;
    P.stats = e->d_ctl->stats;
    P.ctl_words = (uint64_t *)e->d_ctl;
    P.status = &e->d_ctl->status;
    P.first_seq = first_seq;
    P.launch_id = ++e->srv.launch_id;
    P.idle_ns = e->srv.idle_ns;
    P.trace = e->d_trace;
    if (sharded) {
        SrvPeers Q;
        int rc = srv_fill_peers(e, Q);
        if (rc) return rc;
        light_server_sharded_kernel<<<1, LIGHT_SRV_THREADS, sizeof(SrvSmemSharded), e->srv.stream>>>(P, Q);
    } else switch (e->srv.variant) {   // WK_SRV_VARIANT, for A/B runs: threads of the server CTA x warp mode of the interpreter
    case 1: light_server_kernel<256, true><<<1, 256, sizeof(SrvSmem), e->srv.stream>>>(P); break;
    case 2: light_server_kernel<256, false><<<1, 256, sizeof(SrvSmem), e->srv.stream>>>(P); break;
    case 3: light_server_kernel<512, true><<<1, 512, sizeof(SrvSmem), e->srv.stream>>>(P); break;
    default: light_server_kernel<LIGHT_SRV_THREADS, true><<<1, LIGHT_SRV_THREADS, sizeof(SrvSmem), e->srv.stream>>>(P); break;
    }
    CUDA_TRY(cudaGetLastError());
    e->launches++;
    e->srv.launches++;
    e->srv.quitting = false;
    e->srv.sharded = sharded;
    return WK_SUCCESS;
}

// wait until the current instance has left (it was told to, or it is idling out)
static int srv_wait_exit(wk_engine *e) {
    uint32_t spins = 0;
    while (!srv_exited(e)) {
        if ((++spins & 0x3FFF) == 0) {
            cudaError_t q = cudaStreamQuery(e->srv.stream);
            if (q == cudaSuccess) break;              // the kernel is gone (its exit word may still be in flight)
            if (q != cudaErrorNotReady) CUDA_TRY(q);
        }
    }
    return WK_SUCCESS;
}

static int srv_ensure_running(wk_engine *e, uint64_t first_seq, bool sharded = false) {
    int rc = srv_init(e);
    if (rc) return rc;
    if (!e->srv.quitting && !srv_exited(e) && e->srv.sharded != sharded) {
        // the other kind of server is resident (a plain query on an engine of a sharded group, or the reverse): swap.
        // The QUIT takes a sequence number; the caller's first_seq was computed before it.
        srv_park(e);
        first_seq = e->srv.seq + 1;
    }
    if (e->srv.quitting) {
        rc = srv_wait_exit(e);
        if (rc) return rc;
        e->srv.quitting = false;
        return srv_launch(e, first_seq, sharded);
    }
    if (srv_exited(e)) return srv_launch(e, first_seq, sharded);
    return WK_SUCCESS;
}

static void srv_post(wk_engine *e, const SrvChunk *ch, uint64_t seq) {
    volatile SrvChunk *q = e->srv.h_box->req;
    for (int i = 0; i < SRV_CHUNKS; i++) { q[i].w0 = ch[i].w0; q[i].w1 = ch[i].w1; q[i].w2 = ch[i].w2; }
    __atomic_thread_fence(__ATOMIC_RELEASE);   // payload words before the tags (a compiler barrier on x86)
    for (int i = 0; i < SRV_CHUNKS; i++) q[i].tag = (uint32_t)seq;
    __atomic_thread_fence(__ATOMIC_SEQ_CST);
}

// The server occupies one CTA slot of one SM.  The fused step kernels are persistent grids that fill every slot and stride
// statically over their tiles, so a CTA that cannot become resident would run after all the others: ask the server to
// leave before such a kernel is launched.  It is relaunched when the heavy query is over (wk_query_execute) or on demand.
static void srv_park(wk_engine *e) {
    if (!e->srv.h_box || e->srv.launch_id == 0 || e->srv.quitting || srv_exited(e)) return;
    SrvChunk ch[SRV_CHUNKS];
    memset(ch, 0, sizeof(ch));
    ch[0].w0 = (uint32_t)SRV_F_QUIT << 8;
    srv_post(e, ch, ++e->srv.seq);
    e->srv.quitting = true;
}

static void srv_stop(wk_engine *e) {
    if (!e->srv.h_box) return;
    srv_park(e);
    srv_wait_exit(e);
    e->srv.quitting = false;
    if (e->srv.stream) cudaStreamSynchronize(e->srv.stream);
}

static bool srv_usable(const wk_engine *e) {
    return e->srv.enabled && e->store->nsegslots > 0 && e->store->nsegslots < (1 << 15) && e->store->d_segtab;
}

// post one request to the (right kind of) server and wait for its record; an instance that idled out is replaced
static int srv_roundtrip(wk_engine *e, const SrvChunk *ch, int nsteps, int table_cols, bool sharded, RecView &rv) {
    int rc = srv_ensure_running(e, e->srv.seq + 1, sharded);
    if (rc) return rc;
    const uint64_t seq = ++e->srv.seq;
    srv_post(e, ch, seq);
    e->srv.requests++;
    const volatile uint64_t *rec = (const volatile uint64_t *)&e->srv.h_box->rec;
    uint32_t spins = 0;
    while (!record_valid_at(rec, e, seq, nsteps, table_cols, rv)) {
        if ((++spins & 0xFFF) != 0) continue;
        if (srv_exited(e)) {
            // the instance idled out (or was leaving) without seeing this request: a new one picks it up
            if (record_valid_at(rec, e, seq, nsteps, table_cols, rv)) break;
            rc = srv_launch(e, seq, sharded);
            if (rc) return rc;
        } else if ((spins & 0xFFFFF) == 0) {
            cudaError_t q = cudaStreamQuery(e->srv.stream);
            if (q == cudaSuccess) {   // the kernel is gone although its exit word never showed up
                if (record_valid_at(rec, e, seq, nsteps, table_cols, rv)) break;
                rc = srv_launch(e, seq, sharded);
                if (rc) return rc;
            } else if (q != cudaErrorNotReady) {
                CUDA_TRY(q);
            }
        }
    }
    const volatile uint64_t *t = (const volatile uint64_t *)e->srv.h_box->times;
    const uint64_t t0 = t[0], t1 = t[1];
    e->srv.last_ns = t1 >= t0 ? t1 - t0 : 0;
    return WK_SUCCESS;
}

// epoch != 0: this engine is one shard of a group and owns the query's constant (in-place execution over peer memory)
static int run_light_resident(wk_engine *e, const std::vector<PlannedStep> &steps, bool project,
                              const std::vector<int32_t> &proj_cols, RecView &rv, uint64_t epoch = 0) {
    SrvChunk ch[SRV_CHUNKS];
    memset(ch, 0, sizeof(ch));
    const uint32_t flags = (project ? SRV_F_PROJECT : 0u) | (e->profiling >= 2 ? SRV_F_STATS : 0u) | (e->profiling >= 3 ? SRV_F_TRACE : 0u);
    ch[0].w0 = (uint32_t)steps.size() | (flags << 8) | ((uint32_t)proj_cols.size() << 16);
    for (size_t j = 0; j < proj_cols.size(); j++) {
        SrvChunk &c = ch[1 + j / 12];
        uint32_t &w = (j % 12) < 4 ? c.w0 : ((j % 12) < 8 ? c.w1 : c.w2);
        w |= ((uint32_t)proj_cols[j] & 0xFFu) << (8 * (j & 3));
    }
    for (size_t i = 0; i < steps.size(); i++) {
        const PlannedStep &ps = steps[i];
        const bool seed = ps.kind == KIND_I2U || ps.kind == KIND_C2U;
        const bool index_mode = !seed && ps.kind == KIND_K2U && ps.pid == WK_TYPE_ID && ps.dir == WK_DIR_IN;
        const wk_segmeta_t *m = seed ? seg_of_key(e->store, ps.vid, ps.pid, ps.dir)
                                     : (index_mode ? find_seg(e->store, 1, WK_PREDICATE_ID, ps.dir) : find_seg(e->store, 0, ps.pid, ps.dir));
        if (!m) return WK_ERR_NO_SEGMENT;
        const int slot = e->store->seg_slot[SegKey(m->index, m->pid, m->dir)];
        SrvChunk &c = ch[SRV_HDR_CHUNKS + i];
        c.w0 = srv_pack_w0(ps.kind, ps.col_start, ps.col_end, ps.dir, index_mode ? 1 : 0, ps.in_cols);
        c.w1 = seed ? (uint32_t)ps.vid : ps.end_const;
        c.w2 = (ps.pid & 0x1FFFFu) | ((uint32_t)slot << 17);
    }
    ch[0].w1 = (uint32_t)epoch;
    ch[0].w2 = (uint32_t)(epoch >> 32);
    int rc = srv_roundtrip(e, ch, (int)steps.size(), project ? (int)proj_cols.size() : 0, epoch != 0, rv);
    if (rc) return rc;
    for (int i = 0; i < rv.resume && i < (int)steps.size(); i++) {
        e->recs.emplace_back();
        StepRecord &r = e->recs.back();
        r.kind = steps[i].kind;
        r.in_cols = steps[i].in_cols;
        r.s = i;
        r.launches = 0;
    }
    return WK_SUCCESS;
}

static int run_light(wk_engine *e, const std::vector<PlannedStep> &steps, int mt_tid, int mt_factor, bool project,
                     const std::vector<int32_t> &proj_cols, RecView &rv) {
    LightPlan lp;
    memset(&lp, 0, sizeof(lp));
    lp.vertices = e->store->d_vertices;
    lp.edges = e->store->d_edges;
    lp.buf[0] = e->buf[0];
    lp.buf[1] = e->buf[1];
    lp.counts = e->d_ctl->counts;
    lp.stats = e->d_ctl->stats;
    lp.status = &e->d_ctl->status;
    lp.ctl_words = (uint64_t *)e->d_ctl;
    lp.ctl_nwords = (int)(sizeof(CtlBlock) / sizeof(uint64_t));
    lp.rec = e->d_rec;
    lp.host_table = e->d_stage;
    lp.host_table_words = e->stage_words;
    lp.cap_words = e->cap_words;
    lp.nsteps = (int)steps.size();
    lp.do_project = project ? 1 : 0;
    lp.collect_stats = e->profiling >= 2 ? 1 : 0;
    lp.proj_n = (int)proj_cols.size();
    for (size_t i = 0; i < proj_cols.size(); i++) lp.proj_cols[i] = (int8_t)proj_cols[i];
    int frc = fill_light_steps(e, steps, mt_tid, mt_factor, lp.steps);
    if (frc) return frc;
    lp.seq = ++e->seq;
    if (e->profiling >= 3) {
        if (!e->d_trace) CUDA_TRY(cudaMalloc((void **)&e->d_trace, LIGHT_TRACE_WORDS * sizeof(long long)));
        CUDA_TRY(cudaMemsetAsync(e->d_trace, 0, LIGHT_TRACE_WORDS * sizeof(long long), e->stream));
        lp.trace = e->d_trace;
    }
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (e->profiling >= 2) { ev0 = get_event(e); ev1 = get_event(e); if (ev0) cudaEventRecord(ev0, e->stream); }
    light_query_kernel<<<1, LIGHT_THREADS, 0, e->stream>>>(lp);
    CUDA_TRY(cudaGetLastError());
    if (ev0 && ev1) cudaEventRecord(ev1, e->stream);
    if (e->profiling) { cudaEventRecord(e->q_ev1, e->stream); e->q_timed = true; }
    e->launches++;
    int rc = wait_record(e, lp.seq, (int)steps.size(), project ? (int)proj_cols.size() : 0, rv);
    if (rc) return rc;
    // one record per step the fused kernel actually ran; the single launch (and its event time)
    // is attributed to the first of them
    for (int i = 0; i < rv.resume && i < (int)steps.size(); i++) {
        e->recs.emplace_back();
        StepRecord &r = e->recs.back();
        r.kind = steps[i].kind;
        r.in_cols = steps[i].in_cols;
        r.s = i;
        r.launches = (i == 0) ? 1 : 0;
        if (i == 0 && ev0 && ev1) { r.ev0 = ev0; r.ev1 = ev1; r.timed = true; }
    }
    return WK_SUCCESS;
}

// steps[i..j) are consecutive known_to_known / known_to_const filters on bound columns: one launch
static int enqueue_filter_chain(wk_engine *e, const std::vector<PlannedStep> &steps, size_t i, size_t j, const DirectOut *direct) {
    std::vector<size_t> order;
    for (size_t k = i; k < j; k++) if (steps[k].kind == KIND_K2K) order.push_back(k);
    for (size_t k = i; k < j; k++) if (steps[k].kind == KIND_K2C) order.push_back(k);
    ChainFilter ex[MAX_CHAIN];
    for (size_t k = 1; k < order.size(); k++) {
        const PlannedStep &x = steps[order[k]];
        ex[k - 1] = ChainFilter{x.kind, x.col_start, x.col_end, x.dir, x.pid, x.end_const};
    }
    const PlannedStep &p0 = steps[order[0]];
    return enqueue_known(e, p0.kind, p0.col_start, p0.pid, p0.dir, p0.col_end, p0.end_const, ex, (int)order.size() - 1, direct);
}

int wk_query_execute(wk_engine_t *e, const wk_pattern_t *patterns, int npatterns, int nvars,
                     const int32_t *required_vars, int nrequired, int mt_tid, int mt_factor, int blind,
                     wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols) {
    wk_query_opts_t o;
    memset(&o, 0, sizeof(o));
    o.mt_tid = mt_tid;
    o.mt_factor = mt_factor;
    o.blind = blind;
    o.limit = -1;
    return wk_query_execute_ex(e, patterns, npatterns, nvars, required_vars, nrequired, &o, table, cap_words, out_rows, out_cols);
}

int wk_query_execute_ex(wk_engine_t *e, const wk_pattern_t *patterns, int npatterns, int nvars,
                        const int32_t *required_vars, int nrequired, const wk_query_opts_t *opts,
                        wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols) {
    if (!e || !patterns || !opts) return WK_ERR_BAD_ARG;
    const int mt_tid = opts->mt_tid, mt_factor = opts->mt_factor, blind = opts->blind;
    // DISTINCT / OFFSET / LIMIT are part of final_process, which a blind query skips (sparql.hpp:1425-1426)
    const bool post = !blind && (opts->distinct || opts->offset > 0 || opts->limit >= 0);
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (out_rows) *out_rows = 0;
    if (out_cols) *out_cols = 0;
    std::vector<int> v2c;
    std::vector<PlannedStep> steps;
    int rc = plan_steps(patterns, npatterns, nvars, v2c, steps);
    if (rc) return rc;
    if ((int)steps.size() > MAX_STEPS - 2) return WK_ERR_BAD_ARG;
    const int final_cols = steps.back().in_cols + ((steps.back().kind == KIND_K2K || steps.back().kind == KIND_K2C) ? 0 : 1);
    // projection columns (final_process, sparql.hpp:1507-1550)
    std::vector<int32_t> proj_cols;
    // final_process raises NO_REQUIRED_VAR only when there is a non-empty table to project
    // (sparql.hpp:1425-1426, 1511): run the pattern phase first and report afterwards
    const bool no_required = !blind && (nrequired <= 0 || !required_vars);
    const bool want_table = !blind && !no_required;
    if (want_table) {
        for (int i = 0; i < nrequired; i++) {
            const int idx = -(required_vars[i] + 1);
            if (required_vars[i] >= 0 || idx >= nvars) return WK_VERTEX_INVALID;
            if (v2c[idx] == 0xFFFF) return WK_VERTEX_INVALID;
            proj_cols.push_back(v2c[idx]);
        }
        if (nrequired > MAX_COLS) return WK_ERR_BAD_ARG;
    }
    e->q_timed = false;
    bool light = steps[0].kind == KIND_C2U && steps.size() <= MAX_LIGHT_STEPS && !post;
    for (const PlannedStep &ps : steps)
        if (ps.kind == KIND_C2K) light = false;   // const_to_known runs on the multi-CTA path only
    if (e->profiling && !(light && srv_usable(e))) CUDA_TRY(cudaEventRecord(e->q_ev0, e->stream));
    const bool resident = light && srv_usable(e);
    e->last_resident = false;
    if (light) {   // the fused kernel clears the control block itself
        e->step = 0;
        e->recs.clear();
        e->event_next = 0;
    } else {
        srv_park(e);   // the persistent step kernels want every CTA slot of the device
        rc = reset_ctl(e);
        if (rc) return rc;
    }
    e->ncols = 0;

    uint64_t rows = 0;
    int cols = final_cols;
    bool table_in_host = false;
    size_t next = 0;
    if (light) {
        RecView rv;
        rc = resident ? run_light_resident(e, steps, want_table, proj_cols, rv)
                      : run_light(e, steps, mt_tid, mt_factor, want_table, proj_cols, rv);
        if (rc) return rc;
        if (rv.status & 1u) return WK_ERR_RBUF_OVERFLOW;
        e->last_resident = resident;
        next = (size_t)rv.resume;
        e->step = (int)next;
        e->ncols = (next == steps.size()) ? final_cols : steps[next].in_cols;
        rows = rv.rows;
        if (next == steps.size() && want_table && rows > 0) {
            // the fused kernel projected straight into the mapped staging area
            table_in_host = true;
            cols = nrequired;
        }
    }
    bool direct_done = false;
    if (next < steps.size()) {
        // multi-CTA path: one fused kernel per remaining step, no host sync in between
        if (resident && e->profiling) CUDA_TRY(cudaEventRecord(e->q_ev0, e->stream));   // the events then cover the continuation only
        // final_process fused into the last step: projected rows go straight into the caller's buffer when that is pinned
        // host memory the device can address (wk_host_alloc / cudaHostAlloc / cudaHostRegister)
        DirectOut dout{nullptr, 0, 0, nullptr};
        const int lk = steps.back().kind;
        if (want_table && !post && table && e->direct_out && e->variant >= 4 && (lk == KIND_K2U || lk == KIND_K2K || lk == KIND_K2C)) {
            if (table != e->dout_host) {
                cudaPointerAttributes pa;
                e->dout_host = table;
                e->dout_dev = nullptr;
                if (cudaPointerGetAttributes(&pa, table) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer)
                    e->dout_dev = (uint32_t *)pa.devicePointer;
                cudaGetLastError();
            }
            if (e->dout_dev) dout = DirectOut{e->dout_dev, cap_words, nrequired, proj_cols.data()};
        }
        for (size_t i = next; i < steps.size(); i++) {
            const PlannedStep &ps = steps[i];
            if (ps.kind == KIND_I2U) rc = enqueue_seed(e, KIND_I2U, 0, ps.pid, ps.dir, mt_tid, mt_factor);
            else if (ps.kind == KIND_C2U) rc = enqueue_seed(e, KIND_C2U, ps.vid, ps.pid, ps.dir, 0, 1);
            else if (ps.kind == KIND_C2K) rc = enqueue_to_known(e, KIND_C2K, ps.vid, ps.pid, ps.dir, ps.col_end, 0, 1);
            else if ((ps.kind == KIND_K2K || ps.kind == KIND_K2C) && e->fuse_filters && e->variant >= 4) {
                // a run of consecutive filters is one launch.  The conjunction does not depend on the order of its terms:
                // known_to_known (a join condition, usually the selective one) goes through the pipelined probe, the
                // others are evaluated only for the rows that survive it
                size_t j = i + 1;
                while (j < steps.size() && j - i < MAX_CHAIN && (steps[j].kind == KIND_K2K || steps[j].kind == KIND_K2C)) j++;
                const bool last = (j == steps.size()) && dout.dev_ptr;
                rc = enqueue_filter_chain(e, steps, i, j, last ? &dout : nullptr);
                direct_done = last;
                i = j - 1;
            }
            else {
                const bool last = (i + 1 == steps.size()) && dout.dev_ptr;
                rc = enqueue_known(e, ps.kind, ps.col_start, ps.pid, ps.dir, ps.col_end, ps.end_const, nullptr, 0, last ? &dout : nullptr);
                direct_done = last;
            }
            if (rc) return rc;
        }
        if (want_table && post) {
            // final_process order: DISTINCT, OFFSET, LIMIT, then the projection (sparql.hpp:1428-1550)
            if (opts->distinct) {
                rc = sync_rows(e, &rows);   // the sort is sized on the host
                if (rc) return rc;
                if (rows > 0) {
                    rc = enqueue_distinct(e, proj_cols.data(), nrequired, rows);
                    if (rc) return rc;
                }
            }
            if (opts->offset > 0 || opts->limit >= 0) {
                rc = enqueue_slice(e, (uint64_t)std::max<int64_t>(opts->offset, 0), opts->limit, e->cap_words / (uint64_t)std::max(1, e->ncols));
                if (rc) return rc;
            }
        }
        // final_process projection -- unless the table already is the projection (SELECT lists every column in table order)
        bool identity = want_table && (nrequired == final_cols) && (int)proj_cols.size() == nrequired;
        for (int i = 0; i < nrequired && identity; i++) identity = proj_cols[i] == i;
        if (want_table && !direct_done && !identity) {
            rc = enqueue_project(e, proj_cols.data(), nrequired);
            if (rc) return rc;
        }
        rc = sync_rows(e, &rows, e->profiling ? e->q_ev1 : nullptr);
        if (direct_done) {
            // the table is in the caller's buffer, not in the engine: leave an empty engine table behind
            e->ncols = 0;
            const uint64_t claimed = rows;
            reset_ctl(e);
            if (rc == WK_ERR_RBUF_OVERFLOW && claimed * (uint64_t)nrequired > cap_words) return WK_ERR_BAD_ARG;   // the caller's buffer is too small
        }
        if (rc) return rc;
        if (e->profiling) e->q_timed = true;
        e->last_resident = false;
        if (want_table) {
            // final_process leaves an empty table untouched (sparql.hpp:1425-1426)
            cols = rows > 0 ? nrequired : final_cols;
        }
        // the device is idle again: bring the light-query server back while the result is copied out
        if (e->srv.enabled && e->srv.launch_id != 0 && srv_usable(e)) {
            rc = srv_ensure_running(e, e->srv.seq + 1);
            if (rc) return rc;
        }
    }
    if (out_rows) *out_rows = rows;
    if (out_cols) *out_cols = cols;
    if (no_required && rows > 0) return WK_NO_REQUIRED_VAR;
    if (want_table && rows > 0 && table && !direct_done) {
        const uint64_t words = rows * (uint64_t)cols;
        if (words > cap_words) return WK_ERR_BAD_ARG;
        if (table_in_host) {
            memcpy(table, e->h_stage, words * sizeof(uint32_t));
        } else {
            CUDA_TRY(cudaMemcpyAsync(table, e->buf[e->step & 1], words * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
            CUDA_TRY(cudaStreamSynchronize(e->stream));
        }
    }
    return WK_SUCCESS;
}

// Throughput path (the reference's open-loop emulator keeps many light queries in flight, proxy.hpp:391-545):
// nqueries independent const-start plans, ONE launch, one CTA per query, blind replies.
int wk_query_execute_batch(wk_engine_t *e, const wk_pattern_t *patterns, const int32_t *pat_off, const int32_t *nvars,
                           int nqueries, uint64_t *out_rows, int32_t *out_status) {
    if (!e || !patterns || !pat_off || !nvars || !out_rows || !out_status || nqueries <= 0) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (nqueries > e->batch_cap) {
        if (e->d_bplans) { cudaFree(e->d_bplans); cudaFree(e->d_bres); cudaFreeHost(e->h_bplans); cudaFreeHost(e->h_bres); }
        e->batch_cap = nqueries;
        CUDA_TRY(cudaMalloc((void **)&e->d_bplans, (size_t)nqueries * sizeof(BatchPlan)));
        CUDA_TRY(cudaMalloc((void **)&e->d_bres, (size_t)nqueries * sizeof(BatchResult)));
        CUDA_TRY(cudaHostAlloc((void **)&e->h_bplans, (size_t)nqueries * sizeof(BatchPlan), cudaHostAllocDefault));
        CUDA_TRY(cudaHostAlloc((void **)&e->h_bres, (size_t)nqueries * sizeof(BatchResult), cudaHostAllocDefault));
    }
    std::vector<int> v2c;
    std::vector<PlannedStep> steps;
    for (int q = 0; q < nqueries; q++) {
        BatchPlan &bp = e->h_bplans[q];
        bp.nsteps = 0;
        steps.clear();
        int rc = plan_steps(patterns + pat_off[q], pat_off[q + 1] - pat_off[q], nvars[q], v2c, steps);
        if (rc == WK_SUCCESS && (steps[0].kind != KIND_C2U || (int)steps.size() > BATCH_STEPS)) rc = WK_UNKNOWN_PATTERN;
        for (const PlannedStep &ps : steps)
            if (ps.kind == KIND_C2K) rc = WK_UNKNOWN_PATTERN;
        if (rc == WK_SUCCESS) rc = fill_light_steps(e, steps, 0, 1, bp.steps);
        out_status[q] = rc;
        if (rc == WK_SUCCESS) bp.nsteps = (int)steps.size();
    }
    CUDA_TRY(cudaMemcpyAsync(e->d_bplans, e->h_bplans, (size_t)nqueries * sizeof(BatchPlan), cudaMemcpyHostToDevice, e->stream));
    srv_park(e);
    const int grid = std::min(nqueries, e->num_sms * 4);
    light_batch_kernel<<<grid, CTA_THREADS, 0, e->stream>>>(e->d_bplans, e->d_bres, nqueries, e->store->d_vertices, e->store->d_edges);
    CUDA_TRY(cudaGetLastError());
    e->launches++;
    CUDA_TRY(cudaMemcpyAsync(e->h_bres, e->d_bres, (size_t)nqueries * sizeof(BatchResult), cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int q = 0; q < nqueries; q++) {
        if (out_status[q] != WK_SUCCESS) { out_rows[q] = 0; continue; }
        if (e->h_bres[q].status == 2u) {   // outgrew shared memory: the general path answers it
            int cols = 0;
            out_status[q] = wk_query_execute(e, patterns + pat_off[q], pat_off[q + 1] - pat_off[q], nvars[q], nullptr, 0, 0, 1, 1,
                                             nullptr, 0, &out_rows[q], &cols);
        } else {
            out_rows[q] = e->h_bres[q].rows;
        }
    }
    return WK_SUCCESS;
}

int wk_engine_num_steps(wk_engine_t *e) {
    if (!e) return 0;
    if (cudaSetDevice(e->store->device) != cudaSuccess) return 0;
    if (snapshot_stats(e) != WK_SUCCESS) return 0;
    return (int)e->stats.size();
}

int wk_engine_step_stats(wk_engine_t *e, int step, wk_step_stats_t *out) {
    if (!e || !out || step < 0 || step >= (int)e->stats.size()) return WK_ERR_BAD_ARG;
    *out = e->stats[step];
    return WK_SUCCESS;
}

uint64_t wk_engine_launch_count(wk_engine_t *e) { return e ? e->launches : 0; }

__global__ void flush_read_kernel(const uint4 *p, size_t n, uint32_t *sink) {
    uint32_t acc = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = __ldcg(p + i);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
    }
    if (acc == 0x12345679u) *sink = acc;   // never true in practice; keeps the loads alive
}

// Evict the L2 between timed iterations: overwrite a scratch buffer several times the 50 MB L2, then read
// 256 MB of it back so that the cache is left full of CLEAN foreign lines (a write-only flush leaves
// an L2 full of dirty lines whose write-back would be charged to the next timed query).
int wk_engine_flush_l2(wk_engine_t *e) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (!e->d_flush) {
        e->flush_bytes = (size_t)384 << 20;
        CUDA_TRY(cudaMalloc(&e->d_flush, e->flush_bytes));
    }
    CUDA_TRY(cudaMemsetAsync(e->d_flush, ++e->flush_gen & 0xFF, e->flush_bytes, e->stream));
    flush_read_kernel<<<e->num_sms * 8, 256, 0, e->stream>>>((const uint4 *)e->d_flush, ((size_t)256 << 20) / sizeof(uint4),
                                                          (uint32_t *)e->d_flush);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return WK_SUCCESS;
}

int wk_host_alloc(uint64_t bytes, void **out) {
    if (!out) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable | cudaHostAllocMapped));
    return WK_SUCCESS;
}

int wk_host_free(void *p) {
    if (p) CUDA_TRY(cudaFreeHost(p));
    return WK_SUCCESS;
}

int wk_engine_last_query_device_us(wk_engine_t *e, float *us) {
    if (!e || !us) return WK_ERR_BAD_ARG;
    *us = 0;
    if (e->last_resident) {   // answered by the resident server: %globaltimer span inside the kernel (request acquired -> record stored)
        *us = (float)((double)e->srv.last_ns / 1000.0);
        return WK_SUCCESS;
    }
    if (!e->q_timed) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    CUDA_TRY(cudaEventSynchronize(e->q_ev1));
    float ms = 0;
    CUDA_TRY(cudaEventElapsedTime(&ms, e->q_ev0, e->q_ev1));
    *us = ms * 1000.0f;
    return WK_SUCCESS;
}

}  // extern "C"

#include "wk_sharded.cuh"

static uint64_t comm_bytes_pushed(const wk_engine *e) { return e->comm ? e->comm->bytes_pushed : 0; }

// the sharded light-query server's view of the group (wk_server.cuh)
static int srv_fill_peers(wk_engine *e, SrvPeers &Q) {
    memset(&Q, 0, sizeof(Q));
    wk_comm *c = e->comm;
    if (!c || !c->peer_stores || !c->p2p || !c->d_xctl || !c->d_segr_tab || c->nranks > LIGHT_PEERS) return WK_ERR_BAD_ARG;
    for (int r = 0; r < c->nranks; r++) {
        Q.pv[r] = c->peer_v[r];
        Q.pe[r] = c->peer_e[r];
        Q.peer_flag[r] = (r == c->rank) ? nullptr : &c->p2p->ctl[r]->flagL[c->rank];
    }
    Q.my_flag = c->d_xctl->flagL;
    Q.segr_tab = c->d_segr_tab;
    Q.nranks = (uint32_t)c->nranks;
    Q.rank = (uint32_t)c->rank;
    return WK_SUCCESS;
}

// [my segment slot][rank]: bucket range and modulo magic of that (index, pid, dir) segment in every shard.  A shard without
// the segment gets bucket 0 of its store, whose keys belong to another (pid, dir) and never compare equal: the probe misses.
static int comm_build_segr_tab(wk_engine *e) {
    wk_comm *c = e->comm;
    srv_stop(e);   // a resident sharded server reads the old table
    if (c->d_segr_tab) { cudaFree(c->d_segr_tab); c->d_segr_tab = nullptr; }
    const int ns = e->store->nsegslots;
    if (ns <= 0 || (int)c->peer_segs.size() < c->nranks) return WK_SUCCESS;
    SegLite none;
    memset(&none, 0, sizeof(none));
    none.bucket_start = 0;
    none.fm = make_fastmod(1);
    std::vector<SegLite> tab((size_t)ns * LIGHT_PEERS, none);
    for (auto &kv : e->store->seg_slot) {
        for (int r = 0; r < c->nranks; r++) {
            auto it = c->peer_segs[r].find(kv.first);
            if (it == c->peer_segs[r].end() || it->second.num_buckets == 0) continue;
            SegLite &sl = tab[(size_t)kv.second * LIGHT_PEERS + r];
            sl.bucket_start = it->second.bucket_start;
            sl.fm = make_fastmod(it->second.num_buckets);
        }
    }
    CUDA_TRY(cudaMalloc((void **)&c->d_segr_tab, tab.size() * sizeof(SegLite)));
    CUDA_TRY(cudaMemcpy(c->d_segr_tab, tab.data(), tab.size() * sizeof(SegLite), cudaMemcpyHostToDevice));
    return WK_SUCCESS;
}

static void comm_free(wk_engine *e) {
    wk_comm *c = e->comm;
    if (!c) return;
    for (void *p : c->ipc_opened) cudaIpcCloseMemHandle(p);
    if (c->comm && nccl_api().CommDestroy) nccl_api().CommDestroy(c->comm);
    if (c->d_counts) cudaFree(c->d_counts);
    if (c->d_cursor) cudaFree(c->d_cursor);
    if (c->d_matrix) cudaFree(c->d_matrix);
    if (c->h_matrix) cudaFreeHost(c->h_matrix);
    if (c->d_xctl) cudaFree(c->d_xctl);
    if (c->d_p2p_local) cudaFree(c->d_p2p_local);
    if (c->d_segr_tab) cudaFree(c->d_segr_tab);
    delete c->p2p;
    delete c;
    e->comm = nullptr;
}

static int comm_alloc(wk_engine *e, int nranks, int rank) {
    if (nranks < 1 || nranks > MAX_PARTS || rank < 0 || rank >= nranks) return WK_ERR_BAD_ARG;
    wk_comm *c = new wk_comm();
    c->nranks = nranks;
    c->rank = rank;
    CUDA_TRY(cudaMalloc((void **)&c->d_counts, MAX_PARTS * sizeof(uint64_t)));
    CUDA_TRY(cudaMalloc((void **)&c->d_cursor, MAX_PARTS * sizeof(uint64_t)));
    CUDA_TRY(cudaMalloc((void **)&c->d_matrix, (size_t)nranks * MAX_PARTS * sizeof(uint64_t)));
    CUDA_TRY(cudaHostAlloc((void **)&c->h_matrix, (size_t)nranks * MAX_PARTS * sizeof(uint64_t), cudaHostAllocDefault));
    e->comm = c;
    return WK_SUCCESS;
}

// bucketise the current table (buf[step&1], counts[step]) by row[col] % nparts into buf[(step+1)&1]
static int partition_table(wk_engine *e, int col, int nparts) {
    wk_comm *c = e->comm;
    if (e->ncols <= 0 || col < 0 || col >= e->ncols) return WK_VERTEX_INVALID;
    if (nparts < 1 || nparts >= MAX_PARTS) return WK_ERR_BAD_ARG;   // the last counter carries the overflow verdict
    srv_park(e);
    const int s = e->step;
    CUDA_TRY(cudaMemsetAsync(c->d_counts, 0, MAX_PARTS * sizeof(uint64_t), e->stream));
    const int grid = e->num_sms * 4;
    part_count_kernel<<<grid, CTA_THREADS, 0, e->stream>>>(e->buf[s & 1], &e->d_ctl->counts[s], e->ncols, col, (uint32_t)nparts, c->d_counts,
                                                           &e->d_ctl->status);
    part_scan_kernel<<<1, 1, 0, e->stream>>>(c->d_counts, c->d_cursor, (uint32_t)nparts);
    part_scatter_kernel<<<grid, CTA_THREADS, 0, e->stream>>>(e->buf[s & 1], &e->d_ctl->counts[s], e->ncols, col, (uint32_t)nparts,
                                                             c->d_cursor, e->buf[(s + 1) & 1], &e->d_ctl->status);
    CUDA_TRY(cudaGetLastError());
    e->launches += 3;
    return WK_SUCCESS;
}

// all-to-all(v) of the table.  col >= 0: rows go to rank row[col] % nranks, result stays in buf[step&1];
// col == -2: every rank receives every row (type-index lookups), result in buf[(step+1)&1], step advances.
static int exchange_table(wk_engine *e, int col, uint64_t *out_rows) {
    wk_comm *c = e->comm;
    NcclApi &nc = nccl_api();
    if (!c || !c->comm || !nc.ok) return WK_ERR_COMM;
    const int n = c->nranks, me = c->rank, s = e->step, C = e->ncols;
    if (C <= 0) return WK_ERR_BAD_ARG;
    const bool dup = (col == -2);
    if (!dup) {
        int rc = partition_table(e, col, n);
        if (rc) return rc;
    } else {
        // every destination gets the whole table: counts[d] = N for all d
        dup_counts_kernel<<<1, MAX_PARTS, 0, e->stream>>>(c->d_counts, &e->d_ctl->counts[s], n, &e->d_ctl->status);
        CUDA_TRY(cudaGetLastError());
        e->launches++;
    }
    // counts: all-gather the per-destination vectors, then every rank knows the whole n x n matrix
    NCCL_TRY(nc.AllGather(c->d_counts, c->d_matrix, MAX_PARTS, ncclUint64, c->comm, e->stream));
    CUDA_TRY(cudaMemcpyAsync(c->h_matrix, c->d_matrix, (size_t)n * MAX_PARTS * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    // every rank evaluates every rank's receive total, so an overflow is seen by all of them alike; so is an overflow
    // that happened in the step before the exchange on any rank (its verdict travels in the last counter)
    bool overflow = false;
    for (int r = 0; r < n; r++)
        if (c->h_matrix[(size_t)r * MAX_PARTS + MAX_PARTS - 1] != 0) overflow = true;
    for (int r = 0; r < n; r++) {
        uint64_t tot = 0;
        for (int src = 0; src < n; src++) tot += c->h_matrix[(size_t)src * MAX_PARTS + r];
        if (tot * (uint64_t)C > e->cap_words) overflow = true;
    }
    if (overflow) return WK_ERR_RBUF_OVERFLOW;
    uint64_t send_off[MAX_PARTS], recv_off[MAX_PARTS], acc = 0, racc = 0;
    for (int d = 0; d < n; d++) {
        send_off[d] = dup ? 0 : acc;
        acc += c->h_matrix[(size_t)me * MAX_PARTS + d];
        recv_off[d] = racc;
        racc += c->h_matrix[(size_t)d * MAX_PARTS + me];
    }
    const uint32_t *send_base = dup ? e->buf[s & 1] : e->buf[(s + 1) & 1];
    uint32_t *recv_base = dup ? e->buf[(s + 1) & 1] : e->buf[s & 1];
    NCCL_TRY(nc.GroupStart());
    for (int peer = 0; peer < n; peer++) {
        const uint64_t sc = c->h_matrix[(size_t)me * MAX_PARTS + peer], rcnt = c->h_matrix[(size_t)peer * MAX_PARTS + me];
        if (peer == me) continue;
        if (sc) NCCL_TRY(nc.Send(send_base + send_off[peer] * (uint64_t)C, sc * (uint64_t)C, ncclUint32, peer, c->comm, e->stream));
        if (rcnt) NCCL_TRY(nc.Recv(recv_base + recv_off[peer] * (uint64_t)C, rcnt * (uint64_t)C, ncclUint32, peer, c->comm, e->stream));
    }
    NCCL_TRY(nc.GroupEnd());
    {   // own share: device-to-device copy
        const uint64_t sc = c->h_matrix[(size_t)me * MAX_PARTS + me];
        if (sc) CUDA_TRY(cudaMemcpyAsync(recv_base + recv_off[me] * (uint64_t)C, send_base + send_off[me] * (uint64_t)C,
                                         sc * (uint64_t)C * sizeof(uint32_t), cudaMemcpyDeviceToDevice, e->stream));
    }
    const int dst_step = dup ? s + 1 : s;
    set_count_kernel<<<1, 1, 0, e->stream>>>(&e->d_ctl->counts[dst_step], racc);
    CUDA_TRY(cudaGetLastError());
    e->launches++;
    e->step = dst_step;
    c->exchanges++;
    c->rows_sent += acc - c->h_matrix[(size_t)me * MAX_PARTS + me];
    c->rows_recv += racc - c->h_matrix[(size_t)me * MAX_PARTS + me];
    c->partitioned = false;
    if (out_rows) *out_rows = racc;
    return WK_SUCCESS;
}

// exchange over peer memory: result in buf[(step+1)&1], step advances; no host synchronisation, one pass over the table
static int exchange_table_p2p(wk_engine *e, int col) {
    wk_comm *c = e->comm;
    if (!c || !c->p2p_ready) return WK_ERR_COMM;
    if (c->poisoned) return WK_ERR_COMM;
    const int s = e->step, C = e->ncols;
    if (C <= 0) return WK_ERR_BAD_ARG;
    const bool dup = (col == -2);
    if (!dup && (col < 0 || col >= C)) return WK_VERTEX_INVALID;
    srv_park(e);
    const uint64_t epoch = ++c->epoch;
    const uint64_t cap_rows = e->cap_words / (uint64_t)C;
    // ranks of one process may share a device: there only single-CTA kernels wait (a grid of waiting CTAs could keep a peer's
    // kernel from becoming resident) and the grid leaves room for the peers; ranks on devices of their own take barrier A
    // inside the push kernel (one launch less)
    const bool ready_inside = !c->local_group;
    // tile = 1024 / 512 / 256 rows: two row buffers (the next tile is in flight while this one is grouped) + the staging area
    // = 36 KB of shared memory for three columns, 4-5 CTAs per SM (large tiles: the fetch of the next tile has a whole tile's
    // work to hide behind)
    const int rpt = C <= 4 ? 4 : (C <= 8 ? 2 : 1);
    const size_t smem = 3 * (size_t)CTA_THREADS * rpt * C * sizeof(uint32_t);
    void (*kfn)(P2PTable, XchCtl *, P2PLocal *, const uint32_t *, const uint64_t *, int, int, int, int, uint64_t, uint64_t, uint32_t *, int, int, int, uint32_t) =
        rpt == 4 ? p2p_push_kernel<4> : (rpt == 2 ? p2p_push_kernel<2> : p2p_push_kernel<1>);
    if (smem > 40 * 1024) CUDA_TRY(cudaFuncSetAttribute((const void *)kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // several CTAs per SM hide the barriers of the tile pipeline and the round trip of the remote reservations
    int per_sm = (int)std::min<size_t>(5, std::max<size_t>(1, (200 * 1024) / std::max<size_t>(smem + 1024, 1)));
    // experiment knobs of scripts/exchange_bench.py: tiles per reservation, CTAs per SM, timing-only debug modes
    const char *ev_g = getenv("WK_P2P_G"), *ev_c = getenv("WK_P2P_CTAS"), *ev_d = getenv("WK_P2P_DEBUG");
    const int k_gmax = ev_g ? std::max(1, atoi(ev_g)) : (int)P2P_CHUNK_TILES;
    const int k_ctas = ev_c ? atoi(ev_c) : 0;
    const int k_dbg = ev_d ? atoi(ev_d) : 0;
    if (k_ctas > 0) per_sm = std::min(per_sm, k_ctas);
    const int grid = c->local_group ? std::max(1, e->num_sms * 4 / std::max(1, c->nranks)) : e->num_sms * per_sm;
    StepRecord &r = begin_step(e, KIND_EXCHANGE, C);
    if (!ready_inside) p2p_ready_kernel<<<1, 64, 0, e->stream>>>(*c->p2p, c->d_xctl, c->d_p2p_local, epoch, &e->d_ctl->status);
    kfn<<<grid, CTA_THREADS, smem, e->stream>>>(*c->p2p, c->d_xctl, c->d_p2p_local, e->buf[s & 1], &e->d_ctl->counts[s], C, dup ? 0 : col,
                                                dup ? 1 : 0, (s + 1) & 1, epoch, cap_rows, &e->d_ctl->status, ready_inside ? 1 : 0, k_gmax, k_dbg,
                                                c->nranks > 1 ? (uint32_t)(((1ull << 32) + (uint64_t)c->nranks - 1) / (uint64_t)c->nranks) : 0u);
    p2p_wait_kernel<<<1, 64, 0, e->stream>>>(*c->p2p, c->d_xctl, c->d_p2p_local, epoch, cap_rows, &e->d_ctl->counts[s + 1], &e->d_ctl->status,
                                             &e->d_ctl->stats[2 * s]);
    CUDA_TRY(cudaGetLastError());
    end_step(e, r, ready_inside ? 2 : 3);
    e->step = s + 1;
    c->exchanges++;
    return WK_SUCCESS;
}

extern "C" {

// ---- peer-memory communicator (CUDA IPC): every rank exports 3 handles (its two result buffers and its exchange
// control block, 64 bytes each), all ranks gather the 192-byte records and import them ------------------------------
int wk_comm_p2p_export(wk_engine_t *e, int nranks, int rank, void *out192) {
    if (!e || !out192) return WK_ERR_BAD_ARG;
    if (nranks < 1 || nranks > P2P_MAX_RANKS) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (!e->comm) {
        int rc = comm_alloc(e, nranks, rank);
        if (rc) return rc;
    }
    wk_comm *c = e->comm;
    c->nranks = nranks;
    c->rank = rank;
    if (!c->d_xctl) {
        CUDA_TRY(cudaMalloc((void **)&c->d_xctl, sizeof(XchCtl)));
        CUDA_TRY(cudaMemset(c->d_xctl, 0, sizeof(XchCtl)));
        CUDA_TRY(cudaMalloc((void **)&c->d_p2p_local, sizeof(P2PLocal)));
        CUDA_TRY(cudaMemset(c->d_p2p_local, 0, sizeof(P2PLocal)));
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    cudaIpcMemHandle_t *h = (cudaIpcMemHandle_t *)out192;
    CUDA_TRY(cudaIpcGetMemHandle(&h[0], e->buf[0]));
    CUDA_TRY(cudaIpcGetMemHandle(&h[1], e->buf[1]));
    CUDA_TRY(cudaIpcGetMemHandle(&h[2], c->d_xctl));
    return WK_SUCCESS;
}

int wk_comm_p2p_import(wk_engine_t *e, const void *all_handles) {
    if (!e || !e->comm || !e->comm->d_xctl || !all_handles) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    wk_comm *c = e->comm;
    if (!c->p2p) c->p2p = new P2PTable();
    memset(c->p2p, 0, sizeof(P2PTable));
    c->p2p->nranks = c->nranks;
    c->p2p->rank = c->rank;
    const cudaIpcMemHandle_t *h = (const cudaIpcMemHandle_t *)all_handles;
    for (int r = 0; r < c->nranks; r++) {
        if (r == c->rank) {
            c->p2p->buf[0][r] = e->buf[0];
            c->p2p->buf[1][r] = e->buf[1];
            c->p2p->ctl[r] = c->d_xctl;
            continue;
        }
        void *p[3];
        for (int k = 0; k < 3; k++) {
            CUDA_TRY(cudaIpcOpenMemHandle(&p[k], h[3 * r + k], cudaIpcMemLazyEnablePeerAccess));
            c->ipc_opened.push_back(p[k]);
        }
        c->p2p->buf[0][r] = (uint32_t *)p[0];
        c->p2p->buf[1][r] = (uint32_t *)p[1];
        c->p2p->ctl[r] = (XchCtl *)p[2];
    }
    c->p2p_ready = true;
    return WK_SUCCESS;
}

// ---- peers' stores for in-place light queries: every rank exports the IPC handles of its header and edge arrays plus
// its segment table (each shard sizes its segments on its own); blob = [2 x 64-byte handles][int32 nsegs][pad][segs] --------
int wk_comm_p2p_export_store(wk_engine_t *e, void *blob, uint64_t cap, uint64_t *size) {
    if (!e || !size) return WK_ERR_BAD_ARG;
    const uint64_t need = 2 * sizeof(cudaIpcMemHandle_t) + 8 + e->store->segs.size() * sizeof(wk_segmeta_t);
    *size = need;
    if (!blob || cap < need) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    uint8_t *p = (uint8_t *)blob;
    cudaIpcMemHandle_t h[2];
    CUDA_TRY(cudaIpcGetMemHandle(&h[0], e->store->d_vertices));
    CUDA_TRY(cudaIpcGetMemHandle(&h[1], e->store->d_edges));
    memcpy(p, h, sizeof(h));
    const int32_t ns = (int32_t)e->store->segs.size();
    memcpy(p + sizeof(h), &ns, 4);
    memset(p + sizeof(h) + 4, 0, 4);
    wk_segmeta_t *dst = (wk_segmeta_t *)(p + sizeof(h) + 8);
    int i = 0;
    for (auto &kv : e->store->segs) dst[i++] = kv.second;
    return WK_SUCCESS;
}

// blobs: the nranks exported blobs back to back, offsets[r] .. offsets[r + 1] delimit rank r's
int wk_comm_p2p_import_store(wk_engine_t *e, const void *blobs, const uint64_t *offsets, int nranks) {
    if (!e || !e->comm || !e->comm->p2p_ready || !blobs || !offsets) return WK_ERR_BAD_ARG;
    wk_comm *c = e->comm;
    if (nranks != c->nranks || nranks > LIGHT_PEERS) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    c->peer_segs.assign(nranks, {});
    for (int r = 0; r < nranks; r++) {
        const uint8_t *p = (const uint8_t *)blobs + offsets[r];
        const uint64_t len = offsets[r + 1] - offsets[r];
        if (len < 2 * sizeof(cudaIpcMemHandle_t) + 8) return WK_ERR_BAD_ARG;
        int32_t ns = 0;
        memcpy(&ns, p + 2 * sizeof(cudaIpcMemHandle_t), 4);
        if (ns < 0 || len < 2 * sizeof(cudaIpcMemHandle_t) + 8 + (uint64_t)ns * sizeof(wk_segmeta_t)) return WK_ERR_BAD_ARG;
        const wk_segmeta_t *sg = (const wk_segmeta_t *)(p + 2 * sizeof(cudaIpcMemHandle_t) + 8);
        for (int i = 0; i < ns; i++) c->peer_segs[r][SegKey(sg[i].index, sg[i].pid, sg[i].dir)] = sg[i];
        if (r == c->rank) {
            c->peer_v[r] = e->store->d_vertices;
            c->peer_e[r] = e->store->d_edges;
            continue;
        }
        cudaIpcMemHandle_t h[2];
        memcpy(h, p, sizeof(h));
        void *q[2];
        for (int k = 0; k < 2; k++) {
            CUDA_TRY(cudaIpcOpenMemHandle(&q[k], h[k], cudaIpcMemLazyEnablePeerAccess));
            c->ipc_opened.push_back(q[k]);
        }
        c->peer_v[r] = (const uint4 *)q[0];
        c->peer_e[r] = (const uint32_t *)q[1];
    }
    c->peer_stores = true;
    return comm_build_segr_tab(e);
}

// Engines of ONE process as a group (several shards per GPU, or one thread per GPU): the peers' buffers, control blocks
// and store arrays are wired directly instead of through CUDA IPC, which cannot open a handle in the process that made it.
// engines[r] becomes rank r.  Every engine still needs its own caller thread: the exchange kernels of a rank wait for
// the other ranks' kernels, so the n calls of one collective query must be in flight together.
int wk_comm_local_group(wk_engine_t **engines, int n) {
    if (!engines || n < 1 || n > P2P_MAX_RANKS || n > LIGHT_PEERS) return WK_ERR_BAD_ARG;
    for (int r = 0; r < n; r++) {
        if (!engines[r]) return WK_ERR_BAD_ARG;
        for (int q = 0; q < r; q++)
            if (engines[q] == engines[r]) return WK_ERR_BAD_ARG;
        if (engines[r]->cap_words != engines[0]->cap_words) return WK_ERR_BAD_ARG;   // owners' capacities are checked by the pushers
    }
    for (int r = 0; r < n; r++) {
        wk_engine *e = engines[r];
        CUDA_TRY(cudaSetDevice(e->store->device));
        if (!e->comm) {
            int rc = comm_alloc(e, n, r);
            if (rc) return rc;
        }
        wk_comm *c = e->comm;
        c->nranks = n;
        c->rank = r;
        if (!c->d_xctl) {
            CUDA_TRY(cudaMalloc((void **)&c->d_xctl, sizeof(XchCtl)));
            CUDA_TRY(cudaMalloc((void **)&c->d_p2p_local, sizeof(P2PLocal)));
        }
        CUDA_TRY(cudaMemset(c->d_xctl, 0, sizeof(XchCtl)));
        CUDA_TRY(cudaMemset(c->d_p2p_local, 0, sizeof(P2PLocal)));
        for (int q = 0; q < n; q++) {
            const int dq = engines[q]->store->device;
            if (dq != e->store->device) {
                int can = 0;
                CUDA_TRY(cudaDeviceCanAccessPeer(&can, e->store->device, dq));
                if (!can) return WK_ERR_COMM;
                cudaError_t pe = cudaDeviceEnablePeerAccess(dq, 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CUDA_TRY(pe);
                cudaGetLastError();
            }
        }
    }
    for (int r = 0; r < n; r++) {
        wk_engine *e = engines[r];
        wk_comm *c = e->comm;
        if (!c->p2p) c->p2p = new P2PTable();
        memset(c->p2p, 0, sizeof(P2PTable));
        c->p2p->nranks = n;
        c->p2p->rank = r;
        c->peer_segs.assign(n, {});
        for (int q = 0; q < n; q++) {
            c->p2p->buf[0][q] = engines[q]->buf[0];
            c->p2p->buf[1][q] = engines[q]->buf[1];
            c->p2p->ctl[q] = engines[q]->comm->d_xctl;
            c->peer_v[q] = engines[q]->store->d_vertices;
            c->peer_e[q] = engines[q]->store->d_edges;
            c->peer_segs[q] = engines[q]->store->segs;
        }
        c->epoch = 0;
        c->poisoned = false;
        c->local_group = true;
        c->p2p_ready = true;
        c->peer_stores = true;
        CUDA_TRY(cudaSetDevice(e->store->device));
        int rc = comm_build_segr_tab(e);
        if (rc) return rc;
    }
    return WK_SUCCESS;
}

// wk_exchange over peer memory instead of NCCL (same semantics; the table moves to the other buffer)
int wk_exchange_p2p(wk_engine_t *e, int col_start, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    int rc = ensure_step_room(e);
    if (rc) return rc;
    rc = exchange_table_p2p(e, col_start);
    if (rc) return rc;
    if (out_rows) {
        rc = sync_rows(e, out_rows);
        if (rc) return rc;
    }
    return WK_SUCCESS;
}

int wk_partition(wk_engine_t *e, int col_start, int nparts, uint64_t *part_rows) {
    if (!e || !part_rows) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (!e->comm) {
        int rc = comm_alloc(e, 1, 0);
        if (rc) return rc;
    }
    int rc = ensure_step_room(e);
    if (rc) return rc;
    rc = partition_table(e, col_start, nparts);
    if (rc) return rc;
    wk_comm *c = e->comm;
    CUDA_TRY(cudaMemcpyAsync(c->h_matrix, c->d_counts, MAX_PARTS * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    if (c->h_matrix[MAX_PARTS - 1] != 0) return WK_ERR_RBUF_OVERFLOW;   // the table overflowed in the step before
    uint64_t acc = 0;
    for (int d = 0; d < nparts; d++) {
        c->part_rows[d] = part_rows[d] = c->h_matrix[d];
        c->part_off[d] = acc;
        acc += c->h_matrix[d];
    }
    if (acc * (uint64_t)e->ncols > e->cap_words) return WK_ERR_RBUF_OVERFLOW;
    c->partitioned = true;
    return WK_SUCCESS;
}

int wk_partition_ptr(wk_engine_t *e, int part, const wk_sid_t **d_ptr, uint64_t *rows) {
    if (!e || !e->comm || !e->comm->partitioned || part < 0 || part >= MAX_PARTS || !d_ptr || !rows) return WK_ERR_BAD_ARG;
    *d_ptr = e->buf[(e->step + 1) & 1] + e->comm->part_off[part] * (uint64_t)e->ncols;
    *rows = e->comm->part_rows[part];
    return WK_SUCCESS;
}

int wk_comm_unique_id(void *id128) {
    NcclApi &nc = nccl_api();
    if (!nc.ok || !id128) return WK_ERR_COMM;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    NCCL_TRY(nc.GetUniqueId((ncclUniqueId *)id128));
    return WK_SUCCESS;
}

int wk_comm_init(wk_engine_t *e, int nranks, int rank, const void *id128) {
    if (!e || !id128) return WK_ERR_BAD_ARG;
    NcclApi &nc = nccl_api();
    if (!nc.ok) return WK_ERR_COMM;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (!e->comm) {
        int rc = comm_alloc(e, nranks, rank);
        if (rc) return rc;
    }
    e->comm->nranks = nranks;
    e->comm->rank = rank;
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    NCCL_TRY(nc.CommInitRank(&e->comm->comm, nranks, id, rank));
    return WK_SUCCESS;
}

int wk_exchange(wk_engine_t *e, int col_start, uint64_t *out_rows) {
    if (!e) return WK_ERR_BAD_ARG;
    CUDA_TRY(cudaSetDevice(e->store->device));
    int rc = ensure_step_room(e);
    if (rc) return rc;
    return exchange_table(e, col_start, out_rows);
}

int wk_comm_stats(wk_engine_t *e, uint64_t *exchanges, uint64_t *rows_sent, uint64_t *rows_recv) {
    if (!e || !e->comm) return WK_ERR_COMM;
    uint64_t sent = e->comm->rows_sent, recv = e->comm->rows_recv;
    if (e->comm->d_p2p_local) {   // the peer-memory exchange keeps its totals on the device (no host sync per exchange)
        CUDA_TRY(cudaSetDevice(e->store->device));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
        P2PLocal loc;
        CUDA_TRY(cudaMemcpy(&loc, e->comm->d_p2p_local, sizeof(loc), cudaMemcpyDeviceToHost));
        sent += loc.rows_sent;
        recv += loc.rows_landed - loc.rows_kept;
        e->comm->bytes_pushed = loc.bytes_pushed;
    }
    if (exchanges) *exchanges = e->comm->exchanges;
    if (rows_sent) *rows_sent = sent;
    if (rows_recv) *rows_recv = recv;
    return WK_SUCCESS;
}

// host-only: which steps of a plan exchange, for `nranks` shards (out[npatterns])
int wk_plan_exchanges(const wk_pattern_t *patterns, int npatterns, int nvars, int32_t *out) {
    if (!patterns || !out) return WK_ERR_BAD_ARG;
    std::vector<int> v2c;
    std::vector<PlannedStep> steps;
    int rc = plan_steps(patterns, npatterns, nvars, v2c, steps);
    if (rc) return rc;
    for (const PlannedStep &ps : steps)
        if (ps.kind == KIND_C2K) return WK_OBJ_ERROR;   // need_fork_join refuses a subject that is not a known variable (sparql.hpp:808)
    std::vector<int> ex;
    plan_exchanges(steps, ex);
    for (size_t i = 0; i < ex.size(); i++) out[i] = ex[i];
    return WK_SUCCESS;
}

int wk_query_execute_sharded(wk_engine_t *e, const wk_pattern_t *patterns, int npatterns, int nvars,
                             const int32_t *required_vars, int nrequired, int mt_tid, int mt_factor, int blind,
                             wk_sid_t *table, uint64_t cap_words, uint64_t *out_rows, int *out_cols) {
    if (!e || !patterns) return WK_ERR_BAD_ARG;
    if (!e->comm || (!e->comm->comm && !e->comm->p2p_ready)) return WK_ERR_COMM;
    CUDA_TRY(cudaSetDevice(e->store->device));
    if (out_rows) *out_rows = 0;
    if (out_cols) *out_cols = 0;
    std::vector<int> v2c;
    std::vector<PlannedStep> steps;
    int rc = plan_steps(patterns, npatterns, nvars, v2c, steps);
    if (rc) return rc;
    if ((int)steps.size() > MAX_STEPS / 2 - 2) return WK_ERR_BAD_ARG;
    // a pattern that starts from a constant after the first step has no owner to fork to: the reference's fork-join
    // raises OBJ_ERROR for a subject that is not a known variable (need_fork_join, sparql.hpp:808)
    for (const PlannedStep &ps : steps)
        if (ps.kind == KIND_C2K) return WK_OBJ_ERROR;
    if (e->comm->poisoned) return WK_ERR_COMM;
    std::vector<int> ex;
    plan_exchanges(steps, ex);
    const int final_cols = steps.back().in_cols + ((steps.back().kind == KIND_K2K || steps.back().kind == KIND_K2C) ? 0 : 1);
    const bool no_required = !blind && (nrequired <= 0 || !required_vars);
    const bool want_table = !blind && !no_required;
    std::vector<int32_t> proj_cols;
    if (want_table) {
        for (int i = 0; i < nrequired; i++) {
            const int idx = -(required_vars[i] + 1);
            if (required_vars[i] >= 0 || idx >= nvars || v2c[idx] == 0xFFFF) return WK_VERTEX_INVALID;
            proj_cols.push_back(v2c[idx]);
        }
    }
    e->q_timed = false;
    e->last_resident = false;
    if (e->profiling) CUDA_TRY(cudaEventRecord(e->q_ev0, e->stream));
    const int n = e->comm->nranks, me = e->comm->rank;
    // In-place execution of a light query (the reference answers small tables with one-sided remote reads instead of a
    // fork-join, sparql.hpp:802-814): the constant's owner walks the other shards through peer memory, nobody exchanges.
    // Every rank takes the same decision from the plan alone; the owner's verdict (answered / outgrew shared memory)
    // reaches the peers through a flag, and an outgrown query is redone by all shards together below.
    bool in_place = e->comm->peer_stores && e->comm->p2p_ready && steps[0].kind == KIND_C2U &&
                    (int)steps.size() <= LIGHT_SHARDED_STEPS && n <= LIGHT_PEERS && getenv("WK_NO_INPLACE") == nullptr;
    for (const PlannedStep &ps : steps)
        if (ps.kind == KIND_C2K || (ps.kind == KIND_K2U && ps.pid == WK_TYPE_ID && ps.dir == WK_DIR_IN)) in_place = false;
    if (in_place) {
        const int owner = (int)(steps[0].vid % (uint64_t)n);
        const uint64_t epoch = ++e->comm->epoch;
        // resident servers on every rank (wk_server.cuh): the owner's server walks the shards, the peers' servers wait for
        // its verdict; nobody launches anything.  The phase trace (profiling 3) stays on the launch path.
        const bool resident = srv_usable(e) && e->comm->d_segr_tab != nullptr && e->profiling < 3;
        e->last_resident = false;
        if (resident) {
            e->step = 0;
            e->recs.clear();
            e->event_next = 0;
            RecView rv;
            if (me == owner) {
                rc = run_light_resident(e, steps, want_table, proj_cols, rv, epoch);
                if (rc == WK_ERR_NO_SEGMENT) {   // nothing was posted; the peers are waiting for a verdict: "answered"
                    p2p_light_verdict_kernel<<<1, 64, 0, e->stream>>>(*e->comm->p2p, 2 * epoch);
                    e->launches++;
                }
                if (rc) return rc;
                if (rv.status & 1u) return WK_ERR_RBUF_OVERFLOW;
                if (rv.resume == (int)steps.size()) {
                    e->last_resident = true;
                    const uint64_t rows = rv.rows;
                    const int cols = (want_table && rows > 0) ? nrequired : final_cols;
                    if (out_rows) *out_rows = rows;
                    if (out_cols) *out_cols = cols;
                    if (no_required && rows > 0) return WK_NO_REQUIRED_VAR;
                    if (want_table && rows > 0 && table) {
                        const uint64_t words = rows * (uint64_t)cols;
                        if (words > cap_words) return WK_ERR_BAD_ARG;
                        memcpy(table, e->h_stage, words * sizeof(uint32_t));
                    }
                    return WK_SUCCESS;
                }
                // outgrew shared memory: every peer has been told; fall through to the collective plan
            } else {
                SrvChunk ch[SRV_CHUNKS];
                memset(ch, 0, sizeof(ch));
                ch[0].w0 = ((uint32_t)SRV_F_WAIT << 8) | ((uint32_t)owner << 16);
                ch[0].w1 = (uint32_t)epoch;
                ch[0].w2 = (uint32_t)(epoch >> 32);
                rc = srv_roundtrip(e, ch, -1, 0, true, rv);
                if (rc) return rc;
                if (rv.status & 2u) { e->comm->poisoned = true; return WK_ERR_COMM; }
                if (!(rv.status & 4u)) {   // answered by the owner: this shard contributes no rows
                    e->last_resident = true;
                    if (out_rows) *out_rows = 0;
                    if (out_cols) *out_cols = want_table ? nrequired : final_cols;
                    return WK_SUCCESS;
                }
            }
        } else if (me == owner) {
            LightPlanSharded sp;
            memset(&sp, 0, sizeof(sp));
            LightPlan &lp = sp.lp;
            lp.vertices = e->store->d_vertices;
            lp.edges = e->store->d_edges;
            lp.buf[0] = e->buf[0];
            lp.buf[1] = e->buf[1];
            lp.counts = e->d_ctl->counts;
            lp.stats = e->d_ctl->stats;
            lp.status = &e->d_ctl->status;
            lp.ctl_words = (uint64_t *)e->d_ctl;
            lp.ctl_nwords = (int)(sizeof(CtlBlock) / sizeof(uint64_t));
            lp.rec = e->d_rec;
            lp.host_table = e->d_stage;
            lp.host_table_words = e->stage_words;
            lp.cap_words = e->cap_words;
            lp.nsteps = (int)steps.size();
            lp.do_project = want_table ? 1 : 0;
            lp.proj_n = (int)proj_cols.size();
            for (size_t i = 0; i < proj_cols.size(); i++) lp.proj_cols[i] = (int8_t)proj_cols[i];
            rc = fill_light_steps(e, steps, 0, 1, lp.steps);
            if (rc) {   // the peers are waiting for a verdict: "answered" (this rank alone reports the error)
                p2p_light_verdict_kernel<<<1, 64, 0, e->stream>>>(*e->comm->p2p, 2 * epoch);
                e->launches++;
                return rc;
            }
            for (int r = 0; r < n; r++) {
                sp.pv[r] = e->comm->peer_v[r];
                sp.pe[r] = e->comm->peer_e[r];
                sp.peer_flag[r] = (r == me) ? nullptr : &e->comm->p2p->ctl[r]->flagL[me];
                for (size_t i = 0; i < steps.size(); i++) {
                    const PlannedStep &ps = steps[i];
                    auto it = e->comm->peer_segs[r].find(SegKey(0, ps.pid, ps.dir));
                    if (it == e->comm->peer_segs[r].end() || it->second.num_buckets == 0) {
                        // that shard has no such segment: bucket 0 belongs to another (pid, dir), whose keys never compare
                        // equal to this step's, so the probe walks that chain to its end and misses
                        sp.segr[i][r].bucket_start = 0;
                        sp.segr[i][r].fm = make_fastmod(1);
                    } else {
                        sp.segr[i][r].bucket_start = it->second.bucket_start;
                        sp.segr[i][r].fm = make_fastmod(it->second.num_buckets);
                    }
                }
            }
            sp.epoch = epoch;
            sp.nranks = (uint32_t)n;
            if (e->profiling >= 3) {
                if (!e->d_trace) CUDA_TRY(cudaMalloc((void **)&e->d_trace, LIGHT_TRACE_WORDS * sizeof(long long)));
                CUDA_TRY(cudaMemsetAsync(e->d_trace, 0, LIGHT_TRACE_WORDS * sizeof(long long), e->stream));
                lp.trace = e->d_trace;
            }
            lp.seq = ++e->seq;
            e->step = 0;
            e->recs.clear();
            e->event_next = 0;
            light_sharded_kernel<<<1, LIGHT_SHARDED_THREADS, 0, e->stream>>>(sp);
            CUDA_TRY(cudaGetLastError());
            if (e->profiling) { cudaEventRecord(e->q_ev1, e->stream); e->q_timed = true; }
            e->launches++;
            RecView rv;
            rc = wait_record(e, lp.seq, (int)steps.size(), want_table ? (int)proj_cols.size() : 0, rv);
            if (rc) return rc;
            if (rv.status & 1u) return WK_ERR_RBUF_OVERFLOW;
            if (rv.resume == (int)steps.size()) {
                const uint64_t rows = rv.rows;
                const int cols = (want_table && rows > 0) ? nrequired : final_cols;
                if (out_rows) *out_rows = rows;
                if (out_cols) *out_cols = cols;
                if (no_required && rows > 0) return WK_NO_REQUIRED_VAR;
                if (want_table && rows > 0 && table) {
                    const uint64_t words = rows * (uint64_t)cols;
                    if (words > cap_words) return WK_ERR_BAD_ARG;
                    memcpy(table, e->h_stage, words * sizeof(uint32_t));
                }
                return WK_SUCCESS;
            }
            // outgrew shared memory: every peer has been told; fall through to the collective plan
        } else {
            rc = reset_ctl(e);
            if (rc) return rc;
            p2p_light_wait_kernel<<<1, 1, 0, e->stream>>>(e->comm->d_xctl, owner, epoch, &e->d_ctl->status);
            CUDA_TRY(cudaGetLastError());
            e->launches++;
            const uint64_t seq = ++e->seq;
            finish_kernel<<<1, 1, 0, e->stream>>>(&e->d_ctl->counts[0], &e->d_ctl->status, e->d_rec, seq, 0);
            CUDA_TRY(cudaGetLastError());
            if (e->profiling) { cudaEventRecord(e->q_ev1, e->stream); e->q_timed = true; }
            e->launches++;
            RecView rv;
            rc = wait_record(e, seq, -1, 0, rv);
            if (rc) return rc;
            if (rv.status & 2u) { e->comm->poisoned = true; return WK_ERR_COMM; }
            if (!(rv.status & 4u)) {   // answered by the owner: this shard contributes no rows
                if (out_rows) *out_rows = 0;
                if (out_cols) *out_cols = want_table ? nrequired : final_cols;
                return WK_SUCCESS;
            }
        }
        if (e->profiling) CUDA_TRY(cudaEventRecord(e->q_ev0, e->stream));
    }
    rc = reset_ctl(e);
    if (rc) return rc;
    e->ncols = 0;
    for (size_t i = 0; i < steps.size(); i++) {
        const PlannedStep &ps = steps[i];
        if (ex[i] != -1) {
            rc = e->comm->p2p_ready ? exchange_table_p2p(e, ex[i]) : exchange_table(e, ex[i], nullptr);
            if (rc) return rc;
        }
        if (ps.kind == KIND_I2U) {
            rc = enqueue_seed(e, KIND_I2U, 0, ps.pid, ps.dir, mt_tid, mt_factor);   // this shard's slice of the index
        } else if (ps.kind == KIND_C2U) {
            if ((int)(ps.vid % (uint64_t)n) == me) {
                rc = enqueue_seed(e, KIND_C2U, ps.vid, ps.pid, ps.dir, 0, 1);       // the constant's owner (proxy.hpp:205)
            } else {   // empty 1-column table on the other shards
                rc = ensure_step_room(e);
                if (!rc) { e->step += 1; e->ncols = 1; }
            }
        } else if ((ps.kind == KIND_K2K || ps.kind == KIND_K2C) && e->fuse_filters && e->variant >= 4) {
            // consecutive filters with no exchange between them start from the same (local) column: one launch
            size_t j = i + 1;
            while (j < steps.size() && j - i < MAX_CHAIN && (steps[j].kind == KIND_K2K || steps[j].kind == KIND_K2C) && ex[j] == -1) j++;
            rc = enqueue_filter_chain(e, steps, i, j, nullptr);
            i = j - 1;
        } else {
            rc = enqueue_known(e, ps.kind, ps.col_start, ps.pid, ps.dir, ps.col_end, ps.end_const);
        }
        if (rc) return rc;
    }
    if (want_table) {
        rc = enqueue_project(e, proj_cols.data(), nrequired);
        if (rc) return rc;
    }
    uint64_t rows = 0;
    rc = sync_rows(e, &rows, e->profiling ? e->q_ev1 : nullptr);
    if (rc == WK_ERR_COMM) e->comm->poisoned = true;
    if (rc) return rc;
    if (e->profiling) e->q_timed = true;
    // the device is idle again: bring this shard's light-query server back while the result is copied out
    if (e->srv.enabled && e->srv.launch_id != 0 && srv_usable(e) && e->comm->peer_stores && e->comm->d_segr_tab) {
        rc = srv_ensure_running(e, e->srv.seq + 1, true);
        if (rc) return rc;
    }
    const int cols = want_table ? nrequired : final_cols;
    if (out_rows) *out_rows = rows;
    if (out_cols) *out_cols = cols;
    if (no_required && rows > 0) return WK_NO_REQUIRED_VAR;
    if (want_table && rows > 0 && table) {
        const uint64_t words = rows * (uint64_t)cols;
        if (words > cap_words) return WK_ERR_BAD_ARG;
        CUDA_TRY(cudaMemcpyAsync(table, e->buf[e->step & 1], words * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    return WK_SUCCESS;
}

// ---- self-test hooks (host-side arithmetic shared with the kernels; callable without a GPU) ----------
uint64_t wk_selftest_hash(uint64_t key) { return hash_u64(key); }
uint64_t wk_selftest_fastmod(uint64_t n, uint64_t d) { FastMod f = make_fastmod(d); return fastmod(n, f); }
uint64_t wk_selftest_make_key(uint64_t vid, uint32_t pid, uint32_t dir) { return make_key(vid, pid, dir); }
uint64_t wk_selftest_ptr_size(uint64_t raw) { return ptr_size(raw); }
uint64_t wk_selftest_ptr_off(uint64_t raw) { return ptr_off(raw); }
// owner of a row in the exchange's push kernel: x % n by multiply-shift (wk_sharded.cuh), with the magic the host passes
uint64_t wk_selftest_owner(uint64_t x, uint64_t n) {
    if (n <= 1) return 0;
    return mod_small((uint32_t)x, (uint32_t)n, (uint32_t)(((1ull << 32) + n - 1) / n));
}

}  // extern "C"

// With lazy module loading (the CUDA 12 default) the first launch of a kernel loads it, and loading may wait for the device
// to drain.  Two places cannot afford that: ranks of one process whose exchange kernels wait for each other (a rank that
// blocks in a load while its peer's kernel spins for it is a deadlock until the barrier times out), and the resident
// light-query server (every first launch of another kernel would wait for the server to idle out).  Touch every kernel of
// this translation unit once per device instead.
static int preload_kernels(wk_engine *e) {
    static bool done[64] = {false};
    const int dev = e->store->device;
    if (dev >= 0 && dev < 64 && done[dev]) return WK_SUCCESS;
    std::vector<const void *> fns;
    for (int m = 0; m < 3; m++)
        for (int C = 0; C <= 4; C++) fns.push_back((const void *)step_kernel_fn(m, e->variant, C == 0 ? 5 : C));
    fns.push_back((const void *)expand_heavy_kernel<0>);
    fns.push_back((const void *)expand_heavy_kernel<1>);
    fns.push_back((const void *)expand_heavy_kernel<2>);
    fns.push_back((const void *)expand_heavy_kernel<3>);
    const void *rest[] = {(const void *)seed_kernel, (const void *)seed_bulk_kernel, (const void *)project_kernel, (const void *)list_probe_kernel,
                          (const void *)list_clear_kernel, (const void *)list_insert_kernel, (const void *)list_filter_kernel,
                          (const void *)set_count_kernel, (const void *)rebase_kernel, (const void *)finish_kernel, (const void *)flush_read_kernel,
                          (const void *)part_count_kernel, (const void *)dup_counts_kernel, (const void *)part_scan_kernel,
                          (const void *)part_scatter_kernel, (const void *)p2p_ready_kernel, (const void *)p2p_push_kernel<1>,
                          (const void *)p2p_push_kernel<2>, (const void *)p2p_push_kernel<4>, (const void *)p2p_light_wait_kernel,
                          (const void *)p2p_light_verdict_kernel, (const void *)p2p_wait_kernel, (const void *)light_query_kernel,
                          (const void *)light_sharded_kernel, (const void *)light_batch_kernel, (const void *)light_server_kernel<LIGHT_SRV_THREADS, true>,
                          (const void *)light_server_kernel<256, true>, (const void *)light_server_kernel<256, false>, (const void *)light_server_kernel<512, true>,
                          (const void *)light_server_sharded_kernel};
    for (const void *f : rest) fns.push_back(f);
    for (const void *f : fns) {
        cudaFuncAttributes a;
        CUDA_TRY(cudaFuncGetAttributes(&a, f));
    }
    if (dev >= 0 && dev < 64) done[dev] = true;
    return WK_SUCCESS;
}
