// Device-side building blocks of the frontier-expansion engine (sm_90a).
//
// Semantics follow the reference's probe (store/gstore.hpp:242-248, 341-361, 393-410) and key
// layout (store/vertex.hpp:47-66, 116-119); the implementation is an H100-first design:
//   * a bucket is 8 x 16 B = 128 B = one L2/HBM line: 8 lanes fetch it with one LDG.128 each
//     (one wavefront per probe), 4 probes per warp instruction, 8 instructions in flight per warp;
//   * the per-segment modulo is a multiply-shift (no 64-bit division on the device);
//   * tables are staged per 256-row tile in shared memory, output space is claimed per tile with
//     one 64-bit atomic, rows are written with coalesced stores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wk_layout.cuh"

namespace wk {

// ---- n % d for a launch-invariant d (round-up multiply-shift with 65-bit magic) --------------
struct FastMod {
    uint64_t magic;
    uint64_t d;
    uint32_t shift;
    uint32_t _pad;
};

__host__ __device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * (unsigned __int128)b) >> 64);
#endif
}

inline FastMod make_fastmod(uint64_t d) {
    FastMod f;
    f.d = d;
    f._pad = 0;
    if (d <= 1) { f.magic = 0; f.shift = 0; return f; }   // n % 1 == 0, handled in fastmod()
    const uint32_t fl = 63u - (uint32_t)__builtin_clzll(d);
    if ((d & (d - 1)) == 0) {
        f.magic = 0;
        f.shift = fl - 1;
    } else {
        const unsigned __int128 num = (unsigned __int128)1 << (64 + fl);
        uint64_t m = (uint64_t)(num / d);
        const uint64_t rem = (uint64_t)(num % d);
        m += m;
        const uint64_t twice_rem = rem + rem;
        if (twice_rem >= d || twice_rem < rem) m += 1;
        f.magic = m + 1;
        f.shift = fl;
    }
    return f;
}

__host__ __device__ __forceinline__ uint64_t fastmod(uint64_t n, const FastMod &f) {
    if (f.d <= 1) return 0;
    const uint64_t q0 = mulhi64(f.magic, n);
    const uint64_t t = ((n - q0) >> 1) + q0;
    const uint64_t q = t >> f.shift;
    return n - q * f.d;
}

// ---- memory access helpers --------------------------------------------------------------------
// store arrays are immutable while an engine runs: read-only (non-coherent) path
__device__ __forceinline__ uint4 ld_slot(const uint4 *p) { return __ldg(p); }
__device__ __forceinline__ uint32_t ld_edge(const uint32_t *p) { return __ldg(p); }
// binding tables are rewritten by every step (and re-read inside the fused light kernel):
// read them through L2 only so that no stale L1 line can ever be observed
__device__ __forceinline__ uint32_t ld_table(const uint32_t *p) { return __ldcg(p); }
__device__ __forceinline__ uint64_t ld_count(const uint64_t *p) { return __ldcg((const unsigned long long *)p); }

__device__ __forceinline__ void flush_stats(uint64_t *stats, uint64_t visited, uint64_t edges) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        visited += __shfl_down_sync(0xFFFFFFFFu, visited, o);
        edges += __shfl_down_sync(0xFFFFFFFFu, edges, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (visited) atomicAdd((unsigned long long *)&stats[0], (unsigned long long)visited);
        if (edges) atomicAdd((unsigned long long *)&stats[1], (unsigned long long)edges);
    }
}

// ---- per-step parameters (passed by value) ---------------------------------------------------
enum { MODE_K2U = 0, MODE_K2K = 1, MODE_K2C = 2 };
enum { TILE_ROWS = 256, CTA_THREADS = 256, MAX_COLS = 32 };
static constexpr uint32_t BUCKET_NONE = 0xFFFFFFFFu;
static constexpr int SMALL_DEG = 8;       // rows with <= SMALL_DEG outputs are written by their owner thread
static constexpr int SERIAL_SCAN = 32;    // filter edge lists up to this length are scanned by the owner thread

struct SegParam {
    uint64_t bucket_start;
    FastMod fm;          // % num_buckets
    uint32_t pid, dir;
    uint32_t index_mode; // 1: key = [0 | cur | dir] (type-index lookup of a known vertex)
    uint32_t _pad;
};

struct StepParam {
    const uint4 *vertices;
    const uint32_t *edges;
    const uint32_t *in;
    uint32_t *out;
    const uint64_t *in_count;
    uint64_t *out_count;
    uint64_t out_cap_rows;
    uint64_t *stats;      // [0] buckets visited, [1] edges touched
    uint32_t *status;     // sticky error word
    SegParam seg;
    int32_t C;            // input columns
    int32_t col_start, col_end;
    uint32_t end_const;
    uint32_t inv_c;       // ceil(2^20 / C) for idx -> (row, col)
    uint32_t hq_cap;      // capacity of the heavy-tile queue (0 = disabled)
    struct HeavyTile *hq; // tiles whose fan-out is expanded by expand_heavy_kernel (skewed degrees)
    uint64_t *hq_packed;  // entries:24 | chunks:40, one atomic keeps both consistent
    uint64_t *hq_ticket;
    // fused filter chain: a run of consecutive known_to_known / known_to_const steps is ONE launch.  The first filter runs
    // through the pipelined probe; a row that passes it is tested against the others by its owner thread, so a row is
    // staged once, the intermediate tables are never written and the tile claims its output space once.
    int32_t nextra;
    // final_process fused into the LAST step of a non-blind plan: the projected row (sparql.hpp:1507-1550) is written
    // straight to `out`, which is then the caller's pinned host buffer (zero-copy over PCIe): no separate projection pass,
    // no device-to-host copy after the kernel.  proj_cols[j] == C names the column this step appends.
    int32_t proj_n;                // 0: write whole rows to the device table
    int8_t proj_cols[MAX_COLS];
    struct ExtraFilter {
        SegParam seg;
        int32_t col_start, col_end;   // col_end < 0: known_to_const against end_const
        uint32_t end_const, _pad;
    } extra[3];
};
enum { MAX_CHAIN = 4 };   // filters per launch: the pipelined one + 3

// A tile with a large total fan-out is not expanded in place: it only claims its output range and leaves
// this descriptor; expand_heavy_kernel then spreads its output rows over the whole grid in equal chunks.
enum { HEAVY_TILE_MIN = 4096, HEAVY_CHUNK = 8192 };
struct HeavyTile {
    uint64_t row0, base, total, chunk_base;
    uint32_t nrows, _pad;
    uint64_t pre[TILE_ROWS];   // exclusive prefix of the multiplicities inside the tile
    uint64_t off[TILE_ROWS];   // edge offset of every row
};

__device__ __forceinline__ uint64_t step_key(const SegParam &s, uint32_t cur) {
    // index_mode: the reference builds ikey_t(0, cur, d) whose 17-bit pid bitfield truncates cur
    // (vertex.hpp:47-60); mask the same way so an out-of-range id can never alias a vid field
    return s.index_mode ? make_key(0, cur & ((1u << 17) - 1), s.dir) : make_key(cur, s.pid, s.dir);
}

// shared-memory working set of one tile
struct TileSmem {
    uint64_t key[TILE_ROWS];      // raw ikey_t each row probes for
    uint32_t bucket[TILE_ROWS];
    uint32_t next[TILE_ROWS];
    uint64_t ptr[TILE_ROWS];
    uint64_t wsum[CTA_THREADS / 32];
    uint64_t base;
    uint64_t total;
};

// ---- cooperative cluster-hash probe of one warp's 32 rows ------------------------------------
// Before the call: sm.bucket[row] = first bucket (BUCKET_NONE for inactive rows), sm.key[row] =
// the probed key, sm.ptr[row] = 0, sm.next[row] = 0, followed by __syncwarp().
// After the call sm.ptr[row] holds the raw iptr_t of the key (0 = miss).  Returns the number of
// buckets this lane's own row visited (L_i).
template <int BATCH>   // buckets fetched per lane before the first compare: 8, 4 or 2 (register/MLP trade-off)
__device__ __forceinline__ uint32_t warp_probe(const uint4 *__restrict__ vertices, TileSmem &sm, int warp_row0,
                                               int lane, bool active) {
    const int slot = lane & 7;
    const int grp = lane >> 3;
    const int my_row = warp_row0 + lane;
    bool pending = active;
    uint32_t visited = 0;
    while (true) {
#pragma unroll 1
        for (int part = 0; part < 8 / BATCH; part++) {
            const int rbase = warp_row0 + part * (4 * BATCH);
            uint32_t b[BATCH];
            uint4 v[BATCH];
#pragma unroll
            for (int r = 0; r < BATCH; r++) b[r] = sm.bucket[rbase + 4 * r + grp];
#pragma unroll
            for (int r = 0; r < BATCH; r++) {
                v[r] = make_uint4(0, 0, 0, 0);
                if (b[r] != BUCKET_NONE) v[r] = ld_slot(vertices + ((uint64_t)b[r] * 8 + slot));
            }
#pragma unroll
            for (int r = 0; r < BATCH; r++) {
                if (b[r] != BUCKET_NONE) {
                    const int j = rbase + 4 * r + grp;
                    const uint64_t kk = (uint64_t)v[r].x | ((uint64_t)v[r].y << 32);
                    if (slot < 7) {
                        if (kk == sm.key[j]) sm.ptr[j] = (uint64_t)v[r].z | ((uint64_t)v[r].w << 32);
                    } else {
                        // last slot: key.vid is the next bucket of the chain (0 / empty key = end)
                        sm.next[j] = (uint32_t)(kk >> WK_KEY_VID_SHIFT);
                    }
                }
            }
        }
        __syncwarp();
        if (pending) {
            visited++;
            if (sm.ptr[my_row] != 0) pending = false;
            else if (sm.next[my_row] == 0) pending = false;   // miss
            else { sm.bucket[my_row] = sm.next[my_row]; sm.next[my_row] = 0; }
        }
        if (!pending) sm.bucket[my_row] = BUCKET_NONE;
        const bool more = __any_sync(0xFFFFFFFFu, pending);
        __syncwarp();
        if (!more) break;
    }
    return visited;
}

// Block-wide exclusive scan of the per-row multiplicities + output-space claim for the tile.
// Returns the row's exclusive prefix; sm.total = tile total, sm.base = first output row of the tile
// (~0 when the result buffer would overflow: counted, flagged, not written).
__device__ __forceinline__ uint64_t tile_scan_and_claim(uint32_t mult, TileSmem &sm, int tid, const StepParam &p) {
    const int lane = tid & 31, warp = tid >> 5;
    uint64_t incl;
    // a warp whose 32 multiplicities cannot overflow 32 bits (always, except 2^27-edge hubs) scans in 32 bits
    if (__all_sync(0xFFFFFFFFu, mult < (1u << 26))) {
        uint32_t x = mult;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if (lane >= o) x += y;
        }
        incl = x;
    } else {
        uint64_t x = mult;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if (lane >= o) x += y;
        }
        incl = x;
    }
    if (lane == 31) sm.wsum[warp] = incl;
    __syncthreads();
    uint64_t woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < CTA_THREADS / 32; w++) {
        const uint64_t s = sm.wsum[w];
        if (w < warp) woff += s;
        tot += s;
    }
    if (tid == 0) {
        uint64_t base = 0;
        if (tot) base = atomicAdd((unsigned long long *)p.out_count, (unsigned long long)tot);
        if (base + tot > p.out_cap_rows) {
            atomicOr(p.status, 1u);   // WK_ERR_RBUF_OVERFLOW
            base = ~0ull;
        }
        sm.base = base;
        sm.total = tot;
    }
    __syncthreads();
    return woff + incl - mult;
}

template <int CT>
__device__ __forceinline__ void copy_row(uint32_t *__restrict__ dst, const uint32_t *__restrict__ srow, int C) {
    if (CT > 0) {
#pragma unroll
        for (int c = 0; c < CT; c++) dst[c] = srow[c];
    } else {
        for (int c = 0; c < C; c++) dst[c] = srow[c];
    }
}

// ---- one 256-row tile of a known_to_{unknown,known,const} step --------------------------------
// rows: dynamic shared memory, TILE_ROWS x CP words (CP = C | 1 to spread banks).
// CT > 0: the column count is a compile-time constant (C = 1..4 get their own instantiation).
template <int MODE, int BATCH, int CT>
__device__ __forceinline__ void process_tile(const StepParam &p, uint64_t row0, uint32_t nrows, TileSmem &sm,
                                             uint32_t *rows, uint64_t &acc_visited, uint64_t &acc_edges) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int C = CT > 0 ? CT : p.C;
    const int CP = C | 1;
    const int Cout = (MODE == MODE_K2U) ? C + 1 : C;

    // A. stage the tile's input rows (coalesced, L2-only loads)
    {
        const uint32_t nwords = nrows * (uint32_t)C;
        const uint32_t *src = p.in + row0 * (uint64_t)C;
        for (uint32_t idx = tid; idx < nwords; idx += CTA_THREADS) {
            const uint32_t r = CT > 0 ? idx / (uint32_t)C : (uint32_t)(((uint64_t)idx * p.inv_c) >> 20);
            const uint32_t c = idx - r * (uint32_t)C;
            rows[r * CP + c] = ld_table(src + idx);
        }
    }
    __syncthreads();

    // B. key -> first bucket
    const bool active = (uint32_t)tid < nrows;
    const uint32_t *myrow = rows + tid * CP;
    {
        uint64_t key = 0;
        uint32_t bucket = BUCKET_NONE;
        if (active) {
            key = step_key(p.seg, myrow[p.col_start]);
            bucket = (uint32_t)(p.seg.bucket_start + fastmod(hash_u64(key), p.seg.fm));
        }
        sm.key[tid] = key;
        sm.bucket[tid] = bucket;
        sm.ptr[tid] = 0;
        sm.next[tid] = 0;
    }
    __syncwarp();

    // C. probe
    acc_visited += warp_probe<BATCH>(p.vertices, sm, warp * 32, lane, active);

    // D. multiplicity of each row
    const uint64_t ptr = sm.ptr[tid];
    const uint32_t size = active ? ptr_size(ptr) : 0;
    const uint64_t off = ptr_off(ptr);
    uint32_t mult = 0;
    uint32_t e0 = 0;   // K2U: first edge, fetched while the tile's output space is being claimed
    if (MODE == MODE_K2U) {
        mult = size;
        acc_edges += size;
        if (size != 0 && size <= SMALL_DEG) e0 = ld_edge(p.edges + off);
    } else {
        const uint32_t target = (MODE == MODE_K2K) ? (active ? myrow[p.col_end] : 0) : p.end_const;
        bool found = false;
        if (size <= SERIAL_SCAN) {
            uint32_t k = 0;
            for (; k < size; k++)
                if (ld_edge(p.edges + off + k) == target) { found = true; break; }
            acc_edges += found ? (k + 1) : size;
        }
        // long lists: the whole warp scans one list at a time (coalesced, early exit)
        uint32_t longmask = __ballot_sync(0xFFFFFFFFu, size > SERIAL_SCAN);
        while (longmask) {
            const int src = __ffs(longmask) - 1;
            longmask &= longmask - 1;
            const uint32_t s_size = __shfl_sync(0xFFFFFFFFu, size, src);
            const uint64_t s_off = __shfl_sync(0xFFFFFFFFu, off, src);
            const uint32_t s_target = __shfl_sync(0xFFFFFFFFu, target, src);
            uint32_t scanned = s_size;
            bool hit = false;
            for (uint32_t k0 = 0; k0 < s_size; k0 += 32) {
                const uint32_t k = k0 + lane;
                const bool eq = (k < s_size) && (ld_edge(p.edges + s_off + k) == s_target);
                const uint32_t m = __ballot_sync(0xFFFFFFFFu, eq);
                if (m) { hit = true; scanned = k0 + __ffs(m); break; }
            }
            if (lane == src) { found = hit; acc_edges += scanned; }
        }
        mult = found ? 1u : 0u;
    }

    // E. claim output space for the tile (one 64-bit atomic per tile)
    const uint64_t excl = tile_scan_and_claim(mult, sm, tid, p);
    const uint64_t base = sm.base;

    // F. write the output rows
    if (base != ~0ull && sm.total != 0) {
        if (MODE != MODE_K2U) {
            if (mult) copy_row<CT>(p.out + (base + excl) * (uint64_t)Cout, myrow, C);
        } else {
            // small fan-out: the owner thread writes its rows
            if (mult != 0 && mult <= SMALL_DEG) {
                uint32_t *dst = p.out + (base + excl) * (uint64_t)Cout;
                copy_row<CT>(dst, myrow, C);
                dst[C] = e0;
                for (uint32_t k = 1; k < mult; k++) {
                    dst += Cout;
                    const uint32_t e = ld_edge(p.edges + off + k);
                    copy_row<CT>(dst, myrow, C);
                    dst[C] = e;
                }
            }
            // larger fan-out: the warp cooperates on one source row at a time; consecutive lanes
            // write consecutive output words (coalesced) and read consecutive edges
            uint32_t bigmask = __ballot_sync(0xFFFFFFFFu, mult > SMALL_DEG);
            while (bigmask) {
                const int src = __ffs(bigmask) - 1;
                bigmask &= bigmask - 1;
                const uint32_t s_mult = __shfl_sync(0xFFFFFFFFu, mult, src);
                const uint64_t s_off = __shfl_sync(0xFFFFFFFFu, off, src);
                const uint64_t s_excl = __shfl_sync(0xFFFFFFFFu, excl, src);
                const uint32_t *srow = rows + (warp * 32 + src) * CP;
                uint32_t *dst = p.out + (base + s_excl) * (uint64_t)Cout;
                const uint64_t nwords = (uint64_t)s_mult * (uint64_t)Cout;
                // word w of the run: row = w / Cout, col = w % Cout, advanced incrementally
                uint32_t r = (uint32_t)lane / (uint32_t)Cout;
                uint32_t c = (uint32_t)lane - r * (uint32_t)Cout;
                const uint32_t dr = 32u / (uint32_t)Cout, dc = 32u - dr * (uint32_t)Cout;
                for (uint64_t w = lane; w < nwords; w += 32) {
                    dst[w] = (c == (uint32_t)C) ? ld_edge(p.edges + s_off + r) : srow[c];
                    r += dr;
                    c += dc;
                    if (c >= (uint32_t)Cout) { c -= (uint32_t)Cout; r++; }
                }
            }
        }
    }
    __syncthreads();   // smem is reused by the next tile
}


// =============================================================================================
// Asynchronous staging (cp.async / LDGSTS) + owner-thread bucket scan: building blocks of the v5 pipeline
//
//  * each bucket (128 B) is fetched by 8 lanes with one 16-byte cp.async each (one L1 wavefront per
//    probe, no registers held while the loads are in flight) into a per-warp staging area whose
//    16-byte chunks are XOR-swizzled by the row number,
//  * the row's owner thread then scans its 7 keys from shared memory: one warp instruction covers
//    32 rows (the register-staged variant above covers 4), which is what matters once the kernel is
//    instruction-issue bound,
//  * rare chain hops (a few % of the rows) are walked by the owner thread straight from global.
// =============================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct TileSmem4 {
    uint64_t wsum[CTA_THREADS / 32];
    uint64_t base;
    uint64_t total;
    uint64_t qidx;                        // heavy-queue slot of this tile (~0: expand in place)
    uint64_t pre[CTA_THREADS / 32][32];   // per warp: exclusive prefix of the 32 multiplicities (balanced expand)
    uint64_t off[CTA_THREADS / 32][32];   // per warp: edge offsets of the 32 rows
};
enum { BKT_BYTES = TILE_ROWS * 128 };   // bucket staging area of one CTA

// thread-serial walk of a bucket chain from global memory (slow path: only rows whose first
// bucket neither holds the key nor ends the chain)
__device__ __noinline__ uint64_t chain_walk(const uint4 *__restrict__ vertices, uint64_t key, uint64_t bucket,
                                            uint32_t &visited) {
    while (true) {
        const uint4 *b = vertices + bucket * 8;
        visited++;
        uint64_t found = 0;
#pragma unroll
        for (int i = 0; i < 7; i++) {
            const uint4 v = ld_slot(b + i);
            const uint64_t kk = (uint64_t)v.x | ((uint64_t)v.y << 32);
            if (kk == key) found = (uint64_t)v.z | ((uint64_t)v.w << 32);
        }
        if (found) return found;
        const uint4 v7 = ld_slot(b + 7);
        const uint64_t chain = (uint64_t)v7.x | ((uint64_t)v7.y << 32);
        if (chain == 0) return 0;
        bucket = chain >> WK_KEY_VID_SHIFT;
    }
}

// =============================================================================================
// v5: warp-autonomous software pipeline.  Each warp stages only its own 32 rows of a tile (triple
// buffered) and its own 32 buckets, so the only CTA-wide synchronisation left is the scan/claim;
// the buckets of tile t+1 are already in flight while tile t fetches edges, claims space and writes.
//   cp.async groups of a warp, oldest first, at the top of an iteration:  B(t), R(t+1)
// =============================================================================================
__device__ __forceinline__ void stage_warp_rows(const uint32_t *__restrict__ in, uint64_t row0w, uint32_t n, int C,
                                                uint32_t *dst, int lane) {
    const uint32_t nwords = n * (uint32_t)C;
    const uint32_t *src = in + row0w * (uint64_t)C;   // 16-byte aligned: row0w is a multiple of 32
    const uint32_t nvec = nwords >> 2;
    const uint32_t d0 = smem_u32(dst);
    for (uint32_t i = lane; i < nvec; i += 32) cp_async16(d0 + i * 16, src + i * 4);
    const uint32_t tail = nwords & 3u;
    if ((uint32_t)lane < tail) cp_async4(d0 + (nvec * 4 + lane) * 4, src + nvec * 4 + lane);
}

// membership test over a short edge list with 8 independent loads in flight per round
__device__ __forceinline__ bool list_contains8(const uint32_t *__restrict__ e, uint32_t size, uint32_t target,
                                               uint32_t &scanned) {
    for (uint32_t k0 = 0; k0 < size; k0 += 8) {
        uint32_t x[8];
#pragma unroll
        for (int j = 0; j < 8; j++) x[j] = (k0 + j < size) ? ld_edge(e + k0 + j) : 0u;
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (k0 + j < size && x[j] == target) { scanned = k0 + j + 1; return true; }
    }
    scanned = size;
    return false;
}

// one output row: the input row (+ the new edge for known_to_unknown), or its projection when PROJ
template <int MODE, int CT, bool PROJ>
__device__ __forceinline__ void emit_row(const StepParam &p, uint64_t orow, const uint32_t *srow, int C, uint32_t e) {
    if (!PROJ) {
        uint32_t *dst = p.out + orow * (uint64_t)(MODE == MODE_K2U ? C + 1 : C);
        copy_row<CT>(dst, srow, C);
        if (MODE == MODE_K2U) dst[C] = e;
    } else {
        uint32_t *dst = p.out + orow * (uint64_t)p.proj_n;
        for (int j = 0; j < p.proj_n; j++) {
            const int c = p.proj_cols[j];
            dst[j] = (MODE == MODE_K2U && c == C) ? e : srow[c];
        }
    }
}

template <int MODE, int CT, bool PROJ = false>
__device__ __forceinline__ void step_body_v5(const StepParam &p, uint64_t N, TileSmem4 &sm, unsigned char *dyn) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int C = CT > 0 ? CT : p.C;
    const uint32_t rowbytes = 128u * (uint32_t)C;                    // 32 rows x C words
    unsigned char *bkt = dyn + warp * (32 * 128);                    // this warp's bucket staging area
    unsigned char *rows_base = dyn + BKT_BYTES + (uint32_t)warp * 3u * rowbytes;
    const uint64_t stride = gridDim.x;
    uint64_t tile = blockIdx.x;
    uint64_t acc_visited = 0, acc_edges = 0;
    if (tile * TILE_ROWS >= N) { flush_stats(p.stats, 0, 0); return; }

    auto warp_n = [&](uint64_t t) -> uint32_t {
        const uint64_t r0 = t * TILE_ROWS + (uint64_t)warp * 32;
        return r0 >= N ? 0u : (uint32_t)((N - r0 < 32) ? (N - r0) : 32);
    };
    auto rows_buf = [&](uint32_t k) -> uint32_t * { return (uint32_t *)(rows_base + (k % 3u) * rowbytes); };
    auto issue_buckets = [&](uint32_t bucket) {
        const int slot = lane & 7, grp = lane >> 3;
        const uint32_t wbase = smem_u32(bkt);
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int j = 4 * r + grp;
            const uint32_t b = __shfl_sync(0xFFFFFFFFu, bucket, j);
            if (b != BUCKET_NONE)
                cp_async16(wbase + (uint32_t)j * 128 + (uint32_t)((slot ^ (j & 7)) << 4), p.vertices + ((uint64_t)b * 8 + slot));
        }
    };

    // ---- prologue: rows(t0) -> keys -> B(t0); R(t0+1) ---------------------------------------------
    uint32_t it = 0;
    uint32_t n_cur = warp_n(tile);
    stage_warp_rows(p.in, tile * TILE_ROWS + (uint64_t)warp * 32, n_cur, C, rows_buf(0), lane);
    cp_async_commit();
    cp_async_wait<0>();
    __syncwarp();
    uint64_t key = 0;
    {
        uint32_t bucket = BUCKET_NONE;
        if ((uint32_t)lane < n_cur) {
            key = step_key(p.seg, rows_buf(0)[lane * C + p.col_start]);
            bucket = (uint32_t)(p.seg.bucket_start + fastmod(hash_u64(key), p.seg.fm));
        }
        issue_buckets(bucket);
        cp_async_commit();
    }
    {
        const uint64_t t1 = tile + stride;
        stage_warp_rows(p.in, t1 * TILE_ROWS + (uint64_t)warp * 32, warp_n(t1), C, rows_buf(1), lane);
        cp_async_commit();
    }

    for (; tile * TILE_ROWS < N; tile += stride, it++) {
        const bool active = (uint32_t)lane < n_cur;
        const uint32_t *rows = rows_buf(it);
        const uint32_t *myrow = rows + lane * C;

        // 1. buckets of this tile (issued one iteration ago)
        cp_async_wait<1>();
        __syncwarp();

        // 2. owner thread scans its bucket in shared memory
        uint64_t ptr = 0;
        if (active) {
            const unsigned char *mb = bkt + lane * 128;
            const int sw = lane & 7;
            int hit = -1;
#pragma unroll
            for (int i = 0; i < 7; i++) {
                const uint64_t kk = *(const uint64_t *)(mb + ((i ^ sw) << 4));
                if (kk == key) hit = i;
            }
            uint32_t visited = 1;
            if (hit >= 0) {
                ptr = *(const uint64_t *)(mb + ((hit ^ sw) << 4) + 8);
            } else {
                const uint64_t chain = *(const uint64_t *)(mb + ((7 ^ sw) << 4));
                if (chain != 0) ptr = chain_walk(p.vertices, key, chain >> WK_KEY_VID_SHIFT, visited);
            }
            acc_visited += visited;
        }
        __syncwarp();   // every lane is done with the staging area before it is refilled

        // 3./4. next tile: its rows have landed -> keys -> buckets in flight during the rest of this tile
        cp_async_wait<0>();
        __syncwarp();
        const uint64_t tnext = tile + stride;
        const uint32_t n_next = warp_n(tnext);
        uint64_t key_next = 0;
        {
            uint32_t bucket = BUCKET_NONE;
            if ((uint32_t)lane < n_next) {
                key_next = step_key(p.seg, rows_buf(it + 1)[lane * C + p.col_start]);
                bucket = (uint32_t)(p.seg.bucket_start + fastmod(hash_u64(key_next), p.seg.fm));
            }
            issue_buckets(bucket);
            cp_async_commit();
        }
        // 5. rows of the tile after next (its buffer was last used by the previous tile)
        {
            const uint64_t t2 = tnext + stride;
            stage_warp_rows(p.in, t2 * TILE_ROWS + (uint64_t)warp * 32, warp_n(t2), C, rows_buf(it + 2), lane);
            cp_async_commit();
        }

        // 6a. multiplicity of each row
        const uint32_t size = active ? ptr_size(ptr) : 0;
        const uint64_t off = ptr_off(ptr);
        uint32_t mult = 0;
        uint32_t e0 = 0;
        if (MODE == MODE_K2U) {
            mult = size;
            acc_edges += size;
            if (size != 0 && size <= SMALL_DEG) e0 = ld_edge(p.edges + off);
        } else {
            const uint32_t target = (MODE == MODE_K2K) ? (active ? myrow[p.col_end] : 0) : p.end_const;
            bool found = false;
            if (size <= SERIAL_SCAN) {
                uint32_t scanned;
                found = list_contains8(p.edges + off, size, target, scanned);
                acc_edges += scanned;
            }
            uint32_t longmask = __ballot_sync(0xFFFFFFFFu, size > SERIAL_SCAN);
            while (longmask) {
                const int src = __ffs(longmask) - 1;
                longmask &= longmask - 1;
                const uint32_t s_size = __shfl_sync(0xFFFFFFFFu, size, src);
                const uint64_t s_off = __shfl_sync(0xFFFFFFFFu, off, src);
                const uint32_t s_target = __shfl_sync(0xFFFFFFFFu, target, src);
                uint32_t scanned = s_size;
                bool hitl = false;
                for (uint32_t k0 = 0; k0 < s_size; k0 += 32) {
                    const uint32_t k = k0 + lane;
                    const bool eq = (k < s_size) && (ld_edge(p.edges + s_off + k) == s_target);
                    const uint32_t m = __ballot_sync(0xFFFFFFFFu, eq);
                    if (m) { hitl = true; scanned = k0 + __ffs(m); break; }
                }
                if (lane == src) { found = hitl; acc_edges += scanned; }
            }
            // the other filters of a fused chain, for the rows that are still alive (probe + scan by the owner thread)
            for (int f = 0; f < p.nextra && found; f++) {
                const StepParam::ExtraFilter &x = p.extra[f];
                const uint64_t k2 = step_key(x.seg, myrow[x.col_start]);
                uint32_t visited2 = 0;
                const uint64_t ptr2 = chain_walk(p.vertices, k2, x.seg.bucket_start + fastmod(hash_u64(k2), x.seg.fm), visited2);
                acc_visited += visited2;
                const uint32_t target2 = x.col_end >= 0 ? myrow[x.col_end] : x.end_const;
                uint32_t scanned2;
                found = list_contains8(p.edges + ptr_off(ptr2), ptr_size(ptr2), target2, scanned2);
                acc_edges += scanned2;
            }
            mult = found ? 1u : 0u;
        }

        // 6b. claim output space for the tile (one 64-bit atomic per tile; the only CTA-wide sync)
        uint64_t incl;
        if (__all_sync(0xFFFFFFFFu, mult < (1u << 26))) {
            uint32_t x = mult;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
                if (lane >= o) x += y;
            }
            incl = x;
        } else {
            uint64_t x = mult;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
                if (lane >= o) x += y;
            }
            incl = x;
        }
        if (lane == 31) sm.wsum[warp] = incl;
        __syncthreads();
        uint64_t woff = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < CTA_THREADS / 32; w++) {
            const uint64_t sx = sm.wsum[w];
            if (w < warp) woff += sx;
            tot += sx;
        }
        if (tid == 0) {
            uint64_t b0 = 0;
            if (tot) b0 = atomicAdd((unsigned long long *)p.out_count, (unsigned long long)tot);
            if (b0 + tot > p.out_cap_rows) {
                atomicOr(p.status, 1u);   // WK_ERR_RBUF_OVERFLOW
                b0 = ~0ull;
            }
            sm.base = b0;
            uint64_t q = ~0ull;
            if (MODE == MODE_K2U && p.hq_cap && tot >= HEAVY_TILE_MIN && b0 != ~0ull) {
                const uint64_t nchunks = (tot + HEAVY_CHUNK - 1) / HEAVY_CHUNK;
                const uint64_t pk = atomicAdd((unsigned long long *)p.hq_packed, (unsigned long long)((1ull << 40) + nchunks));
                const uint64_t idx = pk >> 40;
                if (idx < p.hq_cap) {
                    q = idx;
                    HeavyTile *ht = p.hq + idx;
                    ht->row0 = tile * TILE_ROWS;
                    ht->base = b0;
                    ht->total = tot;
                    ht->chunk_base = pk & ((1ull << 40) - 1);
                    ht->nrows = TILE_ROWS;
                }
            }
            sm.qidx = q;
        }
        __syncthreads();
        const uint64_t base = sm.base;
        const uint64_t excl = woff + incl - mult;
        const uint64_t qidx = (MODE == MODE_K2U) ? sm.qidx : ~0ull;

        // 6c. write the output rows
        if (qidx != ~0ull) {
            // skewed tile: leave the expansion to expand_heavy_kernel
            HeavyTile *ht = p.hq + qidx;
            ht->pre[tid] = excl;
            ht->off[tid] = off;
        } else if (base != ~0ull && tot != 0) {
            if (MODE != MODE_K2U) {
                if (mult) emit_row<MODE, CT, PROJ>(p, base + excl, myrow, C, 0);
            } else if (__all_sync(0xFFFFFFFFu, mult <= 1)) {
                // at most one edge per row (the common case on LUBM): the owner thread writes its row
                if (mult) emit_row<MODE, CT, PROJ>(p, base + excl, myrow, C, e0);
            } else {
                // load-balanced expand: every lane takes output rows o = lane, lane+32, ... of the warp's run and
                // finds its source row by binary search in the 32 scanned multiplicities, so skewed degrees
                // (power-law graphs, hubs) keep all lanes busy and all edge loads independent
                const uint64_t wexcl = incl - mult;                      // prefix inside the warp
                const uint64_t wtotal = __shfl_sync(0xFFFFFFFFu, incl, 31);
                uint64_t *wpre = sm.pre[warp], *woffs = sm.off[warp];
                wpre[lane] = wexcl;
                woffs[lane] = off;
                __syncwarp();
                const uint64_t orow0 = base + woff;
                for (uint64_t o0 = lane; o0 < wtotal; o0 += 64) {   // two independent outputs per lane in flight
                    int r[2];
                    uint32_t e[2];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const uint64_t o = o0 + 32 * u;
                        r[u] = 0;
                        if (o < wtotal) {
#pragma unroll
                            for (int st = 16; st > 0; st >>= 1)
                                if (wpre[r[u] + st] <= o) r[u] += st;
                            e[u] = ld_edge(p.edges + woffs[r[u]] + (o - wpre[r[u]]));
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const uint64_t o = o0 + 32 * u;
                        if (o < wtotal) emit_row<MODE, CT, PROJ>(p, orow0 + o, rows + r[u] * C, C, e[u]);
                    }
                }
            }
        }
        __syncwarp();   // rows_buf(it) may be refilled two iterations from now; keep the warp together
        key = key_next;
        n_cur = n_next;
    }
    cp_async_wait<0>();
    flush_stats(p.stats, acc_visited, acc_edges);
}

// ---- expansion of the queued heavy tiles: output-parallel, equal chunks over the whole grid ----------
template <int CT>
__device__ __forceinline__ void expand_heavy_body(const StepParam &p) {
    __shared__ uint64_t s_pre[TILE_ROWS];
    __shared__ uint64_t s_off[TILE_ROWS];
    __shared__ uint64_t s_hdr[4];   // ticket, entry, chunk
    const int tid = threadIdx.x;
    const int C = CT > 0 ? CT : p.C;
    const int Cout = C + 1;
    const uint64_t packed = ld_count(p.hq_packed);
    uint64_t count = packed >> 40;
    if (count > p.hq_cap) count = p.hq_cap;
    const uint64_t total_chunks = packed & ((1ull << 40) - 1);
    if (count == 0) return;
    uint64_t cur = ~0ull, cur_cb = 0, cur_nch = 0;   // thread 0: the entry the previous ticket fell into
    while (true) {
        if (tid == 0) {
            const uint64_t t = atomicAdd((unsigned long long *)p.hq_ticket, 1ull);
            uint64_t entry = ~0ull, chunk = 0;
            if (t < total_chunks) {
                if (cur == ~0ull || t < cur_cb || t >= cur_cb + cur_nch) {
                    // slot index and chunk_base come from one atomic, so both are monotone: binary search for the
                    // last queued entry whose chunk_base <= t
                    uint64_t lo = 0, hi = count;
                    while (hi - lo > 1) {
                        const uint64_t mid = (lo + hi) >> 1;
                        if (ld_count(&p.hq[mid].chunk_base) <= t) lo = mid; else hi = mid;
                    }
                    cur = lo;
                    cur_cb = ld_count(&p.hq[lo].chunk_base);
                    cur_nch = (ld_count(&p.hq[lo].total) + HEAVY_CHUNK - 1) / HEAVY_CHUNK;
                }
                if (t >= cur_cb && t - cur_cb < cur_nch) { entry = cur; chunk = t - cur_cb; }
                else entry = ~1ull;   // ticket of a tile that did not fit the queue and was expanded in place
            }
            s_hdr[0] = t; s_hdr[1] = entry; s_hdr[2] = chunk;
        }
        __syncthreads();
        const uint64_t t = s_hdr[0], entry = s_hdr[1], chunk = s_hdr[2];
        if (t >= total_chunks) break;
        if (entry < count) {
            const HeavyTile *ht = p.hq + entry;
            s_pre[tid] = ht->pre[tid];
            s_off[tid] = ht->off[tid];
            __syncthreads();
            const uint64_t row0 = ht->row0, base = ht->base, total = ht->total;
            const uint64_t o_end = (chunk + 1) * HEAVY_CHUNK < total ? (chunk + 1) * HEAVY_CHUNK : total;
            // 4 independent (search, edge load, row load) per thread in flight, then the stores
            for (uint64_t o0 = chunk * HEAVY_CHUNK + tid; o0 < o_end; o0 += 4 * CTA_THREADS) {
                int r[4];
                uint32_t e[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const uint64_t o = o0 + (uint64_t)u * CTA_THREADS;
                    r[u] = 0;
                    if (o < o_end) {
#pragma unroll
                        for (int st = TILE_ROWS / 2; st > 0; st >>= 1)
                            if (s_pre[r[u] + st] <= o) r[u] += st;
                        e[u] = ld_edge(p.edges + s_off[r[u]] + (o - s_pre[r[u]]));
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const uint64_t o = o0 + (uint64_t)u * CTA_THREADS;
                    if (o < o_end) {
                        uint32_t *dst = p.out + (base + o) * (uint64_t)Cout;
                        const uint32_t *src = p.in + (row0 + r[u]) * (uint64_t)C;   // read-only here: L1-cacheable
                        if (CT > 0) {
#pragma unroll
                            for (int c = 0; c < CT; c++) dst[c] = __ldg(src + c);
                        } else {
                            for (int c = 0; c < C; c++) dst[c] = __ldg(src + c);
                        }
                        dst[C] = e[u];
                    }
                }
            }
        }
        __syncthreads();
    }
}

}  // namespace wk
