// search_kernels.cuh — sm_90a kernels for granne's search path:
//   Granne::search -> find_entrypoint -> search_for_neighbors -> ElementContainer::dist_to_element
//   (reference: src/index/mod.rs:140-150, 962-1037; src/max_size_heap.rs; src/elements/*; src/math.rs)
//
// Execution model: one warp per query (one 32-thread CTA, GB_MIN_BLOCKS resident CTAs per SM, persistent over a
// work counter).  Per query the warp owns
//   * in shared memory, a sorted candidate list L that merges the reference's two heaps: `res` (bounded max-heap of
//     expanded nodes) and `pq` (unbounded min-heap frontier) — see "Exactness" below.  Fast pass (search_layer_fast):
//     split u32 arrays Ld (distance bits | expanded flag) / Li (ids), capacity 32*R; slow pass (search_layer): 64-bit
//     keys in a global-memory workspace, for the rare query whose plateau of equal distances overflows the fast list;
//   * an exact visited set (the reference's FxHashSet): fast pass = a bucketed table in global memory that stays L2
//     resident (4 ids per 16-byte bucket, one 128-bit load per neighbour, no atomics — the warp is the only writer);
//     slow pass = open addressing with CAS in the global workspace;
//   * a tile of up to 32 rows x 36 floats in shared memory used to reproduce the reference's strictly ordered 32-lane
//     partial-sum reduction, plus a staging tile for candidate rows (layout: SmemLayout).
// Candidate rows are gathered from HBM into the staging tile with per-lane cp.async (each lane copies only the bytes it
// reads back, so no cross-lane barrier is needed), all rows of a batch in flight at once; the f32 row layout in HBM is
// lane-permuted so that lane i reads its accumulator chunks with 128-bit shared loads.  The visited table uses an L2
// evict_last policy; the adjacency row of the runner-up candidate is fetched speculatively while the current
// expansion's distances are computed.
//
// Exactness (bit-identical ids AND f32 distances, identical n_dist / n_expand counters):
//   * dot_product_f32 (src/math.rs:16-42): lane i owns accumulator chunk[i]; FMA over chunks in order; the 32
//     partials are then added in lane order by ONE lane per candidate (via the smem tile), then the FMA tail.
//   * L keeps entries sorted by (distance bits, id) — the tuple order of (NotNan<f32>, usize).  Bit 63 of a key marks
//     "expanded" (popped from pq and pushed to res); distances are >= +0 so the sign bit is free.
//     Let E = expanded entries of L in order.  res == first max_search entries of E whenever |E| >= max_search;
//     otherwise res is not full or still holds entries that were evicted from L, which are >= every entry of L, and in
//     both cases the reference neither breaks nor filters anything that could later be expanded.
//     An entry may be dropped from L only if at least max_search entries with STRICTLY smaller distance remain
//     (such an entry can never be expanded nor reported).  If a drop is needed and that does not hold (a plateau of
//     equal distances wider than the slack) the query is flagged and re-run on the slow path with a global-memory
//     workspace (same code, larger capacities).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#ifndef GB_MIN_BLOCKS
#define GB_MIN_BLOCKS 24  // resident one-warp CTAs per SM the fast kernel is register-limited to (tuning knob)
#endif
#ifndef GB_STG_BYTES
#define GB_STG_BYTES 4096  // staging tile per warp for gathered candidate rows (tuning knob)
#endif

namespace granne_b200 {

constexpr int kMaxLayers = 24;
constexpr uint32_t kUnusedId = 0xFFFFFFFFu;
constexpr unsigned long long kFlagExpanded = 1ull << 63;
constexpr unsigned long long kKeyMask = ~kFlagExpanded;
constexpr unsigned kFullMask = 0xFFFFFFFFu;
constexpr int kTileStride = 36;  // floats per tile row: 16-byte aligned rows, conflict-free LDS.128 per quarter warp
// per-warp scratch behind the tile: 32 x u32 compacted candidate ids | 2 x 32 u32 speculative adjacency rows |
// 32 x 16-byte speculative visited buckets.  The 32 x (id, distance bits) keys of a merge are parked in the tile itself
// (idle outside the distance phase), which is therefore at least 256 bytes.
constexpr int kIdScratchBytes = 896;
__host__ __device__ constexpr uint32_t tile_bytes_for_rows(uint32_t rows) {
    return (rows * kTileStride * 4u < 256u ? 256u : rows * kTileStride * 4u) + kIdScratchBytes;
}

enum ElementKind : int { kAngularF32 = 0, kAngularI8 = 1, kSumEmbeddings = 2 };
enum QueryFormat : int { kQueryRawF32 = 0, kQueryElement = 1, kQueryById = 2 };  // ById: builder only (u32 ids)

// The staging and ordered-sum tiles of the engine that serves a container (picked on the host by engine_tiles); the
// argument struct of every one-warp kernel carries them.
struct WarpTiles {
    uint32_t stg_rows;       // candidate rows per staged batch (0 = this element kind loads directly)
    uint32_t stg_row_bytes;  // bytes of one staged row (f32: 128*FULL, i8: a 512-byte pass slot, embeddings: one sum)
    uint32_t tile_rows;      // rows of the ordered-sum tile (0 for i8, which has none)
};

// Shared-memory layout of one warp in the dynamic window: the host sizes every launch from it, the build and re-rank
// kernels place their pointers with it (place_warp_smem), and search_kernel spells out the same walk:
//   tile (ordered-sum rows) + id scratch | reserved 16 bytes | qs | xs (embeddings only) | staging tile | end
// qs holds the query (f32 dim rounded up to 4 floats, or the row_stride bytes of an i8 row), xs one element of the same
// size; both start on 16-byte boundaries, the staging tile (stg_rows x stg_row_bytes) on a 128-byte boundary.  Behind
// `end` each kernel appends its own: the fast list, or the generic list and visited set (search_kernel), the link
// scratch (build kernels: LinkLayout), or the sort keys (rerank_kernel: rerank_keys_offset).
// The layout is walked from `base` in the address type P: the host walks byte offsets (P = size_t, base = 0), the
// kernels walk their shared window (P = unsigned char*, base = smem_raw), so that every pointer is smem_raw + offset
// and the compiler keeps the accesses in the shared address space (LDS/STS with 32-bit addresses).
template <class P>
struct SmemLayout {
    // Once held the mbarrier of a bulk-copy gather.  Kept because moving the offsets behind it reschedules the search
    // kernels, which run at their register cap; removing it needs a measurement of its own.
    static constexpr uint32_t kReservedBytes = 16;
    P ids, qs, xs, stg, end;  // stg = P() without a staging tile

    __host__ __device__ __forceinline__ SmemLayout(P base, int kind, uint32_t dim, uint32_t row_stride,
                                                   const WarpTiles& t) {
        P sp = base;  // the tile starts at base
        ids = sp + tile_bytes_for_rows(t.tile_rows) - kIdScratchBytes;
        sp += tile_bytes_for_rows(t.tile_rows);
        sp += kReservedBytes;
        const uint32_t slot_bytes = (kind == kAngularI8) ? row_stride : ((dim + 3u) & ~3u) * 4u;
        qs = sp;
        sp += (slot_bytes + 15u) & ~15u;
        xs = sp;
        if (kind == kSumEmbeddings) sp += (slot_bytes + 15u) & ~15u;
        stg = P();
        if (t.stg_rows) {
            sp = base + (((size_t)(sp - base) + 127u) & ~(size_t)127u);
            stg = sp;
            sp += (size_t)t.stg_rows * t.stg_row_bytes;
        }
        end = sp;
    }
};

// per-query status bits (device side)
constexpr int kStatusOverflow = 1;   // workspace too small for an exact answer -> slow path
constexpr int kStatusNotFinite = 2;  // NaN distance (reference panics)
constexpr int kStatusBadFilter = 16; // filtered search: a query_filter entry >= num_filters (ERR_INVALID_ARGUMENT)

// The staged index in HBM.
struct DeviceIndex {
    int kind;
    uint32_t dim;
    uint32_t full;        // dim / 32   (number of complete 32-wide chunks, src/math.rs:21)
    uint32_t tail;        // dim % 32
    uint32_t vec_group;   // V: chunks interleaved per lane in the permuted f32 row layout (4, 2 or 1)
    uint32_t row_stride;  // f32: floats per row (multiple of 4); i8: bytes per row (multiple of 16)
    const void* vectors;  // f32 rows (ANGULAR: elements; EMBEDDINGS: embedding table) or i8 rows
    uint64_t num_vectors;
    const unsigned long long* sum_offsets;  // EMBEDDINGS: num_elements + 1
    const uint32_t* sum_terms;
    uint64_t num_elements;
    int num_layers;
    const uint32_t* layer_rows[kMaxLayers];
    uint32_t layer_width[kMaxLayers];
    unsigned long long layer_len[kMaxLayers];
};

// Fused result gather (replicated index, queries sharded over GPUs): instead of leaving the tile in local memory for a
// collective, the kernel stores every result row straight into the gathered buffer of EVERY peer (peer-mapped
// memory over NVLink/NVSwitch; the own buffer is one of the entries) at row `row_offset + query`.  When all stores of
// the launch are done, flags[p][my_rank] = seq is released system-wide so consumers on the peers can tell.
constexpr int kMaxPeers = 8;
struct PeerGather {
    uint32_t* ids[kMaxPeers];
    float* dists[kMaxPeers];
    unsigned int* flags[kMaxPeers];
    uint32_t n_peers;  // 0 = disabled (results go to out_ids / out_dists)
    uint32_t my_rank;
    unsigned long long row_offset;
    unsigned int seq;
    unsigned int* done_counter;
};

struct SearchArgs {
    const void* queries;  // nq x dim (f32 or i8)
    int query_format;
    unsigned long long nq;
    uint32_t max_search;
    uint32_t num_neighbors;
    uint32_t list_cap;        // C for the bottom layer
    uint32_t vis_slots;       // visited slots for the bottom layer
    uint32_t vis_slots_upper; // visited slots for the max_search = 1 descents
    uint32_t* vis_global;     // fast pass: one table of vis_slots u32 per CTA in global memory (L2 resident)
    WarpTiles tiles;
    uint32_t* out_ids;
    float* out_dists;
    uint32_t* out_counts;
    unsigned long long* out_stats;  // nq x 4 or null
    int* query_status;              // nq ints (0 = done ok)
    unsigned int* work_counter;     // persistent scheduling (one counter per pass)
    unsigned int* gate_in;          // passes after the first: run only if *gate_in != 0 (somebody flagged a query)
    unsigned int* gate_out;         // set when this pass flags a query for the next pass
    unsigned long long* retried;    // cumulative count of queries that needed more than the first pass (or null)
    int* error_flag;                // sticky device error word (OR of status bits that are final)
    // slow path only: global workspaces (one per slow CTA)
    unsigned long long* slow_list;
    uint32_t* slow_visited;
    uint32_t slow_list_cap;
    uint32_t slow_vis_slots;
    // Pass ladder: 0 = fast pass over every query; 1 = retry (same kernel shape, longer list, larger visited tables)
    // over the queries the fast pass flagged; 2 = slow pass (global-memory workspaces) over what is still flagged.
    // The last pass of a call reports exhaustion as an error and signals the peers of a fused gather.
    int pass;
    int slow_pass;   // this pass uses the global slow workspaces (list + visited set)
    int final_pass;  // nothing comes after this pass
    PeerGather pg;
    // filtered search only (search_kernel<Dist, R, true>): num_filters bitmaps of filter_words u32 words each; query
    // q keeps the scored bottom-layer candidates i whose bit filter_bit_base + i is set in bitmap query_filter[q]
    // (query_filter null: bitmap 0), in a sorted list of filter_cap = round_up(k, 32) keys behind the pass's own
    // shared memory
    const uint32_t* filters;
    const uint32_t* query_filter;
    unsigned long long filter_words;
    unsigned long long filter_bit_base;
    uint32_t num_filters;
    uint32_t filter_cap;
};

// ------------------------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t key_dbits(unsigned long long key) { return (uint32_t)(key >> 32) & 0x7FFFFFFFu; }
__device__ __forceinline__ uint32_t key_id(unsigned long long key) { return (uint32_t)key; }
__device__ __forceinline__ unsigned long long make_key(float d, uint32_t id) {
    return ((unsigned long long)__float_as_uint(d) << 32) | id;
}
__device__ __forceinline__ unsigned lanemask_lt() {
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// Streaming 32-bit loads of candidate rows: read-only path, do not pollute L1 (each row is used once).
__device__ __forceinline__ float ldg_row_f1(const float* p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ int ldg_row_i32(const int* p) {
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// cmp::max(0.0, 1.0 - r) with NaN detection (angular.rs:70-73, angular_int.rs:55-58)
__device__ __forceinline__ float finish_angular(float r, int* status) {
    float d = __fsub_rn(1.0f, r);
    if (d != d) {
        *status |= kStatusNotFinite;
        return 0.0f;
    }
    return (0.0f <= d) ? d : 0.0f;
}

// The angular_int distance from r = dot(x, y), dx = dot(x, x) and dy = dot(y, y): 1 - r / (sqrt(dx) * sqrt(dy)) in
// IEEE f32, NaN -> 0, max(0, .) (angular_int.rs:47-59).
__device__ __forceinline__ float finish_angular_i8(int r, int dx, int dy) {
    const float rf = (float)r, dxf = (float)dx, dyf = (float)dy;
    float qq = __fdiv_rn(rf, __fmul_rn(__fsqrt_rn(dxf), __fsqrt_rn(dyf)));
    if (qq != qq) qq = 0.0f;  // NotNan::new(..).unwrap_or_else(|_| 0.0)
    const float dd = __fsub_rn(1.0f, qq);
    return (0.0f <= dd) ? dd : 0.0f;
}

// Per-warp working set (pointers may be shared or global memory: the slow path uses global workspaces).
struct WarpCtx {
    unsigned long long* list;  // L
    uint32_t* visited;
    float* tile;       // 32 x kTileStride floats (always shared)
    uint32_t* ids;     // 32 u32 scratch for compacting candidate ids (always shared)
    float* qs;         // query, natural layout: f32[dim] (or i8 words for ANGULAR_INT), shared
    float* xs;         // EMBEDDINGS scratch f32[dim], shared
    unsigned char* stg;  // staging tile for gathered candidate rows (shared, 128-byte aligned)
    uint32_t stg_rows;   // rows that fit in the staging tile (<= 16)
    uint32_t stg_row_bytes;
    unsigned long long pol_keep;    // L2 policy evict_last: the per-warp visited tables are re-read all the time
    int lane;
    int status;
    int q_norm_i8;     // ANGULAR_INT: dy = sum q^2
    uint32_t n_dist, n_expand, n_nbr;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long make_policy_evict_last() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// Points the warp's shared buffers into smem_raw as SmemLayout places them; returns the first byte behind them.
__device__ __forceinline__ unsigned char* place_warp_smem(WarpCtx& c, unsigned char* smem_raw, const DeviceIndex& ix,
                                                          const WarpTiles& t) {
    const SmemLayout<unsigned char*> L(smem_raw, ix.kind, ix.dim, ix.row_stride, t);
    c.tile = reinterpret_cast<float*>(smem_raw);
    c.ids = reinterpret_cast<uint32_t*>(L.ids);
    c.pol_keep = make_policy_evict_last();
    c.qs = reinterpret_cast<float*>(L.qs);
    c.xs = reinterpret_cast<float*>(L.xs);
    c.stg = L.stg;
    c.stg_rows = t.stg_rows;
    c.stg_row_bytes = t.stg_row_bytes;
    return L.end;
}

// ---- per-lane asynchronous copies (cp.async -> LDGSTS): global -> shared without staging registers ----------------
// Lane l copies (and later reads back) only ITS OWN bytes of a row, so completion needs no cross-lane barrier: the
// issuing thread waits for its own copies with cp.async.wait_all.  One instruction copies 32 x BYTES contiguous bytes.
template <int BYTES>
__device__ __forceinline__ void cp_async_lane(uint32_t dst, const void* src) {
    // (no L2::cache_hint operand: ptxas 12.9 encodes LDGSTS + policy with never-written uniform registers in this
    // kernel and the instruction traps as illegal)
    if (BYTES == 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    else if (BYTES == 8)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
    else
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// waits until at most the most recently committed group is still in flight
__device__ __forceinline__ void cp_async_wait_but_last() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// Strictly ordered sum of the 32 lane partials of ONE value (used where only a single candidate is live):
// r = 0; for i in 0..32 { r += chunk[i] }   (src/math.rs:27-30).  All lanes return the same r.
__device__ __forceinline__ float ordered_lane_sum_bcast(float p) {
    float r = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) r = __fadd_rn(r, __shfl_sync(kFullMask, p, i));
    return r;
}

// The same ordered sum for the 32 lane partials of one candidate parked in row `trow` of the tile (the lane that
// owns the candidate sums; 16-byte aligned rows, one LDS.128 per four partials).
__device__ __forceinline__ float ordered_tile_sum(const float* tile, int trow) {
    float r = 0.0f;
    const float4* t = reinterpret_cast<const float4*>(tile + trow * kTileStride);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float4 v = t[i];
        r = __fadd_rn(r, v.x);
        r = __fadd_rn(r, v.y);
        r = __fadd_rn(r, v.z);
        r = __fadd_rn(r, v.w);
    }
    return r;
}

// normalize_f32 (math.rs:124-150) of x[0..dim) in place, all lanes: norm = sqrt(dot(x, x)) with dot_product_f32's
// order (lane FMA over the full chunks, ordered 32-lane sum, FMA tail); if norm > 0 { x[i] /= norm }.
__device__ __forceinline__ void normalize_f32(float* x, int dim, int full, int lane) {
    float p = 0.0f;
    for (int ch = 0; ch < full; ++ch) {
        const float v = x[ch * 32 + lane];
        p = __fmaf_rn(v, v, p);
    }
    float r = ordered_lane_sum_bcast(p);
    for (int t = full * 32; t < dim; ++t) {
        const float v = x[t];
        r = __fmaf_rn(v, v, r);
    }
    const float norm = __fsqrt_rn(r);
    __syncwarp();  // every lane has finished reading the un-normalised tail before anyone overwrites it
    if (norm > 0.0f)
        for (int i = lane; i < dim; i += 32) x[i] = __fdiv_rn(x[i], norm);
    __syncwarp();
}

// angular_int::Vector::quantize (angular_int.rs:28-45) of x[0..dim) into dst, all lanes: max |x|, then x * 127 / max
// truncated toward zero and clamped to i8 (NaN -> 0).  Sets kStatusNotFinite in *status if x holds a NaN (the
// reference's NotNan max fails on it).
__device__ __forceinline__ void quantize_i8(const float* x, int8_t* dst, int dim, int lane, int* status) {
    float mx = 0.0f;
    bool bad = false;
    for (int i = lane; i < dim; i += 32) {
        const float v = x[i];
        if (v != v) bad = true;
        mx = fmaxf(mx, fabsf(v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, o));
    if (__any_sync(kFullMask, bad)) *status |= kStatusNotFinite;
    for (int i = lane; i < dim; i += 32) {
        const float vi = __fdiv_rn(__fmul_rn(x[i], 127.0f), mx);
        int q;
        if (vi != vi)
            q = 0;
        else if (vi >= 127.0f)
            q = 127;
        else if (vi <= -128.0f)
            q = -128;
        else
            q = (int)vi;  // truncation toward zero
        dst[i] = (int8_t)q;
    }
}

// Position of element e < 32*full in a lane-permuted f32 row (permute_rows_f32_kernel): chunk ch = g*V + v, lane i
// lands at g*32*V + i*V + v.  The tail (e >= 32*full) stays in place.
__device__ __forceinline__ uint32_t permuted_offset(uint32_t e, uint32_t V) {
    const uint32_t ch = e / 32, i = e % 32, g = ch / V, vv = ch % V;
    return g * 32 * V + i * V + vv;
}

// ------------------------------------------------------------------------------------------------------------------
// distance engines.  Contract: on entry lane j (< k) holds candidate id `my_id`; returns d_j in lane j.
// ------------------------------------------------------------------------------------------------------------------

// ANGULAR f32, compile-time chunk count FULL (dim = 32*FULL + tail).  Query chunk values live in registers.
// Candidate rows are gathered into the staging tile with per-lane cp.async (see dists), a whole batch of rows in flight
// at once and no data registers held.  Rows are lane-permuted in HBM (permute_rows_f32_kernel) so that lane i copies
// and then reads its share of G*V chunks with conflict-free LDS.128/64/32.
template <int FULL>
struct DistF32 {
    static constexpr int V = (FULL % 4 == 0) ? 4 : ((FULL % 2 == 0) ? 2 : 1);
    static constexpr int G = FULL / V;
    static constexpr int NQ = FULL > 0 ? FULL : 1;
    float q[NQ];

    __device__ __forceinline__ void load_query(const DeviceIndex& ix, const WarpCtx& c) {
#pragma unroll
        for (int ch = 0; ch < FULL; ++ch) q[ch] = c.qs[ch * 32 + c.lane];
    }

    __device__ __forceinline__ float partial(const unsigned char* row) const {
        const float* r = reinterpret_cast<const float*>(row);
        float p = 0.0f;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            if (V == 4) {
                const float4 v = *reinterpret_cast<const float4*>(r + g * 128);
                p = __fmaf_rn(v.x, q[g * 4 + 0], p);
                p = __fmaf_rn(v.y, q[g * 4 + 1], p);
                p = __fmaf_rn(v.z, q[g * 4 + 2], p);
                p = __fmaf_rn(v.w, q[g * 4 + 3], p);
            } else if (V == 2) {
                const float2 v = *reinterpret_cast<const float2*>(r + g * 64);
                p = __fmaf_rn(v.x, q[g * 2 + 0], p);
                p = __fmaf_rn(v.y, q[g * 2 + 1], p);
            } else {
                p = __fmaf_rn(r[g * 32], q[g], p);
            }
        }
        return p;
    }

    // The ordered 32-lane sum (math.rs:27-30) and the FMA tail (:32-39) for candidate `id`, whose lane partials sit
    // in tile row `trow` (ignored when FULL == 0).
    __device__ __forceinline__ float ordered_finish(const DeviceIndex& ix, WarpCtx& c, uint32_t id, int trow) const {
        float r = 0.0f;
        if (FULL > 0) r = ordered_tile_sum(c.tile, trow);
        const int tail = ix.tail;
        if (tail) {
            const float* row = reinterpret_cast<const float*>(static_cast<const char*>(ix.vectors) +
                                                               (size_t)id * (ix.row_stride * 4u)) + FULL * 32;
            const float* qt = c.qs + FULL * 32;
            for (int t = 0; t < tail; ++t) r = __fmaf_rn(__ldg(row + t), qt[t], r);
        }
        return finish_angular(r, &c.status);
    }

    // Batches of up to stg_rows (<= 8 = tile rows) candidates: gather, lane partials into the tile, ordered sums.
    // Gather: one cp.async per row (per 32-chunk group): lane l copies the V*4 bytes of the permuted row that lane l
    // itself consumes, so a row costs SHFL + address + LDGSTS, all rows of the batch are in flight together, no data
    // registers are held and no cross-lane barrier is needed before the partial sums.
    // `ids_smem` (may be null): the same candidate ids, compacted in shared memory — the search loop has them there
    // anyway, and a broadcast LDS per row is cheaper than a shuffle with its divergence check.
    template <class Hook>
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k, Hook&& after_wait,
                                           const uint32_t* ids_smem = nullptr) {
        float d = 0.0f;
        if (FULL > 0) {
            const uint32_t stride_bytes = ix.row_stride * 4u;
            constexpr uint32_t row_bytes = FULL * 128u;  // the permuted chunk part of a row
            constexpr uint32_t lane_bytes = V * 4u;
            const char* src0 = static_cast<const char*>(ix.vectors) + c.lane * lane_bytes;
            asm volatile("" : "+l"(src0));  // keep the per-lane base in one register pair (one IMAD.WIDE per row)
            const uint32_t dst0 = smem_u32(c.stg) + c.lane * lane_bytes;
            const unsigned char* mine = c.stg + c.lane * lane_bytes;
            const int rb = (int)c.stg_rows;
            const bool has_tail = ix.tail != 0;
            for (int j0 = 0; j0 < k; j0 += rb) {
                const int nb = (k - j0) < rb ? (k - j0) : rb;
#pragma unroll
                for (int b = 0; b < 8; ++b) {
                    if (b >= nb) break;
                    const uint32_t idb = ids_smem ? ids_smem[j0 + b] : __shfl_sync(kFullMask, my_id, j0 + b);
                    const char* src = src0 + (size_t)idb * stride_bytes;
#pragma unroll
                    for (int g = 0; g < G; ++g)
                        cp_async_lane<(int)lane_bytes>(dst0 + b * row_bytes + g * 32 * lane_bytes,
                                                       src + g * 32 * lane_bytes);
                }
                cp_async_wait_all();
                if (j0 == 0) after_wait();  // everything copied before this call has landed too
#pragma unroll
                for (int b = 0; b < 8; ++b) {
                    if (b >= nb) break;
                    c.tile[b * kTileStride + c.lane] = partial(mine + b * row_bytes);
                }
                __syncwarp();
                uint32_t id = 0;
                if (has_tail) id = __shfl_sync(kFullMask, my_id, (j0 + c.lane) & 31);  // lane t: candidate j0 + t
                float db = 0.0f;
                if (c.lane < nb) db = ordered_finish(ix, c, id, c.lane);
                if (j0 == 0) {
                    d = db;  // first batch: lane t already is candidate t
                } else {
                    // hand the distance of candidate j0 + t (computed by lane t) to lane j0 + t
                    const float dj = __shfl_sync(kFullMask, db, (c.lane - j0) & 31);
                    if (c.lane >= j0 && c.lane < j0 + nb) d = dj;
                }
                __syncwarp();  // the next batch rewrites the tile
            }
        } else {
            if (c.lane < k) d = ordered_finish(ix, c, my_id, 0);
            __syncwarp();
            after_wait();
        }
        return d;
    }
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k) {
        return dists(ix, c, my_id, k, [] {});
    }
};

// ANGULAR f32, any dim (runtime chunk count; natural row layout; query read from shared memory): the dims the
// compile-time engines do not cover (dim/32 in {5, 7, 9, ...}: 160, 224, 300 ...).  Staged like DistF32: lane l copies
// float l of every 32-chunk with a 4-byte cp.async (one instruction moves 128 contiguous bytes), reads the same bytes
// back for its accumulator chunk[l], and the ordered 32-lane sums of a batch run through the 8-row tile.  Rows too
// wide for the staging tile (stg_rows == 0) load directly.
struct DistF32Generic {
    __device__ __forceinline__ void load_query(const DeviceIndex&, const WarpCtx&) {}

    static __device__ __forceinline__ float ordered_finish(const DeviceIndex& ix, WarpCtx& c, uint32_t id, int trow) {
        float r = ordered_tile_sum(c.tile, trow);
        const int full = ix.full;
        const float* row = static_cast<const float*>(ix.vectors) + (size_t)id * ix.row_stride + full * 32;
        const float* qt = c.qs + full * 32;
        for (int t2 = 0; t2 < (int)ix.tail; ++t2) r = __fmaf_rn(__ldg(row + t2), qt[t2], r);
        return finish_angular(r, &c.status);
    }

    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k) {
        const float* base = static_cast<const float*>(ix.vectors);
        const size_t stride = ix.row_stride;
        const int full = ix.full;
        float d = 0.0f;
        if (c.stg_rows == 0 || full == 0) {
            // direct loads, one candidate after the other (32-row tile)
            for (int j = 0; j < k; ++j) {
                const uint32_t id = __shfl_sync(kFullMask, my_id, j);
                const float* row = base + (size_t)id * stride + c.lane;
                float p = 0.0f;
                for (int ch = 0; ch < full; ++ch) p = __fmaf_rn(ldg_row_f1(row + ch * 32), c.qs[ch * 32 + c.lane], p);
                c.tile[j * kTileStride + c.lane] = p;
            }
            __syncwarp();
            if (c.lane < k) d = ordered_finish(ix, c, my_id, c.lane);
            __syncwarp();
            return d;
        }
        const uint32_t row_bytes = (uint32_t)full * 128u;
        const char* src0 = reinterpret_cast<const char*>(base) + c.lane * 4;
        const uint32_t dst0 = smem_u32(c.stg) + c.lane * 4u;
        const float* mine = reinterpret_cast<const float*>(c.stg) + c.lane;
        const int rb = (int)c.stg_rows;  // <= 8 = tile rows
        for (int j0 = 0; j0 < k; j0 += rb) {
            const int nb = (k - j0) < rb ? (k - j0) : rb;
            for (int b = 0; b < nb; ++b) {
                const uint32_t idb = __shfl_sync(kFullMask, my_id, j0 + b);
                const char* src = src0 + (size_t)idb * stride * 4u;
                for (int ch = 0; ch < full; ++ch) cp_async_lane<4>(dst0 + b * row_bytes + ch * 128, src + ch * 128);
            }
            cp_async_wait_all();
            for (int b = 0; b < nb; ++b) {
                const float* r = mine + b * full * 32;
                float p = 0.0f;
                for (int ch = 0; ch < full; ++ch) p = __fmaf_rn(r[ch * 32], c.qs[ch * 32 + c.lane], p);
                c.tile[b * kTileStride + c.lane] = p;
            }
            __syncwarp();
            const uint32_t id = __shfl_sync(kFullMask, my_id, (j0 + c.lane) & 31);  // lane t: candidate j0 + t
            float db = 0.0f;
            if (c.lane < nb) db = ordered_finish(ix, c, id, c.lane);
            const float dj = __shfl_sync(kFullMask, db, (c.lane - j0) & 31);
            if (c.lane >= j0 && c.lane < j0 + nb) d = dj;
            __syncwarp();
        }
        return d;
    }
    template <class Hook>
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k, Hook&& after_wait,
                                           const uint32_t* = nullptr) {
        const float d = dists(ix, c, my_id, k);
        after_wait();
        return d;
    }
};

// ANGULAR_INT i8: exact i32 r, dx via dp4a (src/math.rs:59-89), then 1 - r/(sqrt(dx)*sqrt(dy)) in IEEE f32
// (src/elements/angular_int.rs:47-59).  Rows and the query are zero-padded to row_stride bytes (a multiple of 32: a
// row starts on a sector boundary and touches ceil(dim/32) sectors).
// Sub-warp groups: a row is C = row_stride/16 chunks of 16 bytes; L = next power of two >= C lanes work on one row
// (lane handles chunk lane % L), so one pass of the warp handles 32/L candidate rows at once: every lane copies ITS
// chunk with one cp.async (its own 16-byte slot, no cross-lane hazard), multiplies it with its 16 query bytes held in
// registers (8 dp4a), and the exact integer sums are reduced inside the group with log2(L) xor-shuffles — integer
// addition is order independent.  A 100-byte row costs a quarter of a pass instead of a full-warp pass + 2 REDUX.
struct DistI8 {
    int4 qv;      // the 16 query bytes of this lane's chunk
    uint32_t lg;   // log2(L)
    uint32_t C;    // chunks per row (0: rows wider than 512 bytes, generic path)

    __device__ __forceinline__ void load_query(const DeviceIndex& ix, const WarpCtx& c) {
        const uint32_t chunks = ix.row_stride / 16u;
        C = chunks <= 32u ? chunks : 0u;
        uint32_t L = 1;
        lg = 0;
        while (L < chunks && L < 32u) {
            L <<= 1;
            ++lg;
        }
        const uint32_t chunk = (uint32_t)c.lane & (L - 1u);
        qv = make_int4(0, 0, 0, 0);
        if (C && chunk < C) qv = reinterpret_cast<const int4*>(c.qs)[chunk];
    }

    __device__ __forceinline__ float finish(const WarpCtx& c, int my_r, int my_dx, bool live) const {
        float d = 0.0f;
        if (live) d = finish_angular_i8(my_r, my_dx, c.q_norm_i8);
        return d;
    }

    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k) {
        const uint32_t stride = ix.row_stride;
        const int lane = c.lane;
        int my_r = 0, my_dx = 0;
        if (C == 0) {
            // very wide rows: one candidate at a time, lanes stride over the 32-bit words
            const int words = stride / 4;
            const int* qw = reinterpret_cast<const int*>(c.qs);
            for (int j = 0; j < k; ++j) {
                const uint32_t id = __shfl_sync(kFullMask, my_id, j);
                const int* row = reinterpret_cast<const int*>(static_cast<const char*>(ix.vectors) + (size_t)id * stride);
                int r = 0, dx = 0;
                for (int w = lane; w < words; w += 32) {
                    const int a = ldg_row_i32(row + w);
                    r = __dp4a(a, qw[w], r);
                    dx = __dp4a(a, a, dx);
                }
                r = __reduce_add_sync(kFullMask, r);
                dx = __reduce_add_sync(kFullMask, dx);
                if (lane == j) {
                    my_r = r;
                    my_dx = dx;
                }
            }
            const float d = finish(c, my_r, my_dx, lane < k);
            __syncwarp();
            return d;
        }
        const uint32_t L = 1u << lg;
        const int rp = 32 >> lg;                          // candidate rows per pass
        const int grp = lane >> lg;                       // my row within a pass
        const uint32_t chunk = (uint32_t)lane & (L - 1u);
        const bool has_chunk = chunk < C;
        const int ppb = (int)c.stg_rows;                  // 512-byte pass slots in the staging tile
        const char* src0 = static_cast<const char*>(ix.vectors) + chunk * 16u;
        const uint32_t dst0 = smem_u32(c.stg) + lane * 16u;
        const int4* mine = reinterpret_cast<const int4*>(c.stg) + lane;
        for (int j0 = 0; j0 < k; j0 += rp * ppb) {
            const int left = k - j0;
            const int np = (left + rp - 1) / rp < ppb ? (left + rp - 1) / rp : ppb;
            for (int p = 0; p < np; ++p) {
                const int cand = j0 + p * rp + grp;
                const uint32_t id = __shfl_sync(kFullMask, my_id, cand & 31);
                if (has_chunk && cand < k) cp_async_lane<16>(dst0 + p * 512u, src0 + (size_t)id * stride);
            }
            cp_async_wait_all();
            for (int p = 0; p < np; ++p) {
                const int base = j0 + p * rp;
                int4 a = make_int4(0, 0, 0, 0);
                if (has_chunk && base + grp < k) a = mine[p * 32];
                int r = __dp4a(a.x, qv.x, 0);
                r = __dp4a(a.y, qv.y, r);
                r = __dp4a(a.z, qv.z, r);
                r = __dp4a(a.w, qv.w, r);
                int dx = __dp4a(a.x, a.x, 0);
                dx = __dp4a(a.y, a.y, dx);
                dx = __dp4a(a.z, a.z, dx);
                dx = __dp4a(a.w, a.w, dx);
                for (uint32_t o = L >> 1; o > 0; o >>= 1) {
                    r += __shfl_xor_sync(kFullMask, r, o);
                    dx += __shfl_xor_sync(kFullMask, dx, o);
                }
                // every lane of group g now holds the sums of candidate base + g: hand them to lane base + g
                const int src = ((lane - base) << lg) & 31;
                const int tr = __shfl_sync(kFullMask, r, src);
                const int tdx = __shfl_sync(kFullMask, dx, src);
                if (lane >= base && lane < base + rp) {
                    my_r = tr;
                    my_dx = tdx;
                }
            }
        }
        return finish(c, my_r, my_dx, lane < k);
    }
    template <class Hook>
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k, Hook&& after_wait,
                                           const uint32_t* = nullptr) {
        const float d = dists(ix, c, my_id, k);
        after_wait();
        return d;
    }
};

// EMBEDDINGS: element = ordered sum of embedding rows, normalised, then the f32 angular distance
// (src/elements/embeddings/mod.rs:124-143,164-174; src/math.rs:92-150).  Natural row layout, runtime dim.
struct DistSum {
    __device__ __forceinline__ void load_query(const DeviceIndex&, const WarpCtx&) {}

    // materialises ElementContainer::get(id) into c.xs (all lanes participate)
    static __device__ __forceinline__ void materialise(const DeviceIndex& ix, WarpCtx& c, uint32_t id) {
        const float* emb = static_cast<const float*>(ix.vectors);
        const size_t stride = ix.row_stride;
        const int dim = ix.dim;
        const unsigned long long b = ix.sum_offsets[id], e = ix.sum_offsets[id + 1];
        for (int i = c.lane; i < dim; i += 32) {
            float x = 0.0f;
            if (b < e) {
                x = __ldg(emb + (size_t)ix.sum_terms[b] * stride + i);
                for (unsigned long long t = b + 1; t < e; ++t)
                    x = __fadd_rn(x, __ldg(emb + (size_t)ix.sum_terms[t] * stride + i));  // sum_into_f32
            }
            c.xs[i] = x;
        }
        __syncwarp();
        normalize_f32(c.xs, dim, (int)ix.full, c.lane);
    }

    // Ordered 32-lane sum of tile row `trow` (math.rs:27-30) followed by the FMA tail over x[t]*y[t] (:32-39).
    static __device__ __forceinline__ float ordered_dot(const WarpCtx& c, int trow, const float* x, const float* y,
                                                        int full, int dim) {
        float r = ordered_tile_sum(c.tile, trow);
        for (int e = full * 32; e < dim; ++e) r = __fmaf_rn(x[e], y[e], r);
        return r;
    }

    // Batches of up to stg_rows candidates: their summed vectors live in the staging tile (row b = candidate b), the
    // lane partials of the two dot products (norm, distance) go through the 8-row tile so that the strictly ordered
    // 32-lane sums of a whole batch run in parallel (lane b sums candidate b) instead of two 32-step shuffle chains
    // per candidate.
    template <class Hook>
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k, Hook&& after_wait,
                                           const uint32_t* = nullptr) {
        const float d = dists(ix, c, my_id, k);
        after_wait();
        return d;
    }
    __device__ __forceinline__ float dists(const DeviceIndex& ix, WarpCtx& c, uint32_t my_id, int k) {
        const float* emb = static_cast<const float*>(ix.vectors);
        const size_t stride = ix.row_stride;
        const int dim = ix.dim, full = ix.full;
        const int xstride = (int)(c.stg_row_bytes / 4u);
        float* X = reinterpret_cast<float*>(c.stg);
        const int rb = (int)c.stg_rows;
        float d = 0.0f;
        for (int j0 = 0; j0 < k; j0 += rb) {
            const int nb = (k - j0) < rb ? (k - j0) : rb;
            const uint32_t idl = __shfl_sync(kFullMask, my_id, (j0 + c.lane) & 31);  // lane t: candidate j0 + t
            __syncwarp();
            // get_embedding_internal (embeddings/mod.rs:124-143): ordered sum of the term rows, element-wise.  Lane t
            // holds the id of term t; four 32-float chunks of a row are accumulated per pass, so that four independent
            // 128-byte loads per term are in flight (the adds per element stay in term order: sum_into_f32).
            for (int b = 0; b < nb; ++b) {
                const uint32_t id = __shfl_sync(kFullMask, idl, b);
                const unsigned long long tb = ix.sum_offsets[id], te = ix.sum_offsets[id + 1];
                const uint32_t m = (uint32_t)(te - tb);
                float* xb = X + b * xstride;
                for (int i0 = 0; i0 < dim; i0 += 128) {
                    const int i = i0 + c.lane;
                    const bool in0 = i < dim, in1 = i + 32 < dim, in2 = i + 64 < dim, in3 = i + 96 < dim;
                    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
                    for (uint32_t g = 0; g < m; g += 32) {
                        const uint32_t gm = (m - g) < 32u ? (m - g) : 32u;
                        const uint32_t my_term = ((uint32_t)c.lane < gm) ? __ldg(ix.sum_terms + tb + g + c.lane) : 0u;
                        for (uint32_t t = 0; t < gm; ++t) {
                            const uint32_t term = __shfl_sync(kFullMask, my_term, t);
                            const float* row = emb + (size_t)term * stride + i;
                            const float v0 = in0 ? __ldg(row) : 0.0f;
                            const float v1 = in1 ? __ldg(row + 32) : 0.0f;
                            const float v2 = in2 ? __ldg(row + 64) : 0.0f;
                            const float v3 = in3 ? __ldg(row + 96) : 0.0f;
                            if (g + t == 0) {  // x = row_0, then x += row_t in order
                                a0 = v0, a1 = v1, a2 = v2, a3 = v3;
                            } else {
                                a0 = __fadd_rn(a0, v0);
                                a1 = __fadd_rn(a1, v1);
                                a2 = __fadd_rn(a2, v2);
                                a3 = __fadd_rn(a3, v3);
                            }
                        }
                    }
                    if (in0) xb[i] = a0;
                    if (in1) xb[i + 32] = a1;
                    if (in2) xb[i + 64] = a2;
                    if (in3) xb[i + 96] = a3;
                }
            }
            __syncwarp();
            // normalize_f32 (math.rs:124-150): norm = sqrt(dot(x, x))
            for (int b = 0; b < nb; ++b) {
                const float* xb = X + b * xstride;
                float p = 0.0f;
                for (int ch = 0; ch < full; ++ch) {
                    const float v = xb[ch * 32 + c.lane];
                    p = __fmaf_rn(v, v, p);
                }
                c.tile[b * kTileStride + c.lane] = p;
            }
            __syncwarp();
            float norm = 0.0f;
            if (c.lane < nb) {
                const float* xb = X + c.lane * xstride;
                norm = __fsqrt_rn(ordered_dot(c, c.lane, xb, xb, full, dim));
            }
            __syncwarp();
            for (int b = 0; b < nb; ++b) {
                const float nrm = __shfl_sync(kFullMask, norm, b);
                float* xb = X + b * xstride;
                float p = 0.0f;
                if (nrm > 0.0f)
                    for (int i = c.lane; i < dim; i += 32) xb[i] = __fdiv_rn(xb[i], nrm);
                __syncwarp();
                // angular distance to the query (angular.rs:63-74)
                for (int ch = 0; ch < full; ++ch) p = __fmaf_rn(xb[ch * 32 + c.lane], c.qs[ch * 32 + c.lane], p);
                c.tile[b * kTileStride + c.lane] = p;
            }
            __syncwarp();
            float db = 0.0f;
            if (c.lane < nb) db = finish_angular(ordered_dot(c, c.lane, X + c.lane * xstride, c.qs, full, dim), &c.status);
            const float dj = __shfl_sync(kFullMask, db, (c.lane - j0) & 31);
            if (c.lane >= j0 && c.lane < j0 + nb) d = dj;
        }
        __syncwarp();
        return d;
    }
};

// ------------------------------------------------------------------------------------------------------------------
// visited set: FxHashSet<usize> semantics (src/index/mod.rs:1009-1010,1016,1026), exact.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t vis_hash(uint32_t id, uint32_t slots) {
    return __umulhi(id * 0x9E3779B1u, slots);  // multiply-shift range reduction, slots need not be a power of two
}
// returns true if `id` was newly inserted.  Lanes of one warp may insert concurrently (atomicCAS decides ties).
__device__ __forceinline__ bool vis_insert(uint32_t* tab, uint32_t slots, uint32_t id) {
    uint32_t h = vis_hash(id, slots);
    for (uint32_t probe = 0; probe < slots; ++probe) {
        const uint32_t prev = atomicCAS(tab + h, kUnusedId, id);
        if (prev == kUnusedId) return true;
        if (prev == id) return false;
        h = (h + 1 == slots) ? 0 : h + 1;
    }
    return false;  // unreachable: occupancy is capped below `slots` by the caller
}

// ------------------------------------------------------------------------------------------------------------------
// Bucketed visited set for the fast pass (global memory, private to one warp, L2 resident): buckets of 4 u32 slots
// (16 bytes, one 128-bit load), filled from slot 0 upwards, 0xFFFFFFFF = empty; a full home bucket chains to the next
// one.  A lookup is ONE load per lane; ids that are not found are inserted with plain stores — no atomics are needed
// because the table has a single writer warp and conflicts between lanes of that warp are resolved in registers with
// match.any.  Returns true in lanes whose id was newly inserted.  Sets *overflow when the chain gets too long
// (-> retry pass with a larger table).  Every lane loads (lanes without a valid id read the bucket 0xFFFFFFFF hashes
// to and ignore it), which keeps the probe free of predicate bookkeeping.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldcg_u4(const uint32_t* p, unsigned long long policy) {
    uint4 v;
    asm volatile("ld.global.cg.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(policy));
    return v;
}
__device__ __forceinline__ void stcg_u32(uint32_t* p, uint32_t v, unsigned long long policy) {
    asm volatile("st.global.cg.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(policy) : "memory");
}
__device__ __forceinline__ void stcg_u4(uint4* p, uint4 v, unsigned long long policy) {
    asm volatile("st.global.cg.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w), "l"(policy)
                 : "memory");
}
constexpr uint32_t kVisHashMul = 0x9E3779B1u;
// `pre` (warp-uniform, may be null): shared-memory copy of the home buckets of this very row, taken after the last
// insertion into the table (speculative expansion, see search_layer_fast) — it replaces the first round's loads.
__device__ __forceinline__ bool vis_bucket_insert(uint32_t* tab, uint32_t nbuckets, uint32_t id, bool valid,
                                                  bool* overflow, unsigned long long policy,
                                                  const uint4* pre = nullptr) {
    uint32_t b = __umulhi(id * kVisHashMul, nbuckets);
    bool pending = valid, is_new = false;
    for (int probe = 0;; ++probe) {
        uint32_t* bucket = tab + (size_t)b * 4u;
        uint4 v;
        if (probe == 0 && pre != nullptr)
            v = pre[threadIdx.x];
        else
            v = ldcg_u4(bucket, policy);
        const bool found = (v.x == id) | (v.y == id) | (v.z == id) | (v.w == id);
        pending = pending && !found;
        // slots are filled in order: the bucket is full iff its last slot is used
        bool ins = pending && (v.w == kUnusedId);
        const unsigned ins_mask = __ballot_sync(kFullMask, ins);
        if (ins_mask) {
            // the same id twice in one neighbour list (MultiSetVector allows duplicates): only the first lane inserts
            const unsigned same_id = __match_any_sync(kFullMask, id) & ins_mask;
            if (ins && (same_id & lanemask_lt())) {
                ins = false;
                pending = false;
            }
            // new ids that share a bucket take consecutive free slots
            const unsigned same_b = __match_any_sync(kFullMask, b) & __ballot_sync(kFullMask, ins);
            if (ins) {
                const uint32_t used = (v.x != kUnusedId) + (v.y != kUnusedId) + (v.z != kUnusedId);
                const uint32_t slot = used + __popc(same_b & lanemask_lt());
                if (slot < 4u) {
                    stcg_u32(bucket + slot, id, policy);
                    is_new = true;
                    pending = false;
                }
            }
        }
        if (pending) b = (b + 1 == nbuckets) ? 0 : b + 1;  // bucket full: continue in the next one
        __syncwarp();
        if (!__any_sync(kFullMask, pending)) break;
        if (probe >= 64) {
            *overflow = true;
            break;
        }
    }
    return is_new;
}

// ------------------------------------------------------------------------------------------------------------------
// search_for_neighbors (src/index/mod.rs:999-1037) on one layer.  On return the list holds the merged state;
// *out_n is its length.  The result set (`res.into_sorted_vec()`) is the first min(|E|, ef) expanded entries.
//
// Bookkeeping (all warp-uniform): n = entries in L; cursor = every entry before it is expanded; while res is not
// full n_exp counts the expanded entries of L; once res is full n_exp == ef and pos_thr is the position of res.peek()
// (the ef-th expanded entry), thr_bits its distance.  Expanded entries behind pos_thr are dead weight.
// The model of exactly this logic is tests/helpers/list_model.py::search_layer_model_v2 (validated on the CPU).
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t warp_min_u32(unsigned mask, uint32_t v) { return __reduce_min_sync(mask, v); }

// ------------------------------------------------------------------------------------------------------------------
// Filtered search: the admitted list.  Beside the traversal (which it never influences) the bottom layer's search
// offers every candidate it scores to a sorted list of the `cap` smallest make_key keys among those whose filter bit
// is set; the kernel then reports the first k of that list instead of the expanded entries of L.  The ids a layer
// search scores are distinct (the visited set), so keys are unique and the list is exactly the first cap keys of
// S(q) ∩ A in (distance, id) order.  The keys live in shared memory; all fields are warp-uniform.
// ------------------------------------------------------------------------------------------------------------------
struct AdmitList {
    unsigned long long* keys;  // sorted ascending, n valid
    const uint32_t* bits;      // the query's filter bitmap, bit (bit_base + id) LSB first
    unsigned long long bit_base;
    uint32_t cap, n;
};

// Lane l offers (id, d) when `scored`: admitted keys below the list's last (or all, while it is not full) are merged
// in, every lane of the warp takes part.  The merge is search_layer's: each offered key's rank is its lower bound in the
// list plus the offered keys below it, and the entries at or after the first rank move up row by row, top-down.
__device__ __forceinline__ void admit_offer(AdmitList& A, uint32_t id, float d, bool scored, int lane) {
    bool pass = false;
    if (scored) {
        const unsigned long long b = A.bit_base + id;
        pass = (__ldg(A.bits + (b >> 5)) >> (uint32_t)(b & 31u)) & 1u;
    }
    const unsigned long long key = make_key(d, id);
    if (A.n == A.cap) pass = pass && key < A.keys[A.cap - 1];
    const unsigned pm = __ballot_sync(kFullMask, pass);
    if (pm == 0) return;
    uint32_t lo = 0, hi = A.n;
    for (int it = 32 - __clz(A.n); it > 0; --it) {
        const uint32_t mid = (lo + hi) >> 1;
        if (lo < hi) {
            if (A.keys[mid] < key)
                lo = mid + 1;
            else
                hi = mid;
        }
    }
    uint32_t rank_n = 0;
    for (unsigned t = pm; t; t &= t - 1) rank_n += (__shfl_sync(kFullMask, key, __ffs(t) - 1) < key) ? 1u : 0u;
    const uint32_t new_pos = lo + rank_n;
    const uint32_t min_rank = warp_min_u32(kFullMask, pass ? lo : 0xFFFFFFFFu);
    for (int base = (int)((A.n - 1) & ~31u); base >= (int)(min_rank & ~31u); base -= 32) {
        const uint32_t j = base + lane;
        const bool in = (j < A.n) && (j >= min_rank);
        unsigned long long v = 0;
        if (in) v = A.keys[j];
        uint32_t sh = 0;
        for (unsigned t = pm; t; t &= t - 1) sh += (__shfl_sync(kFullMask, lo, __ffs(t) - 1) <= j) ? 1u : 0u;
        __syncwarp();
        if (in && j + sh < A.cap) A.keys[j + sh] = v;
    }
    __syncwarp();
    if (pass && new_pos < A.cap) A.keys[new_pos] = key;
    __syncwarp();
    A.n = min(A.n + (uint32_t)__popc(pm), A.cap);
}

// FILT: when `admit` (the bottom layer), `adm` receives every candidate this layer scores (admit_offer).
template <class Dist, bool FILT = false>
__device__ __forceinline__ void search_layer(const DeviceIndex& ix, WarpCtx& c, Dist& dist, const uint32_t* rows,
                                             const uint32_t width, const uint32_t entrypoint, const uint32_t ef,
                                             const uint32_t cap, const uint32_t vis_slots, uint32_t* out_n,
                                             AdmitList* adm = nullptr, bool admit = false) {
    unsigned long long* L = c.list;
    const int lane = c.lane;
    for (uint32_t i = lane; i < vis_slots; i += 32) c.visited[i] = kUnusedId;
    __syncwarp();
    const uint32_t vis_limit = vis_slots - (vis_slots >> 3);  // keep load factor <= 7/8
    uint32_t vis_count = 1;

    // seed (:1012-1016)
    {
        const float d0 = dist.dists(ix, c, entrypoint, 1);
        c.n_dist += 1;
        if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
            c.status |= kStatusNotFinite;
            *out_n = 0;
            return;
        }
        if (lane == 0) {
            L[0] = make_key(d0, entrypoint);
            vis_insert(c.visited, vis_slots, entrypoint);
        }
        __syncwarp();
        if constexpr (FILT) {
            if (admit) {
                adm->n = 0;
                admit_offer(*adm, entrypoint, d0, lane == 0, lane);
            }
        }
    }
    uint32_t n = 1;
    uint32_t n_exp = 0;
    uint32_t cursor = 0;
    uint32_t pos_thr = 0;
    uint32_t thr_bits = 0;

    while (true) {
        // ---- pq.pop(): first unexpanded entry at or after the cursor ----
        int px = -1;
        for (uint32_t base = cursor & ~31u; base < n; base += 32) {
            const uint32_t j = base + lane;
            const bool un = (j < n) && (j >= cursor) && !(L[j] >> 63);
            const unsigned m = __ballot_sync(kFullMask, un);
            if (m) {
                px = base + __ffs(m) - 1;
                break;
            }
        }
        if (px < 0) break;  // pq empty
        const unsigned long long x = L[px];
        const uint32_t xid = key_id(x);
        if (n_exp >= ef && key_dbits(x) > thr_bits) break;  // res.is_full() && d > res.peek().0  (:1019-1021)

        // ---- res.push((d, idx)) (:1023; max_size_heap.rs:18-32) ----
        __syncwarp();
        if (lane == 0) L[px] = x | kFlagExpanded;
        __syncwarp();
        cursor = px + 1;
        n_exp += 1;
        if (n_exp == ef) {
            // res just became full: res.peek() is the last expanded entry of L
            for (int base = (int)((n - 1) & ~31u); base >= 0; base -= 32) {
                const uint32_t j = base + lane;
                const unsigned m = __ballot_sync(kFullMask, (j < n) && (L[j] >> 63));
                if (m) {
                    pos_thr = base + 31 - __clz(m);
                    break;
                }
            }
            thr_bits = key_dbits(L[pos_thr]);
        } else if (n_exp > ef) {
            n_exp = ef;
            if ((uint32_t)px < pos_thr) {
                // the push evicted res.peek(): the new maximum is the previous expanded entry
                for (int base = (int)((pos_thr - 1) & ~31u); base >= 0; base -= 32) {
                    const uint32_t j = base + lane;
                    const unsigned m = __ballot_sync(kFullMask, (j < pos_thr) && (L[j] >> 63));
                    if (m) {
                        pos_thr = base + 31 - __clz(m);
                        break;
                    }
                }
                thr_bits = key_dbits(L[pos_thr]);
            }
            // else: an equal-distance entry behind res.peek(): expanded but rejected by MaxSizeHeap::push
        }
        c.n_expand += 1;

        // ---- for neighbor in layer.get_neighbors(idx) (:1025-1033) ----
        const uint32_t* row = rows + (size_t)xid * width;
        for (uint32_t w0 = 0; w0 < width; w0 += 32) {
            const uint32_t nb = (w0 + lane < width) ? __ldg(row + w0 + lane) : kUnusedId;
            const bool valid = nb != kUnusedId;
            const unsigned vm = __ballot_sync(kFullMask, valid);
            if (vm == 0) break;  // rows are padded at the end only
            c.n_nbr += __popc(vm);
            const bool is_new = valid && vis_insert(c.visited, vis_slots, nb);
            const unsigned nm = __ballot_sync(kFullMask, is_new);
            const int k = __popc(nm);
            if (k == 0) continue;
            vis_count += k;
            if (vis_count > vis_limit) {
                c.status |= kStatusOverflow;
                *out_n = n;
                return;
            }
            // compact the new ids to lanes 0..k-1 (any order: the push set is order independent, SURVEY §3.1)
            if (is_new) c.ids[__popc(nm & lanemask_lt())] = nb;
            __syncwarp();
            const uint32_t my_id = c.ids[lane < k ? lane : 0];
            c.n_dist += k;
            const float d = dist.dists(ix, c, my_id, k);
            if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
                c.status |= kStatusNotFinite;
                *out_n = n;
                return;
            }
            if constexpr (FILT) {
                if (admit) admit_offer(*adm, my_id, d, lane < k, lane);
            }
            const unsigned long long my_key = make_key(d, my_id);
            // !res.is_full() || distance < res.peek().0   (:1029)
            const bool pass = (lane < k) && (n_exp < ef || key_dbits(my_key) < thr_bits);
            const unsigned pm = __ballot_sync(kFullMask, pass);
            if (pm == 0) continue;
            const uint32_t m = __popc(pm);

            // ---- pq.push for all passing keys at once: rank-based merge into the sorted list ----
            // rank of my key among the current entries (binary search, all lanes in lock step)
            uint32_t lo = 0, hi = n;
            for (int it = 32 - __clz(n); it > 0; --it) {
                const uint32_t mid = (lo + hi) >> 1;
                const bool less = (lo < hi) && ((L[mid < n ? mid : n - 1] & kKeyMask) < my_key);
                if (lo < hi) {
                    if (less)
                        lo = mid + 1;
                    else
                        hi = mid;
                }
            }
            const uint32_t rank_l = lo;
            uint32_t rank_n = 0;  // rank among the passing keys
            for (unsigned t = pm; t; t &= t - 1) {
                const unsigned long long kb = __shfl_sync(kFullMask, my_key, __ffs(t) - 1);
                rank_n += (kb < my_key) ? 1u : 0u;
            }
            const uint32_t new_pos = rank_l + rank_n;
            const uint32_t min_rank = warp_min_u32(kFullMask, pass ? rank_l : 0xFFFFFFFFu);
            const uint32_t total = n + m;
            uint32_t drop_min = 0xFFFFFFFFu;   // smallest distance among dropped entries
            uint32_t drop_flagged = 0;
            // existing entries at positions >= min_rank move up by the number of new keys ranked at or before them;
            // rows are processed top-down so a write never lands on an entry that has not been read yet.
            for (int base = (int)((n - 1) & ~31u); base >= (int)(min_rank & ~31u); base -= 32) {
                const uint32_t j = base + lane;
                const bool in = (j < n) && (j >= min_rank);
                unsigned long long v = 0;
                if (in) v = L[j];
                uint32_t sh = 0;
                for (unsigned t = pm; t; t &= t - 1) {
                    const uint32_t r = __shfl_sync(kFullMask, rank_l, __ffs(t) - 1);
                    sh += (r <= j) ? 1u : 0u;
                }
                const uint32_t np = j + sh;
                __syncwarp();
                if (in && np < cap) L[np] = v;
                if (total > cap) {
                    const bool dropped = in && np >= cap;
                    const unsigned dm = __ballot_sync(kFullMask, dropped);
                    if (dm) {
                        drop_flagged += __popc(__ballot_sync(kFullMask, dropped && (v >> 63)));
                        drop_min = min(drop_min, warp_min_u32(kFullMask, dropped ? key_dbits(v) : 0xFFFFFFFFu));
                    }
                }
            }
            __syncwarp();
            if (pass && new_pos < cap) L[new_pos] = my_key;
            __syncwarp();
            if (total > cap) {
                drop_min = min(drop_min, warp_min_u32(kFullMask, (pass && new_pos >= cap) ? key_dbits(my_key)
                                                                                            : 0xFFFFFFFFu));
                n = cap;
                // an entry may leave L only if >= ef strictly closer entries remain (see "Exactness")
                if (!(key_dbits(L[ef - 1]) < drop_min)) {
                    c.status |= kStatusOverflow;
                    *out_n = n;
                    return;
                }
                if (n_exp >= ef) {
                    if (pos_thr + m >= cap) {
                        // res.peek() itself left L: res now spans evicted entries ("not full" regime); recount
                        uint32_t cnt = 0;
                        for (uint32_t base = 0; base < n; base += 32) {
                            const uint32_t j = base + lane;
                            cnt += __popc(__ballot_sync(kFullMask, (j < n) && (L[j] >> 63)));
                        }
                        n_exp = cnt < ef ? cnt : ef - 1;
                    } else {
                        pos_thr += m;  // every passing key is closer than res.peek()
                    }
                } else {
                    n_exp -= drop_flagged;
                }
            } else {
                n = total;
                if (n_exp >= ef) pos_thr += m;
            }
            const uint32_t min_pos = warp_min_u32(kFullMask, pass ? new_pos : 0xFFFFFFFFu);
            if (min_pos < cursor) cursor = min_pos;
        }
    }
    *out_n = n;
}

// ------------------------------------------------------------------------------------------------------------------
// search_for_neighbors, fast variant: same state machine as search_layer (above) with a cheaper list representation.
//   * keys are split into two u32 arrays in SHARED memory (`Ld` must point into the kernel's shared window so that
//     every access is an LDS/STS with a 32-bit address): Ld[j] = distance bits | expanded flag (bit 31), Li[j] = id,
//     sorted by (distance, id); capacity 32*R, position j lives in bank j % 32 (row-major: row r = positions
//     [32r, 32r+32)); Ld is padded to a power of two with flagged +inf-like sentinels, so the rank search is a
//     branch-free lower bound and the pop scan needs no length check;
//   * all passing keys of one expansion are merged in one pass: every lane ranks its key among the old entries
//     (lower bound) and among the other new keys (compare loop over the keys parked in shared memory), which gives the
//     final position of every new key; the rows of the list at or after the first insertion point are then rebuilt
//     top-down as a GATHER: output position p either receives a new key or the old entry p - (#new keys below p),
//     where the count comes from a per-row occupancy mask (REDUX.OR) and popc — one LDS/STS pair per array and row;
//   * keys strictly farther than the tail of a full list are dropped up front (they can never matter);
//   * the visited set is the bucketed global-memory table (vis_bucket_insert): one 16-byte load per neighbour.
// ------------------------------------------------------------------------------------------------------------------
__host__ __device__ constexpr uint32_t fast_list_pow2(int R) {
    uint32_t p = 32;
    while (p <= 32u * (uint32_t)R) p <<= 1;
    return p;
}
// bytes of shared memory the fast list needs: Ld[P] + Li[32*R]
__host__ __device__ constexpr uint32_t fast_list_bytes(int R) { return (fast_list_pow2(R) + 32u * (uint32_t)R) * 4u; }

// FILT: `adm` receives every candidate this layer scores (admit_offer); only the bottom layer is searched with it.
template <class Dist, int R, bool FILT = false>
__device__ __forceinline__ void search_layer_fast(const DeviceIndex& ix, WarpCtx& c, Dist& dist, uint32_t* Ld,
                                                  const uint32_t* rows, const uint32_t width,
                                                  const uint32_t entrypoint, const uint32_t ef,
                                                  const uint32_t vis_slots, uint32_t* out_n,
                                                  AdmitList* adm = nullptr) {
    constexpr uint32_t cap = 32u * R;
    constexpr uint32_t P = fast_list_pow2(R);  // Ld is padded to a power of two > cap with sentinels
    constexpr uint32_t kFlag = 0x80000000u, kDMask = 0x7FFFFFFFu;
    uint32_t* Li = Ld + P;
    const int lane = c.lane;
    const unsigned lt = lanemask_lt();
    const uint32_t nbuckets = vis_slots >> 2;
    {
        uint4* v4 = reinterpret_cast<uint4*>(c.visited);
        const uint4 e = make_uint4(kUnusedId, kUnusedId, kUnusedId, kUnusedId);
        for (uint32_t i = lane; i < nbuckets; i += 32) stcg_u4(v4 + i, e, c.pol_keep);
    }
    // sentinel: masked distance larger than any real one; flagged, so the pop scan never selects it
    for (uint32_t i = lane; i < P; i += 32) Ld[i] = 0xFFFFFFFFu;
    __syncwarp();
    const uint32_t vis_limit = vis_slots - (vis_slots >> 2);  // keep the bucket load factor <= 3/4
    uint32_t vis_count = 1;

    {
        const float d0 = dist.dists(ix, c, entrypoint, 1);
        c.n_dist += 1;
        if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
            c.status |= kStatusNotFinite;
            *out_n = 0;
            return;
        }
        bool ovf = false;
        vis_bucket_insert(c.visited, nbuckets, entrypoint, lane == 0, &ovf, c.pol_keep);
        if (lane == 0) {
            Ld[0] = __float_as_uint(d0);
            Li[0] = entrypoint;
        }
        __syncwarp();
        if constexpr (FILT) {
            adm->n = 0;
            admit_offer(*adm, entrypoint, d0, lane == 0, lane);
        }
    }
    uint32_t n = 1, n_exp = 0, cursor = 0, pos_thr = 0, thr_bits = 0;
    uint32_t spec_id = kUnusedId, spec_slot = 0;
    bool spec_bk = false;  // the speculative row's home buckets were copied (valid until the next insertion)
    uint32_t* const spec_rows = c.ids + 32;
    uint4* const spec_buckets = reinterpret_cast<uint4*>(c.ids + 96);

    while (true) {
        // ---- pq.pop(): first unexpanded entry at or after the cursor; also find the runner-up ----
        int px = -1;
        uint32_t base_sel = cursor & ~31u;
        unsigned sel_mask = 0;
        for (; base_sel < n; base_sel += 32) {
            const uint32_t j = base_sel + lane;
            sel_mask = __ballot_sync(kFullMask, (j >= cursor) && !(Ld[j] & kFlag));  // positions >= n are flagged
            if (sel_mask) {
                px = base_sel + __ffs(sel_mask) - 1;
                break;
            }
        }
        if (px < 0) break;
        const uint32_t xd = Ld[px];  // unflagged
        const uint32_t xid = Li[px];
        if (n_exp >= ef && xd > thr_bits) break;
        // Speculation: the runner-up of this pop (next unexpanded entry of the same 32-entry row) is the most likely
        // next expansion.  Its adjacency row (one lane = one neighbour, width <= 32) is fetched NOW with cp.async
        // into one of two shared slots so that the load latency overlaps this whole expansion; a wrong guess only
        // costs the load.  (A register destination would not work: the consumer of the previous speculation would
        // wait on the same scoreboard as the load issued here.)  Every pop commits exactly one — possibly empty —
        // group, so "all groups but the last" at the consumer is precisely the previous pop's row.
        const bool have_cur = (spec_id == xid) && (width <= 32u);
        const bool have_bk = have_cur && spec_bk;
        const uint32_t* cur_row = spec_rows + 32u * spec_slot;
        spec_id = kUnusedId;
        spec_bk = false;
        {
            const unsigned rest = sel_mask & (sel_mask - 1);
            if (rest && width <= 32u) {
                // the slot written now was last written two pops ago; if no distance phase (and so no wait) happened
                // since, that copy could still be in flight and land AFTER this one — wait for all but the last group
                cp_async_wait_but_last();
                spec_slot ^= 1u;
                spec_id = Li[base_sel + __ffs(rest) - 1];
                if ((uint32_t)lane < width)
                    cp_async_lane<4>(smem_u32(spec_rows + 32u * spec_slot + lane), rows + (size_t)spec_id * width + lane);
            }
            cp_async_commit();
        }

        // ---- res.push ----
        __syncwarp();
        if (lane == 0) Ld[px] = xd | kFlag;
        __syncwarp();
        cursor = px + 1;
        n_exp += 1;
        if (n_exp == ef) {
            for (int base = (int)((n - 1) & ~31u); base >= 0; base -= 32) {
                const uint32_t j = base + lane;
                const unsigned m = __ballot_sync(kFullMask, (j < n) && (Ld[j] & kFlag));
                if (m) {
                    pos_thr = base + 31 - __clz(m);
                    break;
                }
            }
            thr_bits = Ld[pos_thr] & kDMask;
        } else if (n_exp > ef) {
            n_exp = ef;
            if ((uint32_t)px < pos_thr) {
                for (int base = (int)((pos_thr - 1) & ~31u); base >= 0; base -= 32) {
                    const uint32_t j = base + lane;
                    const unsigned m = __ballot_sync(kFullMask, (j < pos_thr) && (Ld[j] & kFlag));
                    if (m) {
                        pos_thr = base + 31 - __clz(m);
                        break;
                    }
                }
                thr_bits = Ld[pos_thr] & kDMask;
            }
        }
        c.n_expand += 1;

        // ---- neighbours ----
        const uint32_t* row = rows + (size_t)xid * width;
        for (uint32_t w0 = 0; w0 < width; w0 += 32) {
            uint32_t nb = kUnusedId;
            if (have_cur) {
                cp_async_wait_but_last();
                if ((uint32_t)lane < width) nb = cur_row[lane];
            } else if (w0 + lane < width) {
                nb = __ldg(row + w0 + lane);
            }
            const bool valid = nb != kUnusedId;
            const unsigned vm = __ballot_sync(kFullMask, valid);
            if (vm == 0) break;
            c.n_nbr += __popc(vm);
            bool ovf = false;
            const bool is_new = vis_bucket_insert(c.visited, nbuckets, nb, valid, &ovf, c.pol_keep,
                                                  have_bk ? spec_buckets : nullptr);
            const unsigned nm = __ballot_sync(kFullMask, is_new);
            const int k = __popc(nm);
            vis_count += k;
            if (ovf || vis_count > vis_limit) {  // (ovf is warp-uniform: it is set on a uniform path of the probe loop)
                c.status |= kStatusOverflow;
                *out_n = n;
                return;
            }
            if (k == 0) continue;
            if (is_new) c.ids[__popc(nm & lt)] = nb;
            __syncwarp();
            const uint32_t my_id = c.ids[lane < k ? lane : 0];
            c.n_dist += k;
            // While this expansion's candidate rows are in flight the speculative adjacency row lands too; as soon as
            // the wait is over (inside dists) its neighbours' home buckets are copied from the visited table into
            // shared memory, so that a correct guess finds them there instead of paying an L2 round trip.  The
            // copies are issued after this expansion's insertions and no insertion follows before they are used.
            const float d = dist.dists(ix, c, my_id, k, [&] {
                if (spec_id != kUnusedId) {
                    cp_async_wait_all();
                    const uint32_t sn = ((uint32_t)lane < width) ? spec_rows[32u * spec_slot + lane] : kUnusedId;
                    cp_async_lane<16>(smem_u32(spec_buckets + lane),
                                      c.visited + (size_t)__umulhi(sn * kVisHashMul, nbuckets) * 4u);
                    cp_async_commit();  // its own group: the consumer waits for all groups but the next pop's
                    spec_bk = true;
                }
            }, c.ids);
            if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
                c.status |= kStatusNotFinite;
                *out_n = n;
                return;
            }
            if constexpr (FILT) admit_offer(*adm, my_id, d, lane < k, lane);
            const uint32_t my_d = __float_as_uint(d);
            // !res.is_full() || distance < res.peek().0   (:1029)
            bool pass = (lane < k) && (n_exp < ef || my_d < thr_bits);
            // a key strictly farther than the last entry of a full list has >= ef strictly closer entries before
            // it (cap > ef): it can never be expanded nor reported, so it need not enter the list at all
            if (n == cap) pass = pass && !(my_d > (Ld[cap - 1] & kDMask));
            const unsigned pm = __ballot_sync(kFullMask, pass);
            if (pm == 0) continue;
            const uint32_t m = __popc(pm);

            // park the passing keys (compacted) in shared memory: key t = (id, distance bits) as one 64-bit word
            uint2* keys = reinterpret_cast<uint2*>(c.tile);
            if (pass) keys[__popc(pm & lt)] = make_uint2(my_id, my_d);
            // rank of my key among the entries: branch-free lower bound on the distance over the padded array
            // (entries at positions >= n are sentinels), refined by id on exact distance ties
            uint32_t lo = 0;
#pragma unroll
            for (uint32_t step = P / 2; step >= 1; step >>= 1)
                if ((Ld[lo + step - 1] & kDMask) < my_d) lo += step;
            while (lo < n && (Ld[lo] & kDMask) == my_d && Li[lo] < my_id) ++lo;  // (d, id) tuple order
            __syncwarp();
            // rank among the new keys (ids are distinct, so the 64-bit (distance, id) keys are too)
            uint32_t rank_n = 0;
            for (uint32_t t = 0; t < m; ++t) {
                const uint2 kt = keys[t];
                rank_n += (kt.y < my_d || (kt.y == my_d && kt.x < my_id)) ? 1u : 0u;
            }
            const uint32_t new_pos = lo + rank_n;
            const uint32_t total = n + m;
            const uint32_t min_pos = warp_min_u32(kFullMask, pass ? new_pos : 0xFFFFFFFFu);
            uint32_t drop_flagged = 0, mdrop = 0;
            if (total > cap) {
                // the last (total - cap) positions of the merged order fall off: mdrop new keys and odrop old entries
                mdrop = __popc(__ballot_sync(kFullMask, pass && new_pos >= cap));
                const uint32_t odrop = (total - cap) - mdrop;
                const uint32_t j = n - odrop + lane;
                drop_flagged = __popc(__ballot_sync(kFullMask, ((uint32_t)lane < odrop) && (Ld[j] >> 31)));
            }
            const uint32_t kept = total > cap ? cap : total;
            // rebuild rows top-down: output position p takes the old entry p - (#new keys below p) unless a new key
            // lands there.  A row only reads old positions <= its own, so writing it after a barrier is race free.
            {
                uint32_t kge = mdrop;  // new keys at positions >= the end of the current row
                const int rt = (int)((kept - 1) >> 5), rbm = (int)(min_pos >> 5);
#pragma unroll
                for (int r = R - 1; r >= 0; --r) {
                    if (r > rt || r < rbm) continue;
                    const unsigned occ = __reduce_or_sync(
                        kFullMask, (pass && (new_pos >> 5) == (uint32_t)r) ? (1u << (new_pos & 31)) : 0u);
                    kge += __popc(occ);
                    const uint32_t p = 32u * r + lane;
                    const uint32_t below = (m - kge) + __popc(occ & lt);  // new keys at positions < p
                    const bool old = !((occ >> lane) & 1u) && p < kept && p >= min_pos;
                    uint32_t vd = 0, vi = 0;
                    if (old) {
                        vd = Ld[p - below];
                        vi = Li[p - below];
                    }
                    __syncwarp();
                    if (old) {
                        Ld[p] = vd;
                        Li[p] = vi;
                    }
                }
            }
            if (pass && new_pos < cap) {
                Ld[new_pos] = my_d;
                Li[new_pos] = my_id;
            }
            __syncwarp();
            if (total > cap) {
                n = cap;
                // entries fell off the end: legal only if >= ef strictly closer entries remain; everything dropped is
                // >= the last kept entry, so "L[ef-1].d < L[cap-1].d" is sufficient (else: retry / slow path)
                if (!((Ld[ef - 1] & kDMask) < (Ld[cap - 1] & kDMask))) {
                    c.status |= kStatusOverflow;
                    *out_n = n;
                    return;
                }
                if (n_exp >= ef) {
                    if (pos_thr + m >= cap) {
                        // res.peek() itself left L: res now spans evicted entries ("not full" regime); recount
                        uint32_t cnt = 0;
                        for (uint32_t base = 0; base < n; base += 32) {
                            const uint32_t j = base + lane;
                            cnt += __popc(__ballot_sync(kFullMask, (j < n) && (Ld[j] & kFlag)));
                        }
                        n_exp = cnt < ef ? cnt : ef - 1;
                    } else {
                        pos_thr += m;
                    }
                } else {
                    n_exp -= drop_flagged;
                }
            } else {
                n = total;
                if (n_exp >= ef) pos_thr += m;
            }
            if (min_pos < cursor) cursor = min_pos;
        }
    }
    *out_n = n;
}

// ElementContainer::get(id) written into the query slot c.qs (natural layout; i8: zero padded words + q_norm_i8).
// Used by the builder (queries are elements of the container, src/index/mod.rs:817) and get_element.
__device__ __forceinline__ void load_element_to_qs(const DeviceIndex& ix, WarpCtx& c, uint32_t id) {
    const int lane = c.lane;
    const uint32_t dim = ix.dim;
    __syncwarp();
    if (ix.kind == kAngularI8) {
        int* qw = reinterpret_cast<int*>(c.qs);
        const int* row = reinterpret_cast<const int*>(static_cast<const int8_t*>(ix.vectors) +
                                                      (size_t)id * ix.row_stride);
        const int words = ix.row_stride / 4;
        int dy = 0;
        for (int w = lane; w < words; w += 32) {
            const int v = __ldg(row + w);
            qw[w] = v;
            dy = __dp4a(v, v, dy);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dy += __shfl_xor_sync(kFullMask, dy, o);
        c.q_norm_i8 = dy;
    } else if (ix.kind == kAngularF32) {
        const float* row = static_cast<const float*>(ix.vectors) + (size_t)id * ix.row_stride;
        const uint32_t V = ix.vec_group;
        for (uint32_t e = lane; e < dim; e += 32) {
            uint32_t o = e;
            if (e < ix.full * 32) o = permuted_offset(e, V);
            c.qs[e] = __ldg(row + o);
        }
    } else {
        DistSum::materialise(ix, c, id);
        for (uint32_t e = lane; e < dim; e += 32) c.qs[e] = c.xs[e];
    }
    __syncwarp();
}

// ElementContainer::get(id) -> the query slot (c.qs / q registers) of the distance engine (the builder's
// select_neighbors and add_and_limit, and diverse_kernel).
template <class Dist>
__device__ __forceinline__ void set_query_from_element(const DeviceIndex& ix, WarpCtx& c, Dist& dist, uint32_t id) {
    load_element_to_qs(ix, c, id);
    dist.load_query(ix, c);
}

// ------------------------------------------------------------------------------------------------------------------
// query construction (the `Elements::Element` the reference's callers build)
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void prepare_query(const DeviceIndex& ix, const SearchArgs& a, WarpCtx& c,
                                              unsigned long long qi) {
    const int dim = ix.dim, lane = c.lane;
    if (a.query_format == kQueryById) {
        load_element_to_qs(ix, c, static_cast<const uint32_t*>(a.queries)[qi]);
        return;
    }
    if (ix.kind == kAngularI8) {
        int* qw = reinterpret_cast<int*>(c.qs);
        int8_t* qb = reinterpret_cast<int8_t*>(c.qs);
        const int words = ix.row_stride / 4;
        for (int w = lane; w < words; w += 32) qw[w] = 0;
        __syncwarp();
        if (a.query_format == kQueryElement) {
            const int8_t* src = static_cast<const int8_t*>(a.queries) + qi * dim;
            for (int i = lane; i < dim; i += 32) qb[i] = src[i];
        } else {
            // Vector::from(Vec<f32>) -> quantize; NaN input is an error (NotNan max)
            quantize_i8(static_cast<const float*>(a.queries) + qi * dim, qb, dim, lane, &c.status);
        }
        __syncwarp();
        int dy = 0;
        for (int w = lane; w < words; w += 32) dy = __dp4a(qw[w], qw[w], dy);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dy += __shfl_xor_sync(kFullMask, dy, o);
        c.q_norm_i8 = dy;
    } else {
        const float* src = static_cast<const float*>(a.queries) + qi * dim;
        for (int i = lane; i < dim; i += 32) c.qs[i] = src[i];
        __syncwarp();
        if (a.query_format == kQueryRawF32)
            normalize_f32(c.qs, dim, (int)ix.full, lane);  // Vector::from(Vec<f32>) (angular.rs:55-61)
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Granne::search for a batch (src/index/mod.rs:140-150, 962-997): persistent warps over a work counter.
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_result(const SearchArgs& a, unsigned long long qi, uint32_t k, uint32_t r,
                                             uint32_t id, float d) {
    if (a.pg.n_peers) {
        const size_t o = (size_t)(a.pg.row_offset + qi) * k + r;
#pragma unroll 1
        for (uint32_t p = 0; p < a.pg.n_peers; ++p) {
            a.pg.ids[p][o] = id;
            a.pg.dists[p][o] = d;
        }
    } else {
        a.out_ids[qi * k + r] = id;
        a.out_dists[qi * k + r] = d;
    }
}

// flags[p][my_rank] = seq for every peer, released system-wide
__device__ __forceinline__ void publish_seq(const PeerGather& pg) {
    for (uint32_t p = 0; p < pg.n_peers; ++p)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(pg.flags[p] + pg.my_rank), "r"(pg.seq) : "memory");
}

// Called by every CTA of the LAST kernel of a search (the slow pass) before it exits: once all CTAs are through,
// publish the sequence number to every peer.
__device__ __forceinline__ void signal_peers(const SearchArgs& a, int lane) {
    if (!a.pg.n_peers) return;
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
        const unsigned int old = atomicAdd(a.pg.done_counter, 1u);
        if (old == gridDim.x - 1) {
            __threadfence_system();
            publish_seq(a.pg);
        }
    }
}

// A gather call without queries has no stores to wait for, but its peers still wait for its sequence number.
__global__ void publish_seq_kernel(const PeerGather pg) {
    __threadfence_system();
    publish_seq(pg);
}

// Resident one-warp CTAs per SM the filtered fast kernel is register-limited to.  The admitted list's state costs a
// few registers, which the widest fixed f32 engine and the embeddings engine cannot spare under GB_MIN_BLOCKS's cap
// without spilling to local memory (DistSum already spills there unfiltered).
template <class Dist>
struct FilteredMinBlocks {
    static constexpr int value = GB_MIN_BLOCKS;
};
template <>
struct FilteredMinBlocks<DistF32<8>> {
    static constexpr int value = 20;
};
template <>
struct FilteredMinBlocks<DistSum> {
    static constexpr int value = 16;
};

// R == 0: generic list (64-bit keys, any capacity, shared or global memory) — the slow pass and very large max_search.
// R  > 0: fast list with capacity 32*R for the bottom layer (upper layers always use R = 1).
// FILT: filtered search (SearchArgs' filter fields): the same traversal, counters and pass ladder, with the bottom
// layer's scored candidates offered to an admitted list (AdmitList) that the results are written from.
template <class Dist, int R, bool FILT = false>
__global__ void __launch_bounds__(32, R > 0 ? (FILT ? FilteredMinBlocks<Dist>::value : GB_MIN_BLOCKS) : 1)
    search_kernel(const DeviceIndex ix, const SearchArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    c.lane = threadIdx.x;
    // shared layout: SmemLayout | list            (fast pass: visited set in global)
    //                SmemLayout | list | visited  (generic pass, slow_pass == 0)
    // The SmemLayout walk is spelled out here rather than called through place_warp_smem: the call compiles to a
    // differently scheduled prologue, and this kernel runs at its register cap.
    unsigned char* sp = smem_raw;
    c.tile = reinterpret_cast<float*>(sp);
    c.ids = reinterpret_cast<uint32_t*>(sp + tile_bytes_for_rows(a.tiles.tile_rows) - kIdScratchBytes);
    sp += tile_bytes_for_rows(a.tiles.tile_rows);
    c.pol_keep = make_policy_evict_last();
    sp += SmemLayout<unsigned char*>::kReservedBytes;
    const uint32_t qbytes = (ix.kind == kAngularI8) ? ix.row_stride : ((ix.dim + 3u) & ~3u) * 4u;
    c.qs = reinterpret_cast<float*>(sp);
    sp += (qbytes + 15u) & ~15u;
    c.xs = reinterpret_cast<float*>(sp);
    if (ix.kind == kSumEmbeddings) sp += (qbytes + 15u) & ~15u;
    c.stg = nullptr;
    c.stg_rows = a.tiles.stg_rows;
    c.stg_row_bytes = a.tiles.stg_row_bytes;
    if (a.tiles.stg_rows) {  // staging tile: gathered candidate rows (f32 / i8) or summed candidates (embeddings)
        sp = smem_raw + (((size_t)(sp - smem_raw) + 127u) & ~(size_t)127u);
        c.stg = sp;
        sp += (size_t)a.tiles.stg_rows * a.tiles.stg_row_bytes;
    }
    // the fast list always lives in this CTA's shared window (derived from smem_raw only, so that the compiler keeps
    // its accesses in the shared address space: LDS/STS with 32-bit addresses)
    uint32_t* const fast_list = reinterpret_cast<uint32_t*>(sp);
    uint32_t list_cap, vis_slots, vis_upper;
    if (a.slow_pass) {
        c.list = a.slow_list + (size_t)blockIdx.x * a.slow_list_cap;
        c.visited = a.slow_visited + (size_t)blockIdx.x * a.slow_vis_slots;
        list_cap = a.slow_list_cap;
        vis_slots = a.slow_vis_slots;
        vis_upper = a.slow_vis_slots < (1u << 16) ? a.slow_vis_slots : (1u << 16);  // max_search = 1 descents stay small
    } else {
        c.list = reinterpret_cast<unsigned long long*>(sp);
        list_cap = a.list_cap;
        vis_slots = a.vis_slots;
        vis_upper = a.vis_slots_upper;
        if (R > 0) {
            c.visited = a.vis_global + (size_t)blockIdx.x * a.vis_slots;
        } else {
            sp += (size_t)a.list_cap * sizeof(unsigned long long);
            c.visited = reinterpret_cast<uint32_t*>(sp);
        }
    }
    AdmitList adm;
    if constexpr (FILT) {
        // behind the pass's own shared memory: the fast list, or the generic list and visited set (the slow pass
        // keeps both in global memory)
        unsigned char* ap = sp;
        if (!a.slow_pass) ap += R > 0 ? (size_t)fast_list_bytes(R > 0 ? R : 1) : (size_t)a.vis_slots * 4u;
        adm.keys = reinterpret_cast<unsigned long long*>(ap);
        adm.cap = a.filter_cap;
        adm.bit_base = a.filter_bit_base;
        adm.n = 0;
    }
    Dist dist;
    if (a.pass && *reinterpret_cast<volatile unsigned int*>(a.gate_in) == 0u) {  // nothing flagged
        if (a.final_pass) signal_peers(a, c.lane);
        return;
    }

    while (true) {
        unsigned int qi0 = 0;
        if (c.lane == 0) qi0 = atomicAdd(a.work_counter, 1u);
        const unsigned long long qi = __shfl_sync(kFullMask, qi0, 0);
        if (qi >= a.nq) break;
        if (a.pass && a.query_status[qi] != kStatusOverflow) continue;  // only flagged queries
        if (a.pass == 1 && a.retried && c.lane == 0) atomicAdd(a.retried, 1ull);

        c.status = 0;
        c.n_dist = c.n_expand = c.n_nbr = 0;
        c.q_norm_i8 = 0;
        prepare_query(ix, a, c, qi);
        dist.load_query(ix, c);
        if constexpr (FILT) {
            const uint32_t f = a.query_filter ? a.query_filter[qi] : 0u;
            if (f >= a.num_filters) c.status |= kStatusBadFilter;
            adm.bits = a.filters + (size_t)(f < a.num_filters ? f : 0u) * a.filter_words;
            adm.n = 0;
        }

        uint32_t n = 0;
        const uint32_t k = a.num_neighbors;
        uint32_t found = 0;
        if (ix.num_layers > 0 && !(c.status & (FILT ? kStatusNotFinite | kStatusBadFilter : kStatusNotFinite))) {
            // find_entrypoint (:984-997): max_search = 1 descent through the upper layers, then the bottom layer
            // with the caller's max_search (:970-973).
            uint32_t entrypoint = 0;
            const int bl = ix.num_layers - 1;
            if (R == 0) {
                const uint32_t cap1 = list_cap < 32 ? list_cap : 32;
                for (int l = 0; l <= bl && c.status == 0; ++l) {
                    const bool bottom = (l == bl);
                    search_layer<Dist, FILT>(ix, c, dist, ix.layer_rows[l], ix.layer_width[l], entrypoint,
                                             bottom ? a.max_search : 1u, bottom ? list_cap : cap1,
                                             bottom ? vis_slots : vis_upper, &n, &adm, bottom);
                    if (bottom || c.status) break;
                    uint32_t ep = 0;  // res[0]: first expanded entry
                    for (uint32_t base = 0; base < n; base += 32) {
                        const uint32_t j = base + c.lane;
                        const unsigned m = __ballot_sync(kFullMask, (j < n) && (c.list[j] >> 63));
                        if (m) {
                            ep = key_id(c.list[base + __ffs(m) - 1]);
                            break;
                        }
                    }
                    entrypoint = ep;
                }
                if (c.status == 0 && !FILT) {
                    // res.into_sorted_vec().take(num_neighbors) (:974-977, :1036)
                    const uint32_t limit = a.max_search < k ? a.max_search : k;
                    uint32_t cnt = 0;
                    for (uint32_t base = 0; base < n && cnt < limit; base += 32) {
                        const uint32_t j = base + c.lane;
                        unsigned long long v = 0;
                        if (j < n) v = c.list[j];
                        const bool fl = (j < n) && (v >> 63);
                        const unsigned m = __ballot_sync(kFullMask, fl);
                        const uint32_t rank = cnt + __popc(m & lanemask_lt());
                        if (fl && rank < limit) store_result(a, qi, k, rank, key_id(v), __uint_as_float(key_dbits(v)));
                        cnt += __popc(m);
                    }
                    found = cnt < limit ? cnt : limit;
                }
            } else {
                constexpr int RB = R > 0 ? R : 1;
                const uint32_t* Ld = fast_list;
                for (int l = 0; l < bl && c.status == 0; ++l) {
                    search_layer_fast<Dist, 1>(ix, c, dist, fast_list, ix.layer_rows[l], ix.layer_width[l],
                                               entrypoint, 1u, vis_upper, &n);
                    if (c.status) break;
                    uint32_t ep = 0;  // res[0] (capacity 32: a single row)
                    const unsigned m = __ballot_sync(kFullMask, ((uint32_t)c.lane < n) && (Ld[c.lane] >> 31));
                    if (m) ep = Ld[fast_list_pow2(1) + __ffs(m) - 1];  // Li = Ld + P for R = 1
                    entrypoint = ep;
                }
                if (c.status == 0)
                    search_layer_fast<Dist, RB, FILT>(ix, c, dist, fast_list, ix.layer_rows[bl], ix.layer_width[bl],
                                                      entrypoint, a.max_search, vis_slots, &n, &adm);
                if (c.status == 0 && !FILT) {
                    const uint32_t* Li = Ld + fast_list_pow2(RB);
                    const uint32_t limit = a.max_search < k ? a.max_search : k;
                    uint32_t cnt = 0;
                    for (uint32_t base = 0; base < n && cnt < limit; base += 32) {
                        const uint32_t j = base + c.lane;
                        uint32_t v = 0;
                        if (j < n) v = Ld[j];
                        const bool fl = (j < n) && (v >> 31);
                        const unsigned m = __ballot_sync(kFullMask, fl);
                        const uint32_t rank = cnt + __popc(m & lanemask_lt());
                        if (fl && rank < limit) store_result(a, qi, k, rank, Li[j], __uint_as_float(v & 0x7FFFFFFFu));
                        cnt += __popc(m);
                    }
                    found = cnt < limit ? cnt : limit;
                }
            }
            if constexpr (FILT) {
                // the first min(k, n) admitted keys (k may exceed max_search)
                if (c.status == 0) {
                    found = adm.n < k ? adm.n : k;
                    for (uint32_t r = c.lane; r < found; r += 32) {
                        const unsigned long long v = adm.keys[r];
                        store_result(a, qi, k, r, key_id(v), __uint_as_float(key_dbits(v)));
                    }
                }
            }
        }
        if constexpr (FILT) {
            if (c.status & kStatusBadFilter) {
                found = 0;
                if (c.lane == 0) atomicOr(a.error_flag, kStatusBadFilter);
            }
        }
        if (c.status & kStatusOverflow) {
            // leave the outputs to the slow path (or report capacity exhaustion if this IS the slow path)
            if (c.lane == 0) {
                a.query_status[qi] = a.final_pass ? (kStatusOverflow | 4) : kStatusOverflow;
                if (a.final_pass)
                    atomicOr(a.error_flag, kStatusOverflow);
                else
                    atomicExch(a.gate_out, 1u);
            }
            if (!a.final_pass) continue;
            found = 0;
        }
        if (c.status & kStatusNotFinite) {
            found = 0;
            if (c.lane == 0) atomicOr(a.error_flag, kStatusNotFinite);
        }
        for (uint32_t r = found + c.lane; r < k; r += 32) store_result(a, qi, k, r, kUnusedId, __int_as_float(0x7f800000));
        if (c.lane == 0) {
            if (a.out_counts) a.out_counts[qi] = found;
            if (a.out_stats) {
                a.out_stats[qi * 4 + 0] = c.n_dist;
                a.out_stats[qi * 4 + 1] = c.n_expand;
                a.out_stats[qi * 4 + 2] = c.n_nbr;
                a.out_stats[qi * 4 + 3] = (unsigned long long)a.pass;
            }
            if (!(c.status & kStatusOverflow)) a.query_status[qi] = 0;
        }
    }
    if (a.final_pass) signal_peers(a, c.lane);
}

// ------------------------------------------------------------------------------------------------------------------
// staging / utility kernels
// ------------------------------------------------------------------------------------------------------------------

// Row-major f32 rows -> lane-permuted HBM layout: element (chunk c, lane i) of a row moves to
// g*32*V + i*V + v with c = g*V + v; the tail (dim % 32) stays in place; the row is padded to `stride` floats.
__global__ void permute_rows_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, uint64_t nrows,
                                        uint32_t dim, uint32_t full, uint32_t V, uint32_t stride) {
    const uint64_t total = nrows * stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total;
         t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / stride;
        const uint32_t o = (uint32_t)(t % stride);
        float v = 0.0f;
        if (o < full * 32) {
            const uint32_t g = o / (32 * V), rem = o % (32 * V);
            const uint32_t i = rem / V, vv = rem % V;
            v = src[r * dim + (g * V + vv) * 32 + i];
        } else if (o < dim) {
            v = src[r * dim + o];
        }
        dst[t] = v;
    }
}

__global__ void pad_rows_i8_kernel(const int8_t* __restrict__ src, int8_t* __restrict__ dst, uint64_t nrows,
                                   uint32_t dim, uint32_t stride) {
    const uint64_t total = nrows * stride;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total;
         t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = t / stride;
        const uint32_t o = (uint32_t)(t % stride);
        dst[t] = o < dim ? src[r * dim + o] : (int8_t)0;
    }
}

// ElementContainer::get(idx) for one element -> `out` (dim f32, or dim i8)
__global__ void __launch_bounds__(32) get_element_kernel(const DeviceIndex ix, unsigned long long idx, void* out) {
    __shared__ float xs[4096];
    const int lane = threadIdx.x;
    const uint32_t dim = ix.dim;
    if (ix.kind == kAngularI8) {
        const int8_t* row = static_cast<const int8_t*>(ix.vectors) + idx * ix.row_stride;
        for (uint32_t i = lane; i < dim; i += 32) static_cast<int8_t*>(out)[i] = row[i];
    } else if (ix.kind == kAngularF32) {
        const float* row = static_cast<const float*>(ix.vectors) + idx * ix.row_stride;
        for (uint32_t e = lane; e < dim; e += 32)
            static_cast<float*>(out)[e] = row[e < ix.full * 32 ? permuted_offset(e, ix.vec_group) : e];
    } else {
        WarpCtx c;
        c.lane = lane;
        c.xs = xs;
        c.status = 0;
        if (dim <= 4096) {
            DistSum::materialise(ix, c, (uint32_t)idx);
            for (uint32_t i = lane; i < dim; i += 32) static_cast<float*>(out)[i] = xs[i];
        }
    }
}

// k-way merge of per-shard result tiles by (distance, global id) — range-partitioned mode (SURVEY.md §8e).
// One thread per query; parts*k is small (<= a few hundred).
__global__ void merge_topk_kernel(const uint32_t* __restrict__ part_ids, const float* __restrict__ part_dists,
                                  const unsigned long long* __restrict__ part_base, uint32_t num_parts,
                                  unsigned long long nq, uint32_t k, unsigned long long* __restrict__ out_ids,
                                  float* __restrict__ out_dists) {
    const unsigned long long q = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (q >= nq) return;
    // each part's tile is already sorted ascending: classic k-way merge with one cursor per part
    uint32_t cur[64];
    for (uint32_t p = 0; p < num_parts; ++p) cur[p] = 0;
    for (uint32_t r = 0; r < k; ++r) {
        int best = -1;
        float bd = 0.0f;
        unsigned long long bid = 0;
        for (uint32_t p = 0; p < num_parts; ++p) {
            if (cur[p] >= k) continue;
            const size_t o = ((size_t)p * nq + q) * k + cur[p];
            const uint32_t lid = part_ids[o];
            if (lid == kUnusedId) continue;
            const float d = part_dists[o];
            const unsigned long long gid = part_base[p] + lid;
            if (best < 0 || d < bd || (d == bd && gid < bid)) {
                best = (int)p;
                bd = d;
                bid = gid;
            }
        }
        if (best < 0) {
            out_ids[q * k + r] = ~0ull;
            out_dists[q * k + r] = __int_as_float(0x7f800000);
        } else {
            out_ids[q * k + r] = bid;
            out_dists[q * k + r] = bd;
            cur[best] += 1;
        }
    }
}

}  // namespace granne_b200
