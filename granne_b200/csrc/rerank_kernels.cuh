// rerank_kernels.cuh — stage 2 of the two-stage search (granne_b200_search_rerank_batch*).
//
// Stage 1 is Granne::search over an angular_int index with k = C candidates (search_kernel, unchanged).  Stage 2, here,
// gives each candidate i its f32 angular distance to the query over the attached container F,
// F.dist_to_element(i, &angular::Vector::from(q)), and keeps the first k by (distance, id), the order of
// into_sorted_vec (src/index/mod.rs:1036).  The distances come from the search path's own engines run over a
// DeviceIndex view of F, so they are the reference's bit for bit:
//   - angular f32 rows: DistF32<FULL> / DistF32Generic (angular.rs:63-74, math.rs:16-42);
//   - a SumEmbeddings container: DistSum, which materialises each candidate (ordered term sum, normalize_f32) in the
//     staging tile, stg_rows at a time, before the f32 angular distance (embeddings/mod.rs:124-143,164-174).
// The result depends only on the set of candidates, not on the order stage 1 wrote them in.
//
// One warp per query, persistent over a work counter: normalise the query (prepare_query), distances of the candidates
// 32 at a time through Dist::dists, their make_key(d, id) keys into shared memory padded with ~0 to a power of two,
// key_sort by the warp, the first k keys out through warp_store_row (keys.cuh).
#pragma once

#include "keys.cuh"

namespace granne_b200 {

// 8-byte key slots a warp sorts for c candidates: the next power of two (at least 1).  At the cap of
// GRANNE_B200_RERANK_MAX_CANDIDATES = 1024 candidates, 8 KB of shared memory.
__host__ __device__ constexpr uint32_t rerank_key_slots(uint32_t c) {
    uint32_t p = 1;
    while (p < c) p <<= 1;
    return p;
}

// Where a warp's keys start in its shared window: the first 16-byte boundary behind the engine's SmemLayout, which
// ends `layout_end` bytes in.
__host__ __device__ constexpr size_t rerank_keys_offset(size_t layout_end) { return (layout_end + 15) & ~(size_t)15; }

struct RerankArgs {
    const float* queries;        // nq x dim raw f32
    unsigned long long nq;
    const uint32_t* cand_ids;    // stage 1: nq x cand_stride ids
    const uint32_t* cand_counts;  // stage 1: nq counts
    uint32_t cand_stride;        // C
    uint32_t num_neighbors;      // k <= C
    uint32_t* out_ids;           // nq x k, padded with kUnusedId
    float* out_dists;            // nq x k, padded with +inf
    uint32_t* out_counts;        // nq (or null)
    unsigned int* work_counter;  // zeroed before the launch
    int* error_flag;             // kStatusNotFinite is or-ed in on a NaN distance
    WarpTiles tiles;
};

template <class Dist>
__global__ void __launch_bounds__(32) rerank_kernel(const DeviceIndex ix, const RerankArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    c.lane = threadIdx.x;
    const unsigned char* end = place_warp_smem(c, smem_raw, ix, a.tiles);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw + rerank_keys_offset(end - smem_raw));
    SearchArgs q{};
    q.queries = a.queries;
    q.query_format = kQueryRawF32;
    const uint32_t k = a.num_neighbors;
    Dist dist;
    while (true) {
        unsigned int qi0 = 0;
        if (c.lane == 0) qi0 = atomicAdd(a.work_counter, 1u);
        const unsigned long long qi = __shfl_sync(kFullMask, qi0, 0);
        if (qi >= a.nq) break;
        c.status = 0;
        c.q_norm_i8 = 0;
        prepare_query(ix, q, c, qi);  // Vector::from(Vec<f32>): normalize_f32
        dist.load_query(ix, c);
        const uint32_t n = a.cand_counts[qi];
        const uint32_t* cand = a.cand_ids + qi * a.cand_stride;
        for (uint32_t b = 0; b < n; b += 32) {
            const int nb = (n - b) < 32u ? (int)(n - b) : 32;
            const uint32_t my_id = c.lane < nb ? cand[b + c.lane] : 0u;
            const float d = dist.dists(ix, c, my_id, nb);
            if (c.lane < nb) keys[b + c.lane] = make_key(d, my_id);
        }
        const uint32_t p = rerank_key_slots(n);
        for (uint32_t i = n + c.lane; i < p; i += 32) keys[i] = ~0ull;
        __syncwarp();
        key_sort(WarpGroup{c.lane}, keys, p);
        uint32_t found = n < k ? n : k;
        if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
            found = 0;
            if (c.lane == 0) atomicOr(a.error_flag, kStatusNotFinite);
        }
        warp_store_row(keys, found, k, qi, a.out_ids, a.out_dists, a.out_counts, c.lane);
        __syncwarp();  // the next query rewrites the keys
    }
}

}  // namespace granne_b200
