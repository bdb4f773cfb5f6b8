// range_kernels.cuh — exact range search (granne_b200_exact_range_count* / granne_b200_exact_range_search*).
//
// Not a reference function: every element i of [0, Index::len) with dist_to_element(q, i) <= radius, sorted by
// (distance, id), the order of into_sorted_vec (src/index/mod.rs:1036) — the key make_key builds.  The distances are the
// exact scan's (exact_kernels.cuh), unchanged: these kernels run on the slab buffer the scan kernels fill.
//   range_count_kernel   per query of a chunk: the number of a slab's distances within the radius, added to a u64 count
//   range_emit_kernel    the same entries appended, as (id, distance) pairs, to the caller's segment of the query at a
//                        per-query cursor; a cursor past the segment's end counts on but writes nothing
//   range_finish_kernel  per query: a segment whose length equals its cursor's count is sorted in place by make_key
//                        (keys.cuh's bitonic network on shared-memory tiles and, for longer segments, the same network's
//                        wider stages as global compare-exchange steps); any other segment is padded (0xFFFFFFFF / +inf)
//                        and kStatusBadSegment is raised
// The output is written in place, so a fill needs no buffer of its results whatever their number.
#pragma once

#include "exact_kernels.cuh"
#include "keys.cuh"

namespace granne_b200 {

constexpr int kStatusBadSegment = 64;  // a range fill segment whose length is not its query's count (ERR_INVALID_ARGUMENT)

constexpr int kRangeThreads = 256;         // count / emit blocks
constexpr int kRangeRowsPerThread = 8;     // rows per thread of a count / emit block
constexpr int kRangeSortThreads = 1024;    // finish blocks
constexpr uint32_t kRangeTile = 4096;      // keys sorted per shared-memory tile (32 KB)

// The per-query rules shared by the count and the fill: entry r of a slab (element base + r) is in the range of query
// q when its distance is <= radius (IEEE: a NaN radius admits nothing, +inf admits every distance), unless the query is
// flagged bad (a bad id of a device call by id: no entries) or the entry is the query's own id (skip: the ids of a
// QUERY_ID_EXCLUDING call, else null).
struct RangeArgs {
    const float* dists;        // the slab buffer: [qc][ld]
    unsigned long long ld;
    unsigned long long nrows;  // rows of this slab
    uint32_t base;             // id of row 0
    float radius;
    const uint32_t* skip;      // [qc] or null
    const int* bad;            // [qc] or null
};

__device__ __forceinline__ bool range_in(const RangeArgs& a, uint32_t q, unsigned long long r) {
    if (r >= a.nrows) return false;
    const uint32_t id = a.base + (uint32_t)r;
    return a.dists[(size_t)q * a.ld + r] <= a.radius && !(a.skip && a.skip[q] == id);
}

// grid (row blocks of kRangeThreads * kRangeRowsPerThread rows, qc): counts[q] += the entries of the slab in range.
__global__ void __launch_bounds__(kRangeThreads) range_count_kernel(const RangeArgs a,
                                                                    unsigned long long* __restrict__ counts) {
    const uint32_t q = blockIdx.y;
    if (a.bad && a.bad[q]) return;
    const unsigned long long r0 = (unsigned long long)blockIdx.x * kRangeThreads * kRangeRowsPerThread;
    int total = 0;
#pragma unroll
    for (int j = 0; j < kRangeRowsPerThread; ++j)
        total += __syncthreads_count(range_in(a, q, r0 + (unsigned long long)j * kRangeThreads + threadIdx.x));
    if (threadIdx.x == 0 && total) atomicAdd(counts + q, (unsigned long long)total);
}

// grid as range_count_kernel: each entry in range takes the next slot of its query's cursor and, when the slot is
// below offsets[q + 1] (the chunk's entries of the caller's offsets), is written there (ids may be null: the caller gave no output, every segment must be empty).
__global__ void __launch_bounds__(kRangeThreads) range_emit_kernel(const RangeArgs a,
                                                                   unsigned long long* __restrict__ cursor,
                                                                   const unsigned long long* __restrict__ offsets,
                                                                   uint32_t* __restrict__ out_ids,
                                                                   float* __restrict__ out_dists) {
    const uint32_t q = blockIdx.y;
    if (a.bad && a.bad[q]) return;
    const int lane = threadIdx.x & 31;
    const unsigned long long r0 = (unsigned long long)blockIdx.x * kRangeThreads * kRangeRowsPerThread;
    const unsigned long long stop = offsets[q + 1];
#pragma unroll
    for (int j = 0; j < kRangeRowsPerThread; ++j) {
        const unsigned long long r = r0 + (unsigned long long)j * kRangeThreads + threadIdx.x;
        const bool in = range_in(a, q, r);
        const unsigned m = __ballot_sync(kFullMask, in);
        if (m == 0) continue;
        unsigned long long slot = 0;
        if (lane == __ffs(m) - 1) slot = atomicAdd(cursor + q, (unsigned long long)__popc(m));
        slot = __shfl_sync(kFullMask, slot, __ffs(m) - 1) + __popc(m & lanemask_lt());
        if (in && slot < stop && out_ids) {
            out_ids[slot] = a.base + (uint32_t)r;
            out_dists[slot] = a.dists[(size_t)q * a.ld + r];
        }
    }
}

// The keys [t0, t0 + p) of a segment of len entries into S (~0 past len), and back.
__device__ __forceinline__ void range_load(unsigned long long* S, const uint32_t* ids, const float* dists,
                                           unsigned long long t0, uint32_t p, unsigned long long len) {
    for (uint32_t i = threadIdx.x; i < p; i += blockDim.x)
        S[i] = t0 + i < len ? make_key(dists[t0 + i], ids[t0 + i]) : ~0ull;
    __syncthreads();
}
__device__ __forceinline__ void range_store(const unsigned long long* S, uint32_t* ids, float* dists,
                                            unsigned long long t0, uint32_t p, unsigned long long len) {
    for (uint32_t i = threadIdx.x; i < p; i += blockDim.x)
        if (t0 + i < len) store_key(ids, dists, t0 + i, S[i], true);
    __syncthreads();
}

// One compare-exchange in global memory (positions i < j of the segment; j >= len is a ~0 key: nothing to do).
__device__ __forceinline__ void range_global_cmpswap(uint32_t* ids, float* dists, unsigned long long i,
                                                     unsigned long long j, unsigned long long len) {
    if (j >= len) return;
    const unsigned long long x = make_key(dists[i], ids[i]), y = make_key(dists[j], ids[j]);
    if (x > y) {
        store_key(ids, dists, i, y, true);
        store_key(ids, dists, j, x, true);
    }
}

// One block per query of a chunk: offsets (the chunk's nq + 1 entries, the caller's) give the segment
// [offsets[q], offsets[q + 1]) and cursor[q] - offsets[q] the query's count.  A segment whose length is the count is
// sorted by make_key in place; the others are padded and flagged, and a segment that ends before it starts writes
// nothing.  Keys are unique (ids are), so the order does not depend on the order of emission.
__global__ void __launch_bounds__(kRangeSortThreads) range_finish_kernel(const unsigned long long* __restrict__ offsets,
                                                                         const unsigned long long* __restrict__ cursor,
                                                                         uint32_t* out_ids, float* out_dists,
                                                                         int* error) {
    __shared__ unsigned long long S[kRangeTile];
    const uint32_t q = blockIdx.x;
    const unsigned long long start = offsets[q], stop = offsets[q + 1];
    const unsigned long long count = cursor[q] - start;
    if (stop < start || (stop > start && !out_ids) || count != stop - start) {
        if (threadIdx.x == 0) atomicOr(error, kStatusBadSegment);
        if (stop > start && out_ids)
            for (unsigned long long i = start + threadIdx.x; i < stop; i += blockDim.x)
                store_key(out_ids, out_dists, i, ~0ull, false);
        return;
    }
    const unsigned long long len = count;
    if (len < 2) return;
    uint32_t* ids = out_ids + start;
    float* dists = out_dists + start;
    unsigned long long p = 2;
    while (p < len) p <<= 1;
    if (p <= kRangeTile) {
        range_load(S, ids, dists, 0, (uint32_t)p, len);
        key_sort(BlockGroup{}, S, (uint32_t)p);
        range_store(S, ids, dists, 0, (uint32_t)p, len);
        return;
    }
    for (unsigned long long t0 = 0; t0 < len; t0 += kRangeTile) {
        range_load(S, ids, dists, t0, kRangeTile, len);
        key_sort(BlockGroup{}, S, kRangeTile);
        range_store(S, ids, dists, t0, kRangeTile, len);
    }
    for (unsigned long long k2 = 2ull * kRangeTile; k2 <= p; k2 <<= 1) {
        for (unsigned long long t = threadIdx.x; t < p / 2; t += blockDim.x) {
            const unsigned long long i = 2 * t - (t & (k2 / 2 - 1));
            range_global_cmpswap(ids, dists, i, i ^ (k2 - 1), len);
        }
        __syncthreads();
        for (unsigned long long j = k2 / 4; j >= kRangeTile; j >>= 1) {
            for (unsigned long long t = threadIdx.x; t < p / 2; t += blockDim.x) {
                const unsigned long long i = 2 * t - (t & (j - 1));
                range_global_cmpswap(ids, dists, i, i + j, len);
            }
            __syncthreads();
        }
        for (unsigned long long t0 = 0; t0 < len; t0 += kRangeTile) {
            range_load(S, ids, dists, t0, kRangeTile, len);
            key_clean(BlockGroup{}, S, kRangeTile, kRangeTile / 2);
            range_store(S, ids, dists, t0, kRangeTile, len);
        }
    }
}

}  // namespace granne_b200
