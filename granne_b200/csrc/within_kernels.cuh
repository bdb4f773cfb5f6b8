// within_kernels.cuh — exact search within caller-given candidate lists (granne_b200_exact_search_within_batch*).
//
// Not a reference function: for query q and its list L_q it applies the reference's distance
// (ElementContainer::dist_to_element, src/index/mod.rs:1012) to every element of set(L_q) and keeps the first k by
// (distance, id), the order of into_sorted_vec (:1036) — the key make_key builds.  The distances come from the search
// path's own engines (DistF32<FULL>, DistF32Generic, DistI8, DistSum), so they are the reference's bit for bit.
//
// The lists are CSR (offsets: nq + 1 u64, ids: offsets[nq] u32).  A call runs in query chunks of at most
// kExactMaxChunk queries:
//   within_segments_kernel  per query the segments of at most kWithinSegment candidates its list splits into, their
//                           prefix over the chunk (block_exclusive_scan), and the offsets check; resets the chunk's
//                           locks, flags and counter
//   within_kernel           persistent warps over the chunk's segments: ids checked against Index::len, distances 32 at
//                           a time through Dist::dists, make_key keys sorted in shared memory (key_sort by the warp),
//                           duplicates dropped.  A query of one segment writes its output row directly (warp_store_row);
//                           the segments of a longer list merge their keys below the query's running k-th key into its
//                           running list (key_merge), under a per-query lock
//   within_write_kernel     the running lists (and the empty or rejected lists) into the search_batch output layout
// The result is the first k keys of the union of the segments' keys, and keys are unique per id, so it does not depend
// on the order segments finish in, nor on the order or multiplicity of the ids in a list.
#pragma once

#include "build_kernels.cuh"
#include "exact_kernels.cuh"
#include "keys.cuh"
#include "rerank_kernels.cuh"

namespace granne_b200 {

constexpr uint32_t kWithinSegment = 1024;  // candidates per segment: the re-rank cap, 8 KB of keys
constexpr int kStatusBadList = 8;          // an offset or an id a device call cannot serve (ERR_INVALID_ARGUMENT)

// Key slots of a warp's shared window for k neighbours: a segment's keys, or the 2P keys (P = rerank_key_slots(k)) of
// a merge with the running list.
__host__ __device__ constexpr uint32_t within_key_slots(uint32_t k) {
    return 2 * rerank_key_slots(k) > kWithinSegment ? 2 * rerank_key_slots(k) : kWithinSegment;
}

struct WithinArgs {
    const void* queries;                    // nq rows in query_format
    int query_format;
    uint32_t nq;                            // queries of this chunk
    const unsigned long long* offsets;      // this chunk's nq + 1 offsets into ids
    const uint32_t* ids;
    unsigned long long len;                 // Index::len: the ids a list may name
    uint32_t num_neighbors;                 // k <= kExactMaxK
    const unsigned long long* seg_prefix;   // nq + 1: segments of the chunk's queries before query q
    unsigned long long* lists;              // nq x k running lists (queries of more than one segment), ~0 padded
    int* locks;                             // nq
    int* qflags;                            // nq: status bits of queries of more than one segment
    unsigned long long* work_counter;
    uint32_t* out_ids;                      // nq x k, padded with kUnusedId
    float* out_dists;                       // nq x k, padded with +inf
    uint32_t* out_counts;                   // nq (or null)
    int* error_flag;                        // kStatusNotFinite / kStatusBadList are or-ed in
    WarpTiles tiles;
};

// Segments of the chunk's lists and their exclusive prefix, one block of kExactMaxChunk threads (thread = query).  A
// list whose offsets go backwards (or, for the call's first query, start anywhere but 0), or that names ids through a
// null pointer, gets no segment; its query is flagged kStatusBadList and writes count 0 and padding.
__global__ void __launch_bounds__(kExactMaxChunk) within_segments_kernel(const unsigned long long* __restrict__ offsets,
                                                                        uint32_t nq, bool first_chunk,
                                                                        const uint32_t* ids,
                                                                        unsigned long long* __restrict__ seg_prefix,
                                                                        int* __restrict__ locks,
                                                                        int* __restrict__ qflags,
                                                                        unsigned long long* __restrict__ work_counter,
                                                                        int* __restrict__ error) {
    const uint32_t q = threadIdx.x;
    unsigned long long segs = 0;
    if (q < nq) {
        const unsigned long long lo = offsets[q], hi = offsets[q + 1];
        const bool bad = hi < lo || (first_chunk && q == 0 && lo != 0) || (hi > lo && !ids);
        segs = bad ? 0 : (hi - lo + kWithinSegment - 1) / kWithinSegment;
        locks[q] = 0;
        qflags[q] = bad ? kStatusBadList : 0;
        if (bad) atomicOr(error, kStatusBadList);
    }
    unsigned long long total;
    const unsigned long long before = block_exclusive_scan(segs, &total);
    if (q < nq) seg_prefix[q + 1] = before + segs;
    if (q == 0) {
        seg_prefix[0] = 0;
        *work_counter = 0;
    }
}

// Drops the keys of keys[0, n) (ascending) equal to their predecessor, in place; returns how many are left.
__device__ __forceinline__ uint32_t warp_unique_keys(unsigned long long* keys, uint32_t n, int lane) {
    uint32_t u = 0;
    unsigned long long carry = 0;
    for (uint32_t b = 0; b < n; b += 32) {
        const uint32_t i = b + lane;
        const unsigned long long x = i < n ? keys[i] : ~0ull;
        unsigned long long prev = __shfl_up_sync(kFullMask, x, 1);
        if (lane == 0) prev = b ? carry : ~x;
        const bool keep = i < n && x != prev;
        const unsigned m = __ballot_sync(kFullMask, keep);
        carry = __shfl_sync(kFullMask, x, 31);
        __syncwarp();  // every lane has read its key before any is moved down
        if (keep) keys[u + __popc(m & lanemask_lt())] = x;
        u += __popc(m);
        __syncwarp();
    }
    return u;
}

template <class Dist>
__global__ void __launch_bounds__(32, 16) within_kernel(const DeviceIndex ix, const WithinArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    c.lane = threadIdx.x;
    const unsigned char* end = place_warp_smem(c, smem_raw, ix, a.tiles);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw + rerank_keys_offset(end - smem_raw));
    SearchArgs sq{};
    sq.queries = a.queries;
    sq.query_format = a.query_format;
    const uint32_t k = a.num_neighbors, P = rerank_key_slots(k);
    const unsigned long long total = a.seg_prefix[a.nq];
    Dist dist;
    while (true) {
        unsigned long long s0 = 0;
        if (c.lane == 0) s0 = atomicAdd(a.work_counter, 1ull);
        const unsigned long long s = __shfl_sync(kFullMask, s0, 0);
        if (s >= total) break;
        // the query of segment s: the last q with seg_prefix[q] <= s
        uint32_t q0 = 0;
        if (c.lane == 0) {
            uint32_t lo = 0, hi = a.nq;
            while (hi - lo > 1) {
                const uint32_t mid = (lo + hi) / 2;
                if (a.seg_prefix[mid] <= s) lo = mid; else hi = mid;
            }
            q0 = lo;
        }
        const uint32_t q = __shfl_sync(kFullMask, q0, 0);
        const unsigned long long first = a.seg_prefix[q], nseg = a.seg_prefix[q + 1] - first;
        const unsigned long long lo = a.offsets[q] + (s - first) * kWithinSegment, hi = a.offsets[q + 1];
        const uint32_t n = (uint32_t)(hi - lo < kWithinSegment ? hi - lo : kWithinSegment);
        const uint32_t* cand = a.ids + lo;
        // every id is checked before any row is read
        bool bad = false;
        for (uint32_t b = c.lane; b < n; b += 32) bad |= cand[b] >= a.len;
        if (__any_sync(kFullMask, bad)) {
            if (c.lane == 0) {
                atomicOr(a.error_flag, kStatusBadList);
                if (nseg > 1) atomicOr(a.qflags + q, kStatusBadList);
            }
            if (nseg == 1) warp_store_row(keys, 0, k, q, a.out_ids, a.out_dists, a.out_counts, c.lane);
            continue;
        }
        if (k == 0) {  // nothing to rank: the ids are checked, no distance is computed
            if (nseg == 1 && c.lane == 0 && a.out_counts) a.out_counts[q] = 0;
            continue;
        }
        c.status = 0;
        c.q_norm_i8 = 0;
        prepare_query(ix, sq, c, q);
        dist.load_query(ix, c);
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
        const bool nan = __any_sync(kFullMask, c.status & kStatusNotFinite);
        if (nan && c.lane == 0) {
            atomicOr(a.error_flag, kStatusNotFinite);
            if (nseg > 1) atomicOr(a.qflags + q, kStatusNotFinite);
        }
        const uint32_t u = nan ? 0u : warp_unique_keys(keys, n, c.lane);
        const uint32_t m = u < k ? u : k;
        if (nseg == 1) {
            warp_store_row(keys, m, k, q, a.out_ids, a.out_dists, a.out_counts, c.lane);
            __syncwarp();  // the next segment rewrites the keys
            continue;
        }
        // keys of this segment below the running k-th key (which only falls, so a stale read admits more, never less)
        unsigned long long* list = a.lists + (size_t)q * k;
        const unsigned long long thr = __ldcg(list + k - 1);
        uint32_t mp = 0;
        for (uint32_t b = 0; b < m; b += 32)
            mp += __popc(__ballot_sync(kFullMask, b + c.lane < m && keys[b + c.lane] < thr));
        if (mp > 0) {
            // keys[0, P): this segment's mp keys ascending, then ~0; keys[P, 2P): the running list, ascending
            node_lock(a.locks, q, c.lane);
            uint32_t listed = 0;
            for (uint32_t j0 = 0; j0 < P; j0 += 32) {
                const uint32_t j = j0 + c.lane;
                const unsigned long long x = j < k ? __ldcg(list + j) : ~0ull;
                listed += __popc(__ballot_sync(kFullMask, x != ~0ull));
                if (j < P) {
                    keys[P + j] = x;
                    if (j >= mp) keys[j] = ~0ull;
                }
            }
            __syncwarp();
            key_merge(WarpGroup{c.lane}, keys, 2 * P);
            const uint32_t merged = warp_unique_keys(keys, mp + listed, c.lane);
            for (uint32_t r = c.lane; r < k; r += 32) __stcg(list + r, r < merged ? keys[r] : ~0ull);
            __threadfence();
            node_unlock(a.locks, q, c.lane);
        }
        __syncwarp();
    }
}

// The running lists of the chunk's queries of zero or more than one segment into search_batch's layout, one block per
// query: ids (u32, 0xFFFFFFFF padded), distances (+inf padded), counts.  A flagged query writes count 0 and padding.
__global__ void within_write_kernel(const unsigned long long* __restrict__ lists,
                                    const unsigned long long* __restrict__ seg_prefix, const int* __restrict__ qflags,
                                    uint32_t k, uint32_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                    uint32_t* __restrict__ out_counts) {
    const uint32_t q = blockIdx.x;
    const unsigned long long nseg = seg_prefix[q + 1] - seg_prefix[q];
    if (nseg == 1) return;  // written by within_kernel
    const bool ok = nseg > 1 && qflags[q] == 0;
    uint32_t found = 0;
    for (uint32_t r0 = 0; r0 < k; r0 += blockDim.x) {
        const uint32_t r = r0 + threadIdx.x;
        const unsigned long long key = (ok && r < k) ? lists[(size_t)q * k + r] : ~0ull;
        if (r < k) store_key(out_ids, out_dists, (size_t)q * k + r, key, key != ~0ull);
        found += __syncthreads_count(key != ~0ull);
    }
    if (threadIdx.x == 0 && out_counts) out_counts[q] = found;
}

}  // namespace granne_b200
