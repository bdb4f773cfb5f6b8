// diverse_kernels.cuh — GranneBuilder::select_neighbors (src/index/mod.rs:849-883) over a list of candidates per query
// (granne_b200_search_diverse_batch*, granne_b200_select_neighbors_batch*).
//
// The reference walks the candidates in (distance, id) order and keeps candidate j only if d(q, j) <=
// dist_to_element(s, get(j)) for every s it has already kept, stopping at max_neighbors; a list no longer than
// max_neighbors comes back untouched (:856-858).  Here the same set is found by elimination: the first candidate still
// alive is kept, it is loaded as the query (set_query_from_element) and every later alive candidate c with
// !(d(q, c) <= d(s, c)) dies.  Every kept s precedes every candidate it judges, so a candidate survives to be kept
// exactly when the reference keeps it.  The pair distance is dist_to_element(c, get(s)) where the reference computes
// dist_to_element(s, get(c)); the engines give both the same bits: the f32 dot products' FMA operands commute in the
// same lane order, the i8 r is exact and sqrt(dx) * sqrt(dy) commutes, and SumEmbeddings compares materialised
// normalised rows on both sides.
//
// One warp per list, persistent over a work counter.  The alive candidates are kept compacted as (id, distance) pairs
// in shared memory behind the engine's SmemLayout; each round computes their distances to the kept one 32 at a time
// through Dist::dists and compacts the survivors in place.  A round costs one element load and ceil(alive / 32) distance
// batches, so a list costs at most k * C pair distances.
#pragma once

#include "search_kernels.cuh"

namespace granne_b200 {

// A standalone list longer than its stride, not ascending by distance (a NaN distance included), or holding an id
// >= Index::len (ERR_INVALID_ARGUMENT)
constexpr int kStatusBadCandidates = 128;

// Where a warp's alive list starts in its shared window: the first 16-byte boundary behind the engine's SmemLayout,
// which ends `layout_end` bytes in; it takes 8 bytes per candidate (4 KB ids | 4 KB distances at the cap of 1024).
__host__ __device__ constexpr size_t diverse_list_offset(size_t layout_end) { return (layout_end + 15) & ~(size_t)15; }
__host__ __device__ constexpr size_t diverse_list_bytes(uint32_t stride) { return (size_t)stride * 8; }

struct DiverseArgs {
    const uint32_t* cand_ids;     // nq x cand_stride ids, each list ascending by distance
    const float* cand_dists;      // nq x cand_stride
    const uint32_t* cand_counts;  // nq
    uint32_t cand_stride;         // C <= GRANNE_B200_DIVERSE_MAX_CANDIDATES
    unsigned long long nq;
    uint32_t num_neighbors;       // k
    int check;                    // check every list (a device call's caller lists): kStatusBadCandidates
    unsigned long long len;       // Index::len, the bound of a checked list's ids
    uint32_t* out_ids;            // nq x k, padded with kUnusedId
    float* out_dists;             // nq x k, padded with +inf
    uint32_t* out_counts;         // nq (or null)
    unsigned int* work_counter;   // zeroed before the launch
    int* error_flag;              // kStatusNotFinite on a NaN pair distance, kStatusBadCandidates
    WarpTiles tiles;
};

template <class Dist>
__global__ void __launch_bounds__(32) diverse_kernel(const DeviceIndex ix, const DiverseArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    c.lane = threadIdx.x;
    const unsigned char* end = place_warp_smem(c, smem_raw, ix, a.tiles);
    uint32_t* alive_id = reinterpret_cast<uint32_t*>(smem_raw + diverse_list_offset(end - smem_raw));
    float* alive_d = reinterpret_cast<float*>(alive_id + a.cand_stride);
    const int lane = c.lane;
    const uint32_t k = a.num_neighbors;
    const float inf = __int_as_float(0x7f800000);
    Dist dist;
    c.q_norm_i8 = 0;
    while (true) {
        unsigned int qi0 = 0;
        if (lane == 0) qi0 = atomicAdd(a.work_counter, 1u);
        const unsigned long long qi = __shfl_sync(kFullMask, qi0, 0);
        if (qi >= a.nq) break;
        c.status = 0;
        uint32_t n = a.cand_counts[qi];
        const uint32_t* ci = a.cand_ids + qi * a.cand_stride;
        const float* cd = a.cand_dists + qi * a.cand_stride;
        uint32_t* oi = a.out_ids + qi * k;
        float* od = a.out_dists + qi * k;
        if (a.check) {
            bool bad = n > a.cand_stride;
            for (uint32_t t = lane; !bad && t < n; t += 32) {
                const float d = cd[t];
                bad = ci[t] >= a.len || d != d || (t > 0 && !(cd[t - 1] <= d));
            }
            if (__any_sync(kFullMask, bad)) {
                if (lane == 0) atomicOr(a.error_flag, kStatusBadCandidates);
                n = 0;
            }
        }
        uint32_t found = 0;
        if (n <= k) {
            // select_neighbors returns a list no longer than max_neighbors untouched (:856-858)
            for (uint32_t t = lane; t < n; t += 32) {
                oi[t] = ci[t];
                od[t] = cd[t];
            }
            found = n;
        } else if (k > 0) {
            for (uint32_t t = lane; t < n; t += 32) {
                alive_id[t] = ci[t];
                alive_d[t] = cd[t];
            }
            __syncwarp();
            uint32_t m = n;  // alive candidates, compacted at the front in candidate order
            while (true) {
                const uint32_t s = alive_id[0];
                if (lane == 0) {
                    oi[found] = s;
                    od[found] = alive_d[0];
                }
                ++found;
                if (found == k || m == 1) break;
                set_query_from_element(ix, c, dist, s);
                uint32_t kept = 0;
                for (uint32_t b = 1; b < m; b += 32) {
                    const int nb = (m - b) < 32u ? (int)(m - b) : 32;
                    const uint32_t my_id = lane < nb ? alive_id[b + lane] : 0u;
                    const float my_d = lane < nb ? alive_d[b + lane] : 0.0f;
                    const float ds = dist.dists(ix, c, my_id, nb);
                    // candidate j stays only if d(q, j) <= d(s, j) for the kept s (:875-878)
                    const bool keep = lane < nb && my_d <= ds;
                    const unsigned km = __ballot_sync(kFullMask, keep);
                    if (keep) {  // in place: every slot written lies below the ones this batch read
                        const uint32_t p = kept + __popc(km & lanemask_lt());
                        alive_id[p] = my_id;
                        alive_d[p] = my_d;
                    }
                    kept += __popc(km);
                    __syncwarp();
                }
                if (kept == 0) break;
                m = kept;
            }
        }
        if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
            found = 0;
            if (lane == 0) atomicOr(a.error_flag, kStatusNotFinite);
        }
        for (uint32_t t = found + lane; t < k; t += 32) {
            oi[t] = kUnusedId;
            od[t] = inf;
        }
        if (lane == 0 && a.out_counts) a.out_counts[qi] = found;
        __syncwarp();  // the next list rewrites the alive list
    }
}

}  // namespace granne_b200
