// ids_kernels.cuh — element ids as queries (GRANNE_B200_QUERY_ID / GRANNE_B200_QUERY_ID_EXCLUDING) and batched
// element reads (granne_b200_get_elements*).
//
// A call by id is the same call on the elements themselves (Granne::get_element, src/index/mod.rs:153-155, then
// Granne::search, :140-150): get_elements_kernel writes each id's element row exactly as get_element_kernel does, the
// unchanged ELEMENT-format kernels run on those rows, and id_results_kernel writes the caller's columns.  The search,
// exact and within kernels therefore need no by-id branch of their own, and their code is the same for every format.
//   get_elements_kernel  ElementContainer::get(ids[i]) for a batch, one warp per id; an id past the container reads
//                        nothing and flags its query
//   id_results_kernel    the caller's k columns of a call run with src_k columns: for QUERY_ID_EXCLUDING (src_k = k + 1)
//                        the query's own id removed and the rest shifted down; a flagged query blanked
#pragma once

#include "search_kernels.cuh"

namespace granne_b200 {

constexpr int kStatusBadId = 32;  // a query or element id >= num_elements (ERR_OUT_OF_RANGE)

// Row i of `out` (dim i8 for ANGULAR_INT, else dim f32) is ElementContainer::get(ids[i]), the bytes get_element_kernel
// writes: the unpermuted stored row, or the normalised ordered sum of an EMBEDDINGS element (dynamic shared memory:
// dim floats for EMBEDDINGS, none otherwise).  One-warp CTAs, persistent over the ids.  An id >= limit reads no
// memory: its row is zeros, bad[i] = 1 (bad may be null) and kStatusBadId is or-ed into *error.
__global__ void __launch_bounds__(32) get_elements_kernel(const DeviceIndex ix, const uint32_t* __restrict__ ids,
                                                          unsigned long long n, unsigned long long limit, void* out,
                                                          int* bad, int* error) {
    extern __shared__ __align__(16) float elem_xs[];
    const int lane = threadIdx.x;
    const uint32_t dim = ix.dim;
    WarpCtx c;
    c.lane = lane;
    c.xs = elem_xs;
    c.status = 0;
    for (unsigned long long i = blockIdx.x; i < n; i += gridDim.x) {
        const uint32_t id = ids[i];
        const bool ok = id < limit;
        if (lane == 0) {
            if (bad) bad[i] = ok ? 0 : 1;
            if (!ok) atomicOr(error, kStatusBadId);
        }
        if (ix.kind == kAngularI8) {
            int8_t* o = static_cast<int8_t*>(out) + i * dim;
            const int8_t* row = static_cast<const int8_t*>(ix.vectors) + (size_t)(ok ? id : 0) * ix.row_stride;
            for (uint32_t e = lane; e < dim; e += 32) o[e] = ok ? row[e] : (int8_t)0;
        } else if (ix.kind == kAngularF32) {
            float* o = static_cast<float*>(out) + i * dim;
            const float* row = static_cast<const float*>(ix.vectors) + (size_t)(ok ? id : 0) * ix.row_stride;
            for (uint32_t e = lane; e < dim; e += 32)
                o[e] = ok ? row[e < ix.full * 32 ? permuted_offset(e, ix.vec_group) : e] : 0.0f;
        } else {
            float* o = static_cast<float*>(out) + i * dim;
            if (ok) {
                DistSum::materialise(ix, c, id);
                __syncwarp();
                for (uint32_t e = lane; e < dim; e += 32) o[e] = elem_xs[e];
                __syncwarp();  // the next id's sum overwrites the scratch
            } else {
                for (uint32_t e = lane; e < dim; e += 32) o[e] = 0.0f;
            }
        }
    }
}

// The caller's results of nq queries by id from a call's result block of src_k columns, one warp per query.
// exclude: the block is the call with k + 1 columns; the entry whose id is qids[q] is removed, the rest shift down, and
// the first k are written with count min(k, remaining).  Otherwise the block is the caller's own output and only
// flagged queries are rewritten.  A query flagged in `bad` (may be null) gets count 0, ids kUnusedId, dists
// +inf and zero stats.  src_counts may be null when !exclude.
__global__ void __launch_bounds__(128) id_results_kernel(const uint32_t* src_ids, const float* src_dists,
                                                         const uint32_t* src_counts, uint32_t src_k,
                                                         const uint32_t* __restrict__ qids, const int* bad,
                                                         bool exclude, unsigned long long nq, uint32_t k,
                                                         uint32_t* out_ids, float* out_dists, uint32_t* out_counts,
                                                         unsigned long long* out_stats) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x / 32);
    for (unsigned long long q = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) / 32; q < nq; q += warps) {
        const bool flagged = bad && bad[q];
        if (!exclude && !flagged) continue;
        const uint32_t cnt = flagged ? 0u : src_counts[q];
        const uint32_t* si = src_ids + q * src_k;
        const float* sd = src_dists + q * src_k;
        uint32_t pos = cnt;  // position of the query's own id among the cnt results (cnt: absent)
        for (uint32_t b = 0; b < cnt; b += 32) {
            const unsigned m = __ballot_sync(kFullMask, b + lane < cnt && si[b + lane] == qids[q]);
            if (m) {
                pos = b + __ffs(m) - 1;
                break;
            }
        }
        const uint32_t left = cnt - (pos < cnt ? 1u : 0u);
        const uint32_t found = left < k ? left : k;
        // entries are read only when exclude, whose block is the workspace's, never the caller's output
        for (uint32_t r = lane; r < k; r += 32) {
            const uint32_t s = r + (r >= pos ? 1u : 0u);
            out_ids[q * k + r] = r < found ? si[s] : kUnusedId;
            out_dists[q * k + r] = r < found ? sd[s] : __int_as_float(0x7f800000);
        }
        if (lane == 0) {
            if (out_counts) out_counts[q] = found;
            if (flagged && out_stats)
                for (int j = 0; j < 4; ++j) out_stats[q * 4 + j] = 0;
        }
    }
}

}  // namespace granne_b200
