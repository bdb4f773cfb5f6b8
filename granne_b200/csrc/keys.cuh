// keys.cuh — what the exact family (exact, within, re-rank and range kernels) does with make_key keys: one bitonic
// network, one block prefix scan and one writer of search_batch output entries.
#pragma once

#include "search_kernels.cuh"

namespace granne_b200 {

// The threads that run a network together, and their barrier: a warp (rank = lane) or the whole block.
struct WarpGroup {
    // A lane takes key positions and exchanges those at the lower end of a pair.  A comparator per lane sorts faster on
    // its own, but measured 7 % slower on within calls over long random lists (tools/within_bench.py long_1m).
    static constexpr bool kByPosition = true;
    int lane;
    __device__ __forceinline__ uint32_t rank() const { return (uint32_t)lane; }
    __device__ __forceinline__ uint32_t size() const { return 32u; }
    __device__ __forceinline__ void sync() const { __syncwarp(); }
};
struct BlockGroup {
    static constexpr bool kByPosition = false;
    __device__ __forceinline__ uint32_t rank() const { return threadIdx.x; }
    __device__ __forceinline__ uint32_t size() const { return blockDim.x; }
    __device__ __forceinline__ void sync() const { __syncthreads(); }
};

// The ascending bitonic network on keys[0, p) (p a power of two; u64 keys or u32 ids), flip form: stage k2 is the
// steps j = k2 / 2 .. 1.  Its first step compares i with its mirror i ^ (k2 - 1) in each run of k2 keys, the others are
// half-cleaners (i against i + j).  Every comparator puts the smaller key first, so ~0 keys at the end stay there: a
// list of any length sorts as if padded with ~0 to a power of two.  The p / 2 comparators of a step are disjoint: a
// block's thread t takes comparators t, t + blockDim.x, .. (comparator t joins i = 2t - (t & (j - 1)) and i ^ m), a
// warp's lane the positions lane, lane + 32, ..  Each step ends with the group's barrier.
// The caller's writes of the keys must precede the first step by a barrier too.
template <class K>
__device__ __forceinline__ void key_cmpswap(K* keys, uint32_t i, uint32_t l) {
    const K x = keys[i], y = keys[l];
    if (x > y) {
        keys[i] = y;
        keys[l] = x;
    }
}

// Steps j, j / 2, .., 1 of stage k2 over keys[0, p).
template <class G, class K>
__device__ __forceinline__ void key_steps(const G& g, K* keys, uint32_t p, uint32_t k2, uint32_t j) {
    for (; j > 0; j >>= 1) {
        const uint32_t m = j == k2 / 2 ? k2 - 1 : j;  // i has bit j clear: i + j is i ^ j
        if constexpr (G::kByPosition) {
            for (uint32_t i = g.rank(); i < p; i += g.size())
                if ((i ^ m) > i) key_cmpswap(keys, i, i ^ m);
        } else {
            for (uint32_t t = g.rank(); t < p / 2; t += g.size()) {
                const uint32_t i = 2 * t - (t & (j - 1)), l = i ^ m;
                key_cmpswap(keys, i, l);
            }
        }
        g.sync();
    }
}

// Sorts keys[0, p) ascending: stages 2 .. p.
template <class G, class K>
__device__ __forceinline__ void key_sort(const G& g, K* keys, uint32_t p) {
    for (uint32_t k2 = 2; k2 <= p; k2 <<= 1) key_steps(g, keys, p, k2, k2 / 2);
}

// Merges the ascending halves keys[0, p / 2) and keys[p / 2, p): the last stage alone.
template <class G, class K>
__device__ __forceinline__ void key_merge(const G& g, K* keys, uint32_t p) {
    key_steps(g, keys, p, p, p / 2);
}

// The half-cleaners j, j / 2, .., 1 over keys[0, p): the steps of stage 4j after its flip step.
template <class G, class K>
__device__ __forceinline__ void key_clean(const G& g, K* keys, uint32_t p, uint32_t j) {
    key_steps(g, keys, p, 4 * j, j);
}

// Exclusive prefix sum over the block (blockDim.x a multiple of 32, at most 1024) of v; *total the sum of all.
template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
    __shared__ T warp_sums[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(kFullMask, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        T w = lane < nw ? warp_sums[lane] : T(0);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(kFullMask, w, o);
            if (lane >= o) w += y;
        }
        warp_sums[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const T before = (warp ? warp_sums[warp - 1] : T(0)) + x - v;
    *total = warp_sums[nw - 1];
    __syncthreads();  // warp_sums may be reused by the caller's next scan
    return before;
}

// The distance of an output entry that holds no element (its id is kUnusedId).
__device__ __forceinline__ float unused_dist() { return __int_as_float(0x7f800000); }

// Entry r of ids / dists: the element of `key` when `used`, else padding.
__device__ __forceinline__ void store_key(uint32_t* ids, float* dists, size_t r, unsigned long long key, bool used) {
    ids[r] = used ? key_id(key) : kUnusedId;
    dists[r] = used ? __uint_as_float(key_dbits(key)) : unused_dist();
}

// Output row `row` of search_batch's layout (k entries per row; counts may be null), by one warp: the first `found`
// of the ascending keys, then padding, then the count.
__device__ __forceinline__ void warp_store_row(const unsigned long long* keys, uint32_t found, uint32_t k,
                                               unsigned long long row, uint32_t* ids, float* dists, uint32_t* counts,
                                               int lane) {
    for (uint32_t r = lane; r < k; r += 32) store_key(ids, dists, row * k + r, r < found ? keys[r] : ~0ull, r < found);
    if (lane == 0 && counts) counts[row] = found;
}

}  // namespace granne_b200
