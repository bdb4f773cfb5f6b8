// exact_kernels.cuh — exact k-nearest-neighbour scan (granne_b200_exact_search_batch*).
//
// Not a reference function: it applies the reference's distance (ElementContainer::dist_to_element,
// src/index/mod.rs:1012) to every element of [0, Index::len) and keeps the first k entries in the order of
// into_sorted_vec (:1036), i.e. by (distance, id) — the key make_key builds.  This is the answer the approximate search
// is measured against.
//
// A call runs in query chunks (at most kExactMaxChunk queries) and row slabs (rows whose distances fit the slab
// buffer):
//   exact_prepare_kernel    the queries as elements (prepare_query: normalise or quantise)
//   exact_scan_f32_kernel   distances of a chunk x slab into the slab buffer, CUDA-core FMAs in the reference order
//   exact_scan_i8_kernel    the same for i8 rows: exact integer dot products, then finish_angular_i8
//   exact_select_kernel     per query: keys of the slab below the running k-th key join the running top-k list (the
//                           block's key_sort, keys.cuh)
//   exact_write_kernel      the lists into the search_batch output layout (store_key)
// EMBEDDINGS rows are materialised window by window by sum_embeddings_kernel + make_elements_kernel and scanned as
// natural-layout f32 rows.
//
// The exact filtered call (granne_b200_exact_search_filtered_batch*) scans lists of ids instead of slabs of rows
// (LISTED = true): per query chunk
//   exact_chunk_filters_kernel  the distinct filters the chunk's queries name (key_sort of their ids, then
//                               block_exclusive_scan)
// then per list of at most a slab of ids
//   exact_list_ids_kernel       the next ids their union admits, ascending, from a cursor in device memory
//   exact_listed_rows_kernel    (EMBEDDINGS) the rows of those ids only
//   exact_scan_*_kernel<true>   row r of the slab is element ids[r]; the row count is read from device memory and the
//                               blocks stride over row tiles, so a short list is a small launch
//   exact_select_kernel<true>   keys make_key(d, ids[r]) of the rows the query's own filter admits; NaN flagged here
//   exact_write_kernel<true>    per-query counts (the admitted keys the list holds)
#pragma once

#include "keys.cuh"

namespace granne_b200 {

constexpr uint32_t kExactMaxK = 1024;      // GRANNE_B200_EXACT_MAX_K
constexpr uint32_t kExactMaxChunk = 1024;  // queries per chunk
constexpr int kExactQB = 64;               // queries per scan block
constexpr int kExactRB = 128;              // rows per scan block
constexpr int kExactBK = 32;               // K steps staged per round
constexpr int kExactSelThreads = 512;
constexpr int kExactSelSlots = 4096;       // select buffer: [0, kExactMaxK) the running list, the rest candidates

// the step modes of the f32 scan (see exact_scan_f32_kernel)
constexpr unsigned char kStepFirst = 1;  // first FMA of a chunk accumulator: start from +0.0
constexpr unsigned char kStepLast = 2;   // last FMA of a chunk accumulator: add it to the ordered sum
constexpr unsigned char kStepTail = 4;   // an FMA of the tail, straight into the sum

struct ExactScanArgs {
    const void* rows;          // f32 rows (lane-permuted when vec_group > 1) or i8 rows
    unsigned long long nrows;  // rows of this slab
    uint32_t row_stride;       // floats (f32) or bytes (i8) per row
    uint32_t vec_group;        // V of permuted_offset (1: natural layout)
    uint32_t dim, full, tail;
    const void* queries;  // prepared queries: f32 [nq][dim] or i8 [nq][row_stride]
    const int* qnorm;     // i8: dy of every query
    uint32_t nq;
    float* dists;         // [nq][ld]
    unsigned long long ld;
    int* error;           // kStatusNotFinite is or-ed in on a NaN distance (not LISTED)
    // LISTED only: the number of rows is row_count[0] (device memory); slab row r is element row_ids[r] of `rows`
    // (null: row r)
    const uint32_t* row_ids;
    const uint32_t* row_count;
};

// A LISTED scan's list and the filters its select applies (exact_select_kernel<true>, exact_write_kernel<true>).
struct ExactList {
    const uint32_t* ids;           // the list's admitted ids, ascending
    const uint32_t* count;         // [0] ids in the list, [1] distinct filters the chunk names, [2] the list cursor
    const uint32_t* filters;       // num_filters bitmaps of filter_words words
    const uint32_t* query_filter;  // the chunk's entries, or null (filter 0)
    unsigned long long filter_words;
    unsigned long long bit_base;   // bit of element 0
    uint32_t num_filters;
    const int* qstatus;            // per query of the chunk: its prepare step's status (a NaN i8 query)
    int* error;
};

// Bit `bit_base + id` of bitmap f (LSB first), the bit filtered search reads.
__device__ __forceinline__ bool filter_admits(const ExactList& l, uint32_t f, uint32_t id) {
    const unsigned long long b = l.bit_base + id;
    return (__ldg(l.filters + (size_t)f * l.filter_words + (b >> 5)) >> (uint32_t)(b & 31u)) & 1u;
}

// A LISTED scan's distance: finish_angular's, except that NaN stays NaN for the select to flag (only the select knows
// whether the query's filter admits the row).
__device__ __forceinline__ float listed_angular(float r) {
    int st = 0;
    const float d = finish_angular(r, &st);
    return st ? __int_as_float(0x7fc00000) : d;
}

// The queries of a chunk as elements, one warp per query: prepare_query writes each one to its row of `out` instead
// of a search warp's query slot.  f32 kinds: [nq][dim]; i8: [nq][row_stride] zero padded, and dy.  A query's status
// (a NaN i8 query) goes to qstatus[q] when qstatus is given, else it is or-ed into *error.
__global__ void __launch_bounds__(32) exact_prepare_kernel(const DeviceIndex ix, const void* __restrict__ queries,
                                                            int fmt, uint32_t nq, void* __restrict__ out,
                                                            int* __restrict__ qnorm, int* __restrict__ error,
                                                            int* __restrict__ qstatus) {
    const bool i8 = ix.kind == kAngularI8;
    SearchArgs q{};
    q.queries = queries;
    q.query_format = fmt;  // kQueryRawF32 or kQueryElement
    WarpCtx c;
    c.lane = threadIdx.x;
    for (uint32_t qi = blockIdx.x; qi < nq; qi += gridDim.x) {
        c.qs = i8 ? reinterpret_cast<float*>(static_cast<int8_t*>(out) + (size_t)qi * ix.row_stride)
                  : static_cast<float*>(out) + (size_t)qi * ix.dim;
        c.status = 0;
        prepare_query(ix, q, c, qi);
        if (c.lane == 0 && i8) qnorm[qi] = c.q_norm_i8;
        if (c.lane == 0 && qstatus)
            qstatus[qi] = c.status;
        else if (c.lane == 0 && c.status)
            atomicOr(error, c.status);
    }
}

// f32 distances of kExactQB queries x kExactRB rows per block; thread (tq, tr) owns 4 queries x 8 rows.
//
// dot_product_f32 (src/math.rs:16-42) is chunk[i] = FMA chain over the full chunks, r = 0 + chunk[0] + ... + chunk[31]
// in lane order, then the FMA tail.  chunk[i] is complete before r uses it, so computing the chunks one after the other
// gives the same bits with one accumulator: the K loop walks the steps s = i * full + ch (element ch * 32 + i), starts
// an accumulator at +0.0 on ch == 0 (kStepFirst), adds it to r after ch == full - 1 (kStepLast), and then walks the
// tail (kStepTail) straight into r.  Every pair therefore costs dim FMAs and 32 adds, like the reference, and the
// operands are staged in shared memory like an SGEMM tile.  No tensor cores: TF32 and 3xTF32 do not round like this.
//
// LISTED: rows are taken from a list (ExactScanArgs::row_ids / row_count) and the blocks stride over its row tiles; each
// tile stages its element ids in shared memory first.  The lane-permuted layout is per element, so a gathered row is
// read exactly like a row of a slab.
template <bool LISTED>
__device__ __forceinline__ void exact_scan_f32_tile(const ExactScanArgs& a, unsigned long long r0,
                                                    unsigned long long nrows, const uint32_t* rid) {
    __shared__ __align__(16) float Qs[kExactBK][kExactQB + 4];
    __shared__ __align__(16) float Xs[kExactBK][kExactRB + 4];
    __shared__ unsigned char mode[kExactBK];
    const int tid = threadIdx.x, tq = tid & 15, tr = tid >> 4;
    const uint32_t q0 = blockIdx.y * kExactQB;
    const uint32_t full = a.full, nfull = full * 32u, steps = nfull + a.tail, V = a.vec_group;
    const float* rows = static_cast<const float*>(a.rows);
    const float* qsrc = static_cast<const float*>(a.queries);
    float acc[4][8], r[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = r[i][j] = 0.0f;

    for (uint32_t s0 = 0; s0 < steps; s0 += kExactBK) {
        // stage the K steps [s0, s0 + 32): warp w loads rows w, w + 8, ... and queries w, w + 8, ...; lane = step
        const uint32_t kk = tid & 31, s = s0 + kk;
        const bool ok = s < steps;
        uint32_t e = s, o = s;
        unsigned char m = 0;
        if (ok && s < nfull) {
            const uint32_t i = s / full, ch = s - i * full;
            e = ch * 32u + i;
            o = V > 1 ? permuted_offset(e, V) : e;
            m = (ch == 0 ? kStepFirst : 0) | (ch == full - 1 ? kStepLast : 0);
        } else if (ok) {
            m = kStepTail;
        }
        if (tid < kExactBK) mode[tid] = m;
#pragma unroll 4
        for (int j = 0; j < kExactRB / 8; ++j) {
            const int row = (tid >> 5) + 8 * j;
            const unsigned long long gr = r0 + row;
            const unsigned long long e_row = LISTED ? rid[row] : gr;
            Xs[kk][row] = (ok && gr < nrows) ? __ldg(rows + e_row * a.row_stride + o) : 0.0f;
        }
#pragma unroll
        for (int j = 0; j < kExactQB / 8; ++j) {
            const int q = (tid >> 5) + 8 * j;
            const uint32_t gq = q0 + q;
            Qs[kk][q] = (ok && gq < a.nq) ? __ldg(qsrc + (size_t)gq * a.dim + e) : 0.0f;
        }
        __syncthreads();
        const int nk = steps - s0 < (uint32_t)kExactBK ? (int)(steps - s0) : kExactBK;
        for (int k2 = 0; k2 < nk; ++k2) {
            const float4 qa = *reinterpret_cast<const float4*>(&Qs[k2][tq * 4]);
            const float4 xa = *reinterpret_cast<const float4*>(&Xs[k2][tr * 8]);
            const float4 xb = *reinterpret_cast<const float4*>(&Xs[k2][tr * 8 + 4]);
            const float qv[4] = {qa.x, qa.y, qa.z, qa.w};
            const float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
            const unsigned char md = mode[k2];
            if (md & kStepTail) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) r[i][j] = __fmaf_rn(xv[j], qv[i], r[i][j]);
            } else {
                if (md & kStepFirst) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[i][j] = __fmaf_rn(xv[j], qv[i], 0.0f);
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[i][j] = __fmaf_rn(xv[j], qv[i], acc[i][j]);
                }
                if (md & kStepLast) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) r[i][j] = __fadd_rn(r[i][j], acc[i][j]);
                }
            }
        }
        __syncthreads();
    }
    int status = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t q = q0 + tq * 4 + i;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned long long row = r0 + tr * 8 + j;
            const float d = LISTED ? listed_angular(r[i][j]) : finish_angular(r[i][j], &status);
            if (q < a.nq && row < nrows) a.dists[(size_t)q * a.ld + row] = d;
        }
    }
    // a padding pair (zero operands) is NaN only if its row or query holds a NaN, and then a real pair is NaN too
    if (!LISTED && status) atomicOr(a.error, status);
}

// The element ids of the LISTED row tile at r0 into rid (0 past the list), then a barrier.
__device__ __forceinline__ void exact_stage_row_ids(const ExactScanArgs& a, unsigned long long r0,
                                                    unsigned long long nrows, uint32_t* rid) {
    for (int i = threadIdx.x; i < kExactRB; i += blockDim.x) {
        const unsigned long long gr = r0 + i;
        rid[i] = gr < nrows ? (a.row_ids ? a.row_ids[gr] : (uint32_t)gr) : 0u;
    }
    __syncthreads();
}

template <bool LISTED>
__global__ void __launch_bounds__(256, 2) exact_scan_f32_kernel(const ExactScanArgs a) {
    if constexpr (LISTED) {
        __shared__ uint32_t rid[kExactRB];
        const unsigned long long nrows = *a.row_count;
        // a tile's last reads of rid precede the barriers that end its K loop
        for (unsigned long long r0 = (unsigned long long)blockIdx.x * kExactRB; r0 < nrows;
             r0 += (unsigned long long)gridDim.x * kExactRB) {
            exact_stage_row_ids(a, r0, nrows, rid);
            exact_scan_f32_tile<true>(a, r0, nrows, rid);
        }
    } else {
        exact_scan_f32_tile<false>(a, (unsigned long long)blockIdx.x * kExactRB, a.nrows, nullptr);
    }
}

// i8 distances of kExactQB queries x kExactRB rows per block: r over the 32-bit words of the padded rows with dp4a
// (integer sums: any order is exact), dx of every row computed once per block by the warp that stages it, then
// finish_angular_i8, DistI8's IEEE sequence.  dx is computed per tile rather than cached per handle: it costs one dp4a per staged
// word, needs no state on the handle and stays right when a builder appends rows.
// LISTED as in exact_scan_f32_kernel: dx is computed from the gathered row as it is staged, like any other.
template <bool LISTED>
__device__ __forceinline__ void exact_scan_i8_tile(const ExactScanArgs& a, unsigned long long r0,
                                                   unsigned long long nrows, const uint32_t* rid) {
    __shared__ __align__(16) int Qs[kExactBK][kExactQB + 4];
    __shared__ __align__(16) int Xs[kExactBK][kExactRB + 4];
    __shared__ int dxs[kExactRB];
    const int tid = threadIdx.x, tq = tid & 15, tr = tid >> 4, lane = tid & 31;
    const uint32_t q0 = blockIdx.y * kExactQB;
    const uint32_t words = a.row_stride / 4u;
    const int* rows = static_cast<const int*>(a.rows);
    const int* qsrc = static_cast<const int*>(a.queries);
    int acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0;
    int dxp[kExactRB / 8];  // this lane's share of the dx of the rows its warp stages
#pragma unroll
    for (int j = 0; j < kExactRB / 8; ++j) dxp[j] = 0;

    for (uint32_t s0 = 0; s0 < words; s0 += kExactBK) {
        const uint32_t s = s0 + lane;
        const bool ok = s < words;
#pragma unroll
        for (int j = 0; j < kExactRB / 8; ++j) {
            const int row = (tid >> 5) + 8 * j;
            const unsigned long long gr = r0 + row;
            const unsigned long long e_row = LISTED ? rid[row] : gr;
            const int v = (ok && gr < nrows) ? __ldg(rows + e_row * words + s) : 0;
            Xs[lane][row] = v;
            dxp[j] = __dp4a(v, v, dxp[j]);
        }
#pragma unroll
        for (int j = 0; j < kExactQB / 8; ++j) {
            const int q = (tid >> 5) + 8 * j;
            const uint32_t gq = q0 + q;
            Qs[lane][q] = (ok && gq < a.nq) ? __ldg(qsrc + (size_t)gq * words + s) : 0;
        }
        __syncthreads();
        const int nk = words - s0 < (uint32_t)kExactBK ? (int)(words - s0) : kExactBK;
        for (int k2 = 0; k2 < nk; ++k2) {
            const int4 qa = *reinterpret_cast<const int4*>(&Qs[k2][tq * 4]);
            const int4 xa = *reinterpret_cast<const int4*>(&Xs[k2][tr * 8]);
            const int4 xb = *reinterpret_cast<const int4*>(&Xs[k2][tr * 8 + 4]);
            const int qv[4] = {qa.x, qa.y, qa.z, qa.w};
            const int xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = __dp4a(xv[j], qv[i], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < kExactRB / 8; ++j) {
        const int dx = __reduce_add_sync(kFullMask, dxp[j]);
        if (lane == 0) dxs[(tid >> 5) + 8 * j] = dx;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t q = q0 + tq * 4 + i;
        const int dy = q < a.nq ? a.qnorm[q] : 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int row = tr * 8 + j;
            if (q < a.nq && r0 + row < nrows)
                a.dists[(size_t)q * a.ld + r0 + row] = finish_angular_i8(acc[i][j], dxs[row], dy);
        }
    }
}

template <bool LISTED>
__global__ void __launch_bounds__(256, 2) exact_scan_i8_kernel(const ExactScanArgs a) {
    if constexpr (LISTED) {
        __shared__ uint32_t rid[kExactRB];
        const unsigned long long nrows = *a.row_count;
        // a tile's last reads of rid precede the barriers that end its K loop
        for (unsigned long long r0 = (unsigned long long)blockIdx.x * kExactRB; r0 < nrows;
             r0 += (unsigned long long)gridDim.x * kExactRB) {
            exact_stage_row_ids(a, r0, nrows, rid);
            exact_scan_i8_tile<true>(a, r0, nrows, rid);
        }
    } else {
        exact_scan_i8_tile<false>(a, (unsigned long long)blockIdx.x * kExactRB, a.nrows, nullptr);
    }
}

// The candidates S[kExactMaxK, kExactMaxK + *cnt) join the running list S[0, k): sort, keep the first k.
__device__ __forceinline__ void exact_flush(unsigned long long* S, int* cnt, uint32_t k) {
    for (uint32_t i = kExactMaxK + *cnt + threadIdx.x; i < (uint32_t)kExactSelSlots; i += blockDim.x) S[i] = ~0ull;
    __syncthreads();
    key_sort(BlockGroup{}, S, kExactSelSlots);
    for (uint32_t i = k + threadIdx.x; i < kExactMaxK; i += blockDim.x) S[i] = ~0ull;
    if (threadIdx.x == 0) *cnt = 0;
    __syncthreads();
}

// One block per query of the chunk: the keys make_key(d, base + r) of the slab's distances that are below the
// running k-th key (the threshold) are collected, and every so often merged into the query's running top-k list
// (lists + q * kExactMaxK, padded with ~0).  Keys are unique (ids are), so the list is exactly the first k keys seen.
//
// LISTED: row r is element l.ids[r] and the slab's rows are l.count[0] (nrows and base are not used).  A query whose
// query_filter entry is >= num_filters is skipped (exact_write_kernel<true> reports it).  When the chunk names more than
// one filter a row joins only if the query's own filter admits it.  A NaN distance of an admitted row, or any admitted
// row of a query flagged NaN by its prepare step, sets kStatusNotFinite; the row then ranks at distance 0, as in the
// unlisted scan.
template <bool LISTED>
__global__ void __launch_bounds__(kExactSelThreads) exact_select_kernel(const float* __restrict__ dists,
                                                                        unsigned long long ld, unsigned long long nrows,
                                                                        uint32_t base, uint32_t k,
                                                                        unsigned long long* __restrict__ lists,
                                                                        const ExactList l) {
    __shared__ unsigned long long S[kExactSelSlots];
    __shared__ int cnt;
    const uint32_t q = blockIdx.x;
    uint32_t f = 0;
    bool own_bits = false, nan = false, nan_query = false;
    if constexpr (LISTED) {
        f = l.query_filter ? l.query_filter[q] : 0u;
        nrows = l.count[0];
        if (f >= l.num_filters || nrows == 0) return;  // uniform over the block
        own_bits = l.count[1] > 1;
        nan_query = l.qstatus[q] & kStatusNotFinite;
    }
    unsigned long long* list = lists + (size_t)q * kExactMaxK;
    const float* row = dists + (size_t)q * ld;
    for (uint32_t i = threadIdx.x; i < kExactMaxK; i += blockDim.x) S[i] = i < k ? list[i] : ~0ull;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    unsigned long long thr = S[k - 1];
    constexpr uint32_t kPer = 4;  // rows per thread and round: a round adds at most 2048 candidates
    for (unsigned long long c0 = 0; c0 < nrows; c0 += (unsigned long long)kPer * blockDim.x) {
#pragma unroll
        for (uint32_t j = 0; j < kPer; ++j) {
            const unsigned long long r = c0 + (unsigned long long)j * blockDim.x + threadIdx.x;
            if (r < nrows) {
                if constexpr (LISTED) {
                    const uint32_t id = l.ids[r];
                    if (!own_bits || filter_admits(l, f, id)) {
                        float d = row[r];
                        nan |= nan_query || d != d;
                        if (d != d) d = 0.0f;
                        const unsigned long long key = make_key(d, id);
                        if (key < thr) S[kExactMaxK + atomicAdd(&cnt, 1)] = key;
                    }
                } else {
                    const unsigned long long key = make_key(row[r], base + (uint32_t)r);
                    if (key < thr) S[kExactMaxK + atomicAdd(&cnt, 1)] = key;
                }
            }
        }
        __syncthreads();
        const int c = cnt;
        __syncthreads();  // every thread has read cnt before the next round appends
        if (c > kExactSelSlots - (int)kExactMaxK - (int)(kPer * kExactSelThreads)) {
            exact_flush(S, &cnt, k);
            thr = S[k - 1];
        }
    }
    if (cnt > 0) exact_flush(S, &cnt, k);
    for (uint32_t i = threadIdx.x; i < k; i += blockDim.x) list[i] = S[i];
    if constexpr (LISTED) {
        if (__syncthreads_or(nan) && threadIdx.x == 0) atomicOr(l.error, kStatusNotFinite);
    }
}

// Running lists -> search_batch's layout: ids (u32, 0xFFFFFFFF padded), distances (+inf padded), counts.
// LISTED: a query's count is the number of keys its list holds (min(k, |A_f(q)|); `count` is not used, and lists is
// null when nothing was scanned), and a query whose query_filter entry is >= num_filters sets kStatusBadFilter.
template <bool LISTED>
__global__ void exact_write_kernel(const unsigned long long* __restrict__ lists, uint32_t nq, uint32_t k,
                                   uint32_t count, uint32_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                   uint32_t* __restrict__ out_counts, const ExactList l) {
    const unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (t < (unsigned long long)nq * k) {
        const uint32_t q = (uint32_t)(t / k), r = (uint32_t)(t % k);
        const bool used = LISTED ? lists && lists[(size_t)q * kExactMaxK + r] != ~0ull : r < count;
        store_key(out_ids, out_dists, t, used ? lists[(size_t)q * kExactMaxK + r] : ~0ull, used);
    }
    if constexpr (LISTED) {
        if (t < nq) {
            const uint32_t f = l.query_filter ? l.query_filter[t] : 0u;
            if (f >= l.num_filters) atomicOr(l.error, kStatusBadFilter);
            // the list holds its keys first and padding behind them: the count is found by bisection
            uint32_t lo = 0, hi = lists ? k : 0u;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (lists[(size_t)t * kExactMaxK + mid] != ~0ull)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            if (out_counts) out_counts[t] = lo;
        }
    } else {
        if (out_counts && t < nq) out_counts[t] = count;
    }
}

// ---- exact filtered search: lists of admitted ids ----------------------------------------------------------------------
constexpr int kExactListThreads = 1024;

// The distinct valid filters the chunk's qc <= kExactMaxChunk queries name (query_filter null: filter 0), ascending,
// into flist, and their number into count[1]; the chunk's list cursor count[2] starts at word 0.  Entries >=
// num_filters are left out.  One block of kExactListThreads.
__global__ void __launch_bounds__(kExactListThreads) exact_chunk_filters_kernel(const uint32_t* __restrict__ query_filter,
                                                                                 uint32_t qc, uint32_t num_filters,
                                                                                 uint32_t* __restrict__ flist,
                                                                                 uint32_t* __restrict__ count) {
    __shared__ uint32_t s[kExactListThreads];
    const uint32_t t = threadIdx.x;
    uint32_t f = t < qc ? (query_filter ? query_filter[t] : 0u) : ~0u;
    s[t] = f < num_filters ? f : ~0u;
    __syncthreads();
    key_sort(BlockGroup{}, s, kExactListThreads);
    f = s[t];
    const bool keep = f != ~0u && (t == 0 || s[t - 1] != f);
    uint32_t total;
    const uint32_t pos = block_exclusive_scan(keep ? 1u : 0u, &total);
    if (keep) flist[pos] = f;
    if (t == 0) {
        count[1] = total;
        count[2] = 0;
    }
}

constexpr uint32_t kListWarpWords = 256;  // words of 32 ids per warp and round of exact_list_ids_kernel

// The next ids in [0, n) that some filter of flist (count[1] of them) admits, ascending, into ids, and their number into
// count[0]: from word count[2] of the ids (32 ids per word) on, whole words while they fit in `cap` ids, and count[2]
// then points at the first word not taken.  So every list but the last holds more than cap - 32 ids, and a chunk needs
// at most ceil(n / (cap - 31)) lists (cap >= 32), however dense its filters: lists that start at or past n are empty.
// Bit i of a bitmap is bit bit_base + i, which need not start a word (a range-partitioned shard's base); bits of ids
// >= n are ignored.  One block of kExactListThreads; per round, warp w owns kListWarpWords consecutive words: their
// popcounts, a prefix scan over the warps, then the warp walks its non-zero words in order and each lane stores the id
// of its bit (one coalesced store per word).  The filters are read twice, |flist| bitmap words per word of ids each time.
__global__ void __launch_bounds__(kExactListThreads) exact_list_ids_kernel(const uint32_t* __restrict__ filters,
                                                                            unsigned long long filter_words,
                                                                            unsigned long long bit_base,
                                                                            const uint32_t* __restrict__ flist,
                                                                            uint32_t* __restrict__ count,
                                                                            unsigned long long n, uint32_t cap,
                                                                            uint32_t* __restrict__ ids) {
    __shared__ unsigned long long stop;  // the first word of the round that did not fit
    __shared__ uint32_t stop_acc;        // the ids before it
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nfl = count[1];
    const unsigned long long nwords = (n + 31) / 32;
    auto word = [&](unsigned long long j) {
        if (j >= nwords) return 0u;
        const unsigned long long b = bit_base + 32ull * j, wi = b >> 5;
        const uint32_t sh = (uint32_t)(b & 31u);
        uint32_t v = 0;
        for (uint32_t i = 0; i < nfl; ++i) {
            const uint32_t* bm = filters + (size_t)flist[i] * filter_words;
            const uint32_t lo = __ldg(bm + wi);
            // bits from the next word belong to ids >= n when that word is past the bitmap
            const uint32_t hi = (sh && wi + 1 < filter_words) ? __ldg(bm + wi + 1) : 0u;
            v |= sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
        }
        const unsigned long long rem = n - 32ull * j;  // ids of [0, n) in this word
        return rem < 32u ? v & ((1u << rem) - 1u) : v;
    };
    unsigned long long w = count[2];
    uint32_t acc = 0;
    while (w < nwords) {
        const unsigned long long j0 = w + (unsigned long long)warp * kListWarpWords;
        uint32_t c = 0;
        for (uint32_t i = lane; i < kListWarpWords; i += 32) c += __popc(word(j0 + i));
        c = __reduce_add_sync(kFullMask, c);
        uint32_t total;
        // its barriers also follow every read of the last round's stop
        const uint32_t before = block_exclusive_scan(lane == 0 ? c : 0u, &total);
        uint32_t pos = acc + __shfl_sync(kFullMask, before, 0);
        if (threadIdx.x == 0) stop = ~0ull;
        __syncthreads();
        unsigned long long my_stop = ~0ull;
        for (uint32_t i0 = 0; i0 < kListWarpWords && my_stop == ~0ull; i0 += 32) {
            const uint32_t mine = word(j0 + i0 + lane);
            for (unsigned nz = __ballot_sync(kFullMask, mine != 0); nz; nz &= nz - 1) {
                const int src = __ffs(nz) - 1;
                const uint32_t v = __shfl_sync(kFullMask, mine, src);
                if (pos + (uint32_t)__popc(v) > cap) {  // the words behind this one do not fit either
                    my_stop = j0 + i0 + src;
                    break;
                }
                if ((v >> lane) & 1u)
                    ids[pos + __popc(v & lanemask_lt())] = (uint32_t)(32ull * (j0 + i0 + src)) + lane;
                pos += __popc(v);
            }
        }
        if (lane == 0 && my_stop != ~0ull) atomicMin(&stop, my_stop);
        __syncthreads();
        const unsigned long long st = stop;
        if (st != ~0ull) {
            // the warp that owns word st stopped there first, with pos = the ids before it
            if (lane == 0 && my_stop == st) stop_acc = pos;
            __syncthreads();
            acc = stop_acc;
            w = st;
            break;
        }
        acc += total;
        w = min(w + 32ull * kListWarpWords, nwords);
    }
    if (threadIdx.x == 0) {
        count[0] = acc;
        count[2] = (uint32_t)w;
    }
}

// EMBEDDINGS: row r of `out` (dim f32) is ElementContainer::get(ids[r]) for r < count[0], the normalised ordered sum
// sum_embeddings_kernel + make_elements_kernel write for the unlisted scan.  One-warp CTAs, dim floats of dynamic
// shared memory.
__global__ void __launch_bounds__(32) exact_listed_rows_kernel(const DeviceIndex ix, const uint32_t* __restrict__ ids,
                                                               const uint32_t* __restrict__ count,
                                                               float* __restrict__ out) {
    extern __shared__ __align__(16) float listed_xs[];
    WarpCtx c;
    c.lane = threadIdx.x;
    c.xs = listed_xs;
    c.status = 0;
    const uint32_t n = count[0];
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
        DistSum::materialise(ix, c, ids[i]);
        __syncwarp();
        for (uint32_t e = c.lane; e < ix.dim; e += 32) out[(size_t)i * ix.dim + e] = listed_xs[e];
        __syncwarp();  // the next id's sum overwrites the scratch
    }
}

}  // namespace granne_b200
