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
//   exact_select_kernel     per query: keys of the slab below the running k-th key join the running top-k list
//   exact_write_kernel      the lists into the search_batch output layout
// EMBEDDINGS rows are materialised window by window by sum_embeddings_kernel + make_elements_kernel and scanned as
// natural-layout f32 rows.
#pragma once

#include "search_kernels.cuh"

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
    int* error;           // kStatusNotFinite is or-ed in on a NaN distance
};

// The queries of a chunk as elements, one warp per query: prepare_query writes each one to its row of `out` instead
// of a search warp's query slot.  f32 kinds: [nq][dim]; i8: [nq][row_stride] zero padded, and dy.
__global__ void __launch_bounds__(32) exact_prepare_kernel(const DeviceIndex ix, const void* __restrict__ queries,
                                                            int fmt, uint32_t nq, void* __restrict__ out,
                                                            int* __restrict__ qnorm, int* __restrict__ error) {
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
        if (c.lane == 0 && i8) {
            qnorm[qi] = c.q_norm_i8;
            if (c.status) atomicOr(error, c.status);
        }
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
__global__ void __launch_bounds__(256, 2) exact_scan_f32_kernel(const ExactScanArgs a) {
    __shared__ __align__(16) float Qs[kExactBK][kExactQB + 4];
    __shared__ __align__(16) float Xs[kExactBK][kExactRB + 4];
    __shared__ unsigned char mode[kExactBK];
    const int tid = threadIdx.x, tq = tid & 15, tr = tid >> 4;
    const unsigned long long r0 = (unsigned long long)blockIdx.x * kExactRB;
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
            Xs[kk][row] = (ok && gr < a.nrows) ? __ldg(rows + gr * a.row_stride + o) : 0.0f;
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
            const float d = finish_angular(r[i][j], &status);
            if (q < a.nq && row < a.nrows) a.dists[(size_t)q * a.ld + row] = d;
        }
    }
    // a padding pair (zero operands) is NaN only if its row or query holds a NaN, and then a real pair is NaN too
    if (status) atomicOr(a.error, status);
}

// i8 distances of kExactQB queries x kExactRB rows per block: r over the 32-bit words of the padded rows with dp4a
// (integer sums: any order is exact), dx of every row computed once per block by the warp that stages it, then
// finish_angular_i8, DistI8's IEEE sequence.  dx is computed per tile rather than cached per handle: it costs one dp4a per staged
// word, needs no state on the handle and stays right when a builder appends rows.
__global__ void __launch_bounds__(256, 2) exact_scan_i8_kernel(const ExactScanArgs a) {
    __shared__ __align__(16) int Qs[kExactBK][kExactQB + 4];
    __shared__ __align__(16) int Xs[kExactBK][kExactRB + 4];
    __shared__ int dxs[kExactRB];
    const int tid = threadIdx.x, tq = tid & 15, tr = tid >> 4, lane = tid & 31;
    const unsigned long long r0 = (unsigned long long)blockIdx.x * kExactRB;
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
            const int v = (ok && gr < a.nrows) ? __ldg(rows + gr * words + s) : 0;
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
            if (q < a.nq && r0 + row < a.nrows)
                a.dists[(size_t)q * a.ld + r0 + row] = finish_angular_i8(acc[i][j], dxs[row], dy);
        }
    }
}

// Bitonic sort of the kExactSelSlots keys in S, ascending (all threads of the block).
__device__ __forceinline__ void exact_sort_slots(unsigned long long* S) {
    for (uint32_t k2 = 2; k2 <= (uint32_t)kExactSelSlots; k2 <<= 1) {
        for (uint32_t j = k2 >> 1; j > 0; j >>= 1) {
            for (uint32_t t = threadIdx.x; t < (uint32_t)kExactSelSlots / 2; t += blockDim.x) {
                const uint32_t i = 2 * t - (t & (j - 1)), ixj = i + j;
                const unsigned long long x = S[i], y = S[ixj];
                const bool up = (i & k2) == 0;
                if ((x > y) == up) {
                    S[i] = y;
                    S[ixj] = x;
                }
            }
            __syncthreads();
        }
    }
}

// The candidates S[kExactMaxK, kExactMaxK + *cnt) join the running list S[0, k): sort, keep the first k.
__device__ __forceinline__ void exact_flush(unsigned long long* S, int* cnt, uint32_t k) {
    for (uint32_t i = kExactMaxK + *cnt + threadIdx.x; i < (uint32_t)kExactSelSlots; i += blockDim.x) S[i] = ~0ull;
    __syncthreads();
    exact_sort_slots(S);
    for (uint32_t i = k + threadIdx.x; i < kExactMaxK; i += blockDim.x) S[i] = ~0ull;
    if (threadIdx.x == 0) *cnt = 0;
    __syncthreads();
}

// One block per query of the chunk: the keys make_key(d, base + r) of the slab's distances that are below the
// running k-th key (the threshold) are collected, and every so often merged into the query's running top-k list
// (lists + q * kExactMaxK, padded with ~0).  Keys are unique (ids are), so the list is exactly the first k keys seen.
__global__ void __launch_bounds__(kExactSelThreads) exact_select_kernel(const float* __restrict__ dists,
                                                                        unsigned long long ld, unsigned long long nrows,
                                                                        uint32_t base, uint32_t k,
                                                                        unsigned long long* __restrict__ lists) {
    __shared__ unsigned long long S[kExactSelSlots];
    __shared__ int cnt;
    const uint32_t q = blockIdx.x;
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
                const unsigned long long key = make_key(row[r], base + (uint32_t)r);
                if (key < thr) S[kExactMaxK + atomicAdd(&cnt, 1)] = key;
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
}

// Running lists -> search_batch's layout: ids (u32, 0xFFFFFFFF padded), distances (+inf padded), counts.
__global__ void exact_write_kernel(const unsigned long long* __restrict__ lists, uint32_t nq, uint32_t k,
                                   uint32_t count, uint32_t* __restrict__ out_ids, float* __restrict__ out_dists,
                                   uint32_t* __restrict__ out_counts) {
    const unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (t < (unsigned long long)nq * k) {
        const uint32_t q = (uint32_t)(t / k), r = (uint32_t)(t % k);
        uint32_t id = kUnusedId;
        float d = __int_as_float(0x7f800000);
        if (r < count) {
            const unsigned long long key = lists[(size_t)q * kExactMaxK + r];
            id = key_id(key);
            d = __uint_as_float(key_dbits(key));
        }
        out_ids[t] = id;
        out_dists[t] = d;
    }
    if (out_counts && t < nq) out_counts[t] = count;
}

}  // namespace granne_b200
