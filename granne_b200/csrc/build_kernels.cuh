// build_kernels.cuh — GPU-side GranneBuilder (SURVEY.md §8f-1): batched `index_element`
// (reference: src/index/mod.rs:645-960).  Candidate generation reuses the search kernel on the layer under
// construction (the reference calls the very same search_for_neighbors, :819-820); this file holds what follows it:
// select_neighbors (:849-883), initialize_node (:886-895), connect_nodes (:899-921), add_and_limit_neighbors
// (:923-959) and the final pruning pass (:794-797), plus element construction (angular.rs:55-61,
// angular_int.rs:28-45).
//
// Parallel semantics: the reference inserts with rayon's par_iter over per-node RwLocks (:755-783), i.e. a batch of
// in-flight insertions that do not see each other's links until they are written.  Here a batch is explicit: all
// elements of a batch search the same snapshot of the layer, then one warp per element links it in under per-node
// spin locks (a warp holds at most one lock at a time).  Like the reference's default build, the resulting graph
// depends on the interleaving; every individual step uses the reference's exact arithmetic.
#pragma once

#include "search_kernels.cuh"

namespace granne_b200 {

struct BuildArgs {
    const uint32_t* ids;        // batch: element ids to index
    uint32_t n_batch;
    const uint32_t* cand_ids;   // [n_batch][cand_stride] search results on the layer under construction (ascending)
    const float* cand_dists;
    const uint32_t* cand_counts;
    uint32_t cand_stride;
    uint32_t* rows;             // the layer under construction, `stride` u32 per node, kUnusedId padded
    uint32_t stride;
    uint32_t node_width;        // node.len() == the builder's num_neighbors (row width of every layer, :394)
    uint32_t max_neighbors;     // config.num_neighbors of THIS layer (halved on upper layers, :665-668)
    int* locks;                 // one spin lock per node
    WarpTiles tiles;
    unsigned int* work_counter;
    uint32_t num_nodes;         // prune pass: nodes in the layer
};

constexpr float kHundredEps = 100.0f * 1.1920929e-07f;  // NotNan::new(100.0 * f32::EPSILON) (:813,829)

__device__ __forceinline__ void node_lock(int* locks, uint32_t i, int lane) {
    if (lane == 0) {
        while (atomicCAS(locks + i, 0, 1) != 0) {
        }
        __threadfence();
    }
    __syncwarp();
}
__device__ __forceinline__ void node_unlock(int* locks, uint32_t i, int lane) {
    __syncwarp();
    if (lane == 0) {
        __threadfence();
        atomicExch(locks + i, 0);
    }
    __syncwarp();
}

// per-warp scratch for linking (shared memory)
struct LinkScratch {
    uint32_t* cid;   // candidate ids   (capacity >= max(cand_stride, node_width + 8, 40))
    float* cd;       // candidate dists
    uint32_t* sid;   // selected ids    (node slots = node_width rounded up to 32)
    float* sd;       // selected dists
    uint32_t* oid;   // the element's own selection (kept while neighbours are pruned)
    float* od;
    uint32_t* tid;   // add_and_limit: the node's current neighbours (+ the extra one) before sorting (node slots + 8)
    float* td;
};
__host__ __device__ constexpr uint32_t link_node_slots(uint32_t node_width) { return (node_width + 31u) & ~31u; }
// candidate scratch: the search results of one element, or a node's neighbours + 1 (whichever is larger)
__host__ __device__ constexpr uint32_t link_cand_cap(uint32_t cand_stride, uint32_t node_width) {
    return cand_stride > node_width + 8 ? (cand_stride > 40 ? cand_stride : 40)
                                        : (node_width + 8 > 40 ? node_width + 8 : 40);
}
// The link scratch behind SmemLayout::end, walked from `base` in the address type P like SmemLayout: the host sizes the
// build launches with its `end` (P = size_t), the kernels place LinkScratch with it (P = unsigned char*).
template <class P>
struct LinkLayout {
    P cid, cd, sid, sd, oid, od, tid, td, end;

    __host__ __device__ __forceinline__ LinkLayout(P base, uint32_t cand_cap, uint32_t node_width) {
        const uint32_t slots = link_node_slots(node_width);
        P sp = base;
        cid = sp;
        sp += (size_t)cand_cap * 4;
        cd = sp;
        sp += (size_t)cand_cap * 4;
        sid = sp;
        sp += slots * 4;
        sd = sp;
        sp += slots * 4;
        oid = sp;
        sp += slots * 4;
        od = sp;
        sp += slots * 4;
        tid = sp;
        sp += (slots + 8) * 4;
        td = sp;
        sp += (slots + 8) * 4;
        end = sp;
    }
};

// select_neighbors (:849-883) over candidates cid/cd[0..nc) sorted by distance; result in sid/sd, returns count.
template <class Dist>
__device__ __forceinline__ int select_neighbors(const DeviceIndex& ix, WarpCtx& c, Dist& dist, LinkScratch& s, int nc,
                                                int max_neighbors) {
    const int lane = c.lane;
    if (nc <= max_neighbors) {
        for (int t = lane; t < nc; t += 32) {
            s.sid[t] = s.cid[t];
            s.sd[t] = s.cd[t];
        }
        __syncwarp();
        return nc;
    }
    int ns = 0;
    for (int ci = 0; ci < nc && ns < max_neighbors; ++ci) {
        const uint32_t j = s.cid[ci];
        const float d = s.cd[ci];
        bool ok = true;
        if (ns > 0) {
            // add j if it is closer to idx than to every neighbour selected so far: d <= dist(n, element j)
            // (32 selected neighbours per distance batch: num_neighbors is not limited to a warp's width)
            set_query_from_element(ix, c, dist, j);
            for (int b = 0; b < ns && ok; b += 32) {
                const int nb = (ns - b) < 32 ? (ns - b) : 32;
                const uint32_t my = s.sid[b + (lane < nb ? lane : 0)];
                const float dn = dist.dists(ix, c, my, nb);
                ok = !__any_sync(kFullMask, (lane < nb) && !(d <= dn));
            }
        }
        if (ok) {
            if (lane == 0) {
                s.sid[ns] = j;
                s.sd[ns] = d;
            }
            ns += 1;
            __syncwarp();
        }
    }
    return ns;
}

// add_and_limit_neighbors (:923-959) for node i (lock held or exclusive access); extra = (ej, ed) if has_extra.
// Rows wider than a warp are handled 32 slots at a time.
template <class Dist>
__device__ __forceinline__ void add_and_limit(const DeviceIndex& ix, WarpCtx& c, Dist& dist, LinkScratch& s,
                                              uint32_t* rows, uint32_t stride, uint32_t node_width, uint32_t i,
                                              bool has_extra, uint32_t ej, float ed, int limit) {
    const int lane = c.lane;
    uint32_t* row = rows + (size_t)i * stride;
    // take_while(!= UNUSED): rows are always written compactly; distances elements.dists(node_id, &neighbors) (:938)
    int cn = 0;
    for (uint32_t base = 0; base < node_width; base += 32) {
        const uint32_t v = (base + lane < node_width) ? __ldcg(row + base + lane) : kUnusedId;
        const unsigned vm = __ballot_sync(kFullMask, v != kUnusedId);
        const int run = __popc(vm & (((vm + 1u) & ~vm) - 1u));  // length of the leading run of valid slots
        if (run > 0) {
            if (cn == 0) set_query_from_element(ix, c, dist, i);
            const float dt = dist.dists(ix, c, v, run);
            if (lane < run) {
                s.tid[cn + lane] = v;
                s.td[cn + lane] = dt;
            }
        }
        cn += run;
        if (run < 32) break;
    }
    if (has_extra && lane == 0) {
        s.tid[cn] = ej;
        s.td[cn] = ed;
    }
    const int ct = cn + (has_extra ? 1 : 0);
    __syncwarp();
    // candidates.sort_unstable_by_key(|&(_, d)| d) (:945); ties keep their position (the reference's order among
    // equal distances is unspecified)
    for (int t = lane; t < ct; t += 32) {
        const float my_d = s.td[t];
        int rank = 0;
        for (int u = 0; u < ct; ++u) {
            const float du = s.td[u];
            rank += (du < my_d || (du == my_d && u < t)) ? 1 : 0;
        }
        s.cid[rank] = s.tid[t];
        s.cd[rank] = my_d;
    }
    __syncwarp();
    const int ns = select_neighbors(ix, c, dist, s, ct, limit);
    // set new neighbors and mark the remaining positions as unused (:950-958)
    for (uint32_t t = lane; t < node_width; t += 32) __stcg(row + t, (int)t < ns ? s.sid[t] : kUnusedId);
    __syncwarp();
}

// connect_nodes (:899-921): tries to add j as a neighbour of i (lock of i held).
template <class Dist>
__device__ __forceinline__ void connect_nodes(const DeviceIndex& ix, WarpCtx& c, Dist& dist, LinkScratch& s,
                                              uint32_t* rows, uint32_t stride, uint32_t node_width, uint32_t i,
                                              uint32_t j, float d) {
    if (i == j) return;
    const int lane = c.lane;
    uint32_t* row = rows + (size_t)i * stride;
    for (uint32_t base = 0; base < node_width; base += 32) {
        const uint32_t v = (base + lane < node_width) ? __ldcg(row + base + lane) : 0u;
        const unsigned hit = __ballot_sync(kFullMask, (base + lane < node_width) && (v == kUnusedId || v == j));
        if (hit) {  // the first free slot, or j is already a neighbour
            if (lane == 0) __stcg(row + base + (__ffs(hit) - 1), j);
            __syncwarp();
            return;
        }
    }
    add_and_limit(ix, c, dist, s, rows, stride, node_width, i, true, j, d, (int)node_width);
}

// The search context (SmemLayout) followed by the link scratch (LinkLayout).
__device__ __forceinline__ void setup_ctx(const DeviceIndex& ix, WarpCtx& c, LinkScratch& s, unsigned char* smem_raw,
                                          const WarpTiles& t, uint32_t cand_cap, uint32_t node_width = 32) {
    c.lane = threadIdx.x;
    const LinkLayout<unsigned char*> L(place_warp_smem(c, smem_raw, ix, t), cand_cap, node_width);
    c.status = 0;
    c.q_norm_i8 = 0;
    c.n_dist = c.n_expand = c.n_nbr = 0;
    c.list = nullptr;
    c.visited = nullptr;
    s.cid = reinterpret_cast<uint32_t*>(L.cid);
    s.cd = reinterpret_cast<float*>(L.cd);
    s.sid = reinterpret_cast<uint32_t*>(L.sid);
    s.sd = reinterpret_cast<float*>(L.sd);
    s.oid = reinterpret_cast<uint32_t*>(L.oid);
    s.od = reinterpret_cast<float*>(L.od);
    s.tid = reinterpret_cast<uint32_t*>(L.tid);
    s.td = reinterpret_cast<float*>(L.td);
}

// index_element (:805-846) after the candidate search, one warp per element of the batch.
template <class Dist>
__global__ void __launch_bounds__(32) build_link_kernel(const DeviceIndex ix, const BuildArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    LinkScratch s;
    const uint32_t cand_cap = link_cand_cap(a.cand_stride, a.node_width);
    setup_ctx(ix, c, s, smem_raw, a.tiles, cand_cap, a.node_width);
    Dist dist;
    const int lane = c.lane;
    while (true) {
        unsigned int w0 = 0;
        if (lane == 0) w0 = atomicAdd(a.work_counter, 1u);
        const uint32_t w = __shfl_sync(kFullMask, w0, 0);
        if (w >= a.n_batch) break;
        const uint32_t idx = a.ids[w];
        // do not index elements that are zero: elements.dist(idx, idx) > 100 eps (:813)
        set_query_from_element(ix, c, dist, idx);
        const float dself = __shfl_sync(kFullMask, dist.dists(ix, c, idx, 1), 0);
        if (dself > kHundredEps) continue;
        // candidates.into_iter().filter(|&(id, _)| id != idx) (:822)
        const uint32_t cnt = a.cand_counts[w];
        int nc = 0;
        for (uint32_t base = 0; base < cnt; base += 32) {
            const uint32_t t = base + lane;
            uint32_t id = kUnusedId;
            float d = 0.0f;
            if (t < cnt) {
                id = a.cand_ids[(size_t)w * a.cand_stride + t];
                d = a.cand_dists[(size_t)w * a.cand_stride + t];
            }
            const bool keep = (t < cnt) && id != idx;
            const unsigned km = __ballot_sync(kFullMask, keep);
            if (keep) {
                const int p = nc + __popc(km & lanemask_lt());
                s.cid[p] = id;
                s.cd[p] = d;
            }
            nc += __popc(km);
        }
        __syncwarp();
        const int ns = select_neighbors(ix, c, dist, s, nc, (int)a.max_neighbors);
        // a duplicate of too many of its potential neighbours stays unconnected (:826-832)
        if ((uint32_t)ns > a.max_neighbors / 2 && s.sd[a.max_neighbors / 2] < kHundredEps) continue;
        for (int t = lane; t < ns; t += 32) {
            s.oid[t] = s.sid[t];
            s.od[t] = s.sd[t];
        }
        __syncwarp();
        // own node: initialize_node if empty, else connect_nodes for every neighbour (:834-841)
        node_lock(a.locks, idx, lane);
        {
            uint32_t* row = a.rows + (size_t)idx * a.stride;
            const uint32_t first = __ldcg(row);
            if (first == kUnusedId) {
                for (int t = lane; t < ns && (uint32_t)t < a.node_width; t += 32) __stcg(row + t, s.oid[t]);
                __syncwarp();
            } else {
                for (int t = 0; t < ns; ++t)
                    connect_nodes(ix, c, dist, s, a.rows, a.stride, a.node_width, idx, s.oid[t], s.od[t]);
            }
        }
        node_unlock(a.locks, idx, lane);
        // reverse links (:843-845)
        for (int t = 0; t < ns; ++t) {
            const uint32_t nb = s.oid[t];
            node_lock(a.locks, nb, lane);
            connect_nodes(ix, c, dist, s, a.rows, a.stride, a.node_width, nb, idx, s.od[t]);
            node_unlock(a.locks, nb, lane);
        }
    }
}

// limit number of neighbors after a pass (:794-797): add_and_limit_neighbors(node, i, &[], config.num_neighbors)
template <class Dist>
__global__ void __launch_bounds__(32) build_prune_kernel(const DeviceIndex ix, const BuildArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    LinkScratch s;
    setup_ctx(ix, c, s, smem_raw, a.tiles, link_cand_cap(0, a.node_width), a.node_width);
    Dist dist;
    while (true) {
        unsigned int w0 = 0;
        if (c.lane == 0) w0 = atomicAdd(a.work_counter, 1u);
        const uint32_t i = __shfl_sync(kFullMask, w0, 0);
        if (i >= a.num_nodes) break;
        add_and_limit(ix, c, dist, s, a.rows, a.stride, a.node_width, i, false, 0u, 0.0f, (int)a.max_neighbors);
    }
}

// Dist::dist between caller-supplied vectors (py compute_distance, py/src/lib.rs:71-89: `Vector::from(a).dist(
// &Vector::from(b))`): the b vectors are staged as the element container, a_i arrives as a raw query (normalised /
// quantised by prepare_query exactly like Vector::from) and pair i is dist_to_element(i, a_i).  One warp per pair.
struct PairArgs {
    const void* queries;  // n x dim raw f32
    uint32_t n;
    float* out;           // n distances
    int* error_flag;
    WarpTiles tiles;
};

template <class Dist>
__global__ void __launch_bounds__(32) pair_distance_kernel(const DeviceIndex ix, const PairArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    WarpCtx c;
    LinkScratch s;
    setup_ctx(ix, c, s, smem_raw, a.tiles, 8);
    Dist dist;
    SearchArgs q{};
    q.queries = a.queries;
    q.query_format = kQueryRawF32;
    for (uint32_t i = blockIdx.x; i < a.n; i += gridDim.x) {
        c.status = 0;
        c.q_norm_i8 = 0;
        prepare_query(ix, q, c, i);
        dist.load_query(ix, c);
        const float d = dist.dists(ix, c, i, 1);
        if (__any_sync(kFullMask, c.status & kStatusNotFinite)) {
            if (c.lane == 0) atomicOr(a.error_flag, kStatusNotFinite);
        }
        if (c.lane == 0) a.out[i] = d;
        __syncwarp();
    }
}

// ids[i] = start + i * step  (step = +1 ascending insert pass, -1 for the reinsertion pass: reverse order, :776-782)
__global__ void iota_kernel(uint32_t* ids, uint32_t n, uint32_t start, int step) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ids[i] = (uint32_t)((long long)start + (long long)i * step);
}

__global__ void fill_u32_kernel(uint32_t* p, unsigned long long n, uint32_t v) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x)
        p[i] = v;
}

// Element construction from caller vectors: angular::Vector::from(Vec<f32>) = normalize_f32 (angular.rs:55-61,
// math.rs:124-150) or angular_int::Vector::quantize (angular_int.rs:28-45).  One warp per row, exact arithmetic.
__global__ void __launch_bounds__(32) make_elements_kernel(const float* __restrict__ raw, unsigned long long n,
                                                           uint32_t dim, int kind, void* __restrict__ out) {
    extern __shared__ float row_s[];
    const int lane = threadIdx.x;
    for (unsigned long long r = blockIdx.x; r < n; r += gridDim.x) {
        const float* src = raw + r * dim;
        __syncwarp();
        for (uint32_t i = lane; i < dim; i += 32) row_s[i] = src[i];
        __syncwarp();
        // The same arithmetic as quantize_i8 and normalize_f32, spelled out: through those helpers a compute_embeddings
        // call spent 12 % (f32) to 16 % (i8) longer in this kernel (H100 80GB HBM3, 700 W, 2M x 100).
        if (kind == kAngularI8) {
            float mx = 0.0f;
            for (uint32_t i = lane; i < dim; i += 32) mx = fmaxf(mx, fabsf(row_s[i]));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, o));
            int8_t* dst = static_cast<int8_t*>(out) + r * dim;
            for (uint32_t i = lane; i < dim; i += 32) {
                const float vi = __fdiv_rn(__fmul_rn(row_s[i], 127.0f), mx);
                int q;
                if (vi != vi)
                    q = 0;
                else if (vi >= 127.0f)
                    q = 127;
                else if (vi <= -128.0f)
                    q = -128;
                else
                    q = (int)vi;
                dst[i] = (int8_t)q;
            }
        } else {
            const uint32_t full = dim / 32;
            float p = 0.0f;
            for (uint32_t ch = 0; ch < full; ++ch) {
                const float v = row_s[ch * 32 + lane];
                p = __fmaf_rn(v, v, p);
            }
            float acc = ordered_lane_sum_bcast(p);
            for (uint32_t t = full * 32; t < dim; ++t) {
                const float v = row_s[t];
                acc = __fmaf_rn(v, v, acc);
            }
            const float norm = __fsqrt_rn(acc);
            float* dst = static_cast<float*>(out) + r * dim;
            for (uint32_t i = lane; i < dim; i += 32) dst[i] = norm > 0.0f ? __fdiv_rn(row_s[i], norm) : row_s[i];
        }
    }
}

// compute_embeddings_and_save_to_disk (embeddings/parsing.rs:102-152), its first step: raw_i =
// SumEmbeddings::get_embedding(i) (embeddings/mod.rs:112-143) for a window of elements, written as raw f32 rows.
// make_elements_kernel then turns them into elements (the second step, `.into()`).
struct SumRowsArgs {
    const float* table;                 // embedding rows, dim f32 each (no padding)
    const unsigned long long* offsets;  // n + 1 term offsets of the window's elements
    unsigned long long term_base;       // the full term list's position of terms[0]: element r's terms are
                                        // terms[offsets[r] - term_base .. offsets[r + 1] - term_base)
    const uint32_t* terms;
    unsigned long long n;
    uint32_t dim;
    int kind;     // output kind: kAngularI8 flags a NaN row, kAngularF32 any non-finite row
    float* out;   // n x dim raw rows
    int* status;  // kStatusNotFinite is or-ed in when a row is flagged
};

// Persistent warps, one element per warp at a time.  The term loop is the one of DistSum::dists: lane t holds the id
// of term t, and four 32-float chunks of the row are accumulated per pass, so that four independent 128-byte loads
// per term are in flight.  The first term's row is copied (-0.0 stays -0.0), the others are added in term order
// (sum_into_f32); an element without terms is a row of zeros.  Four blocks of 8 warps per SM (62 registers: at the
// default bound of one block, ptxas caps the kernel at 48 and spills).
__global__ void __launch_bounds__(256, 4) sum_embeddings_kernel(const SumRowsArgs a) {
    const int lane = threadIdx.x & 31;
    const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x / 32);
    const int dim = (int)a.dim;
    bool bad = false;
    for (unsigned long long r = (unsigned long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; r < a.n;
         r += warps) {
        const unsigned long long tb = a.offsets[r] - a.term_base, te = a.offsets[r + 1] - a.term_base;
        const uint32_t m = (uint32_t)(te - tb);
        float* xb = a.out + r * dim;
        for (int i0 = 0; i0 < dim; i0 += 128) {
            const int i = i0 + lane;
            const bool in0 = i < dim, in1 = i + 32 < dim, in2 = i + 64 < dim, in3 = i + 96 < dim;
            float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
            for (uint32_t g = 0; g < m; g += 32) {
                const uint32_t gm = (m - g) < 32u ? (m - g) : 32u;
                const uint32_t my_term = ((uint32_t)lane < gm) ? __ldg(a.terms + tb + g + lane) : 0u;
                for (uint32_t t = 0; t < gm; ++t) {
                    const uint32_t term = __shfl_sync(kFullMask, my_term, t);
                    const float* row = a.table + (size_t)term * dim + i;
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
            // angular_int: quantize's NotNan::new(|x|).unwrap() panics on NaN (angular_int.rs:31); angular: a
            // non-finite sum normalises to a row holding NaN, and every distance to it panics (angular.rs:70)
            const float lim = a.kind == kAngularI8 ? __int_as_float(0x7f800000) : __int_as_float(0x7f7fffff);
            bad |= (in0 && !(fabsf(a0) <= lim)) || (in1 && !(fabsf(a1) <= lim)) || (in2 && !(fabsf(a2) <= lim)) ||
                   (in3 && !(fabsf(a3) <= lim));
            if (in0) xb[i] = a0;
            if (in1) xb[i + 32] = a1;
            if (in2) xb[i + 64] = a2;
            if (in3) xb[i + 96] = a3;
        }
    }
    if (__any_sync(kFullMask, bad) && lane == 0) atomicOr(a.status, kStatusNotFinite);
}

}  // namespace granne_b200
