// granne_b200.cu — host side of the C ABI declared in include/granne_b200.h: loads granne's files, stages the layer
// graph and the element vectors in HBM, and runs batched Granne::search on the device.
//
// Mirrors the reference's `Granne` (src/index/mod.rs:38-160) + `Index` trait (:54-104) for the three element kinds
// (src/elements/angular.rs, angular_int.rs, embeddings/mod.rs).  There is no CPU search path in this library.
#include "../../include/granne_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <limits>
#include <map>
#include <thread>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "formats.hpp"
#include "reorder.hpp"
#include "build_kernels.cuh"
#include "search_kernels.cuh"

namespace gb = granne_b200;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

#define GB_CUDA(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess) {                                                                        \
            return fail(GRANNE_B200_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));      \
        }                                                                                               \
    } while (0)

// Every entry point runs on its handle's device and leaves the caller's current device as it found it (a host
// application — e.g. one torch process per GPU — must not see its default device change under it).
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        err = cudaSetDevice(device);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define GB_DEVICE(device)          \
    DeviceGuard _device_guard(device); \
    GB_CUDA(_device_guard.err)

// Per-call scratch: device copies of queries/results, status words, stream.  Pooled per handle so that several host
// threads can search concurrently (the reference's `search` is `&self` and reentrant).
struct Workspace {
    cudaStream_t stream = nullptr;
    void* d_queries = nullptr;
    size_t queries_cap = 0;
    uint32_t* d_ids = nullptr;
    float* d_dists = nullptr;
    uint32_t* d_counts = nullptr;
    unsigned long long* d_stats = nullptr;
    size_t out_cap_q = 0, out_cap_k = 0;
    int* d_status = nullptr;  // nq ints
    size_t status_cap = 0;
    // one 64-byte block, zeroed once per call: [0..2] work counters of the three passes, [3] fast pass flagged
    // something, [4] retry pass flagged something, [5] done counter (fused gather); d_error = words [8..11]
    unsigned int* d_counters = nullptr;
    int* d_error = nullptr;              // [0]=sticky error bits of this call (inside the counters block)
    unsigned long long* d_retried = nullptr;  // cumulative: queries that needed more than the fast pass
    unsigned long long* h_retried = nullptr;  // pinned mirror (copied at the end of every call, read without a sync)
    unsigned long long seen_retried = 0, seen_total = 0, total_queries = 0;
    void* h_pinned = nullptr;            // staging for host<->device copies
    size_t pinned_cap = 0;
    // slow path
    unsigned long long* d_slow_list = nullptr;
    uint32_t* d_slow_vis = nullptr;
    size_t slow_vis_cap = 0;  // u32 entries allocated for d_slow_vis
    // fast pass: per-CTA visited tables in global memory
    uint32_t* d_vis = nullptr;
    size_t vis_cap = 0;  // u32 entries
    // retry pass: fewer CTAs, larger tables
    uint32_t* d_vis_retry = nullptr;
    size_t vis_retry_cap = 0;
};

}  // namespace

struct granne_b200_index {
    int device = 0;
    int num_sms = 0;
    size_t smem_optin = 0;
    gb::DeviceIndex dev{};
    std::vector<std::shared_ptr<void>> allocations;  // device memory (shared with builder snapshots)
    uint64_t device_bytes = 0;
    uint64_t index_len = 0;  // Index::len
    std::vector<uint32_t> layer_max_degree;
    std::atomic<uint64_t> launches{0};
    std::atomic<int> sticky_error{0};
    std::mutex pool_mu;
    std::vector<std::unique_ptr<Workspace>> pool;                     // host-pointer API: one per concurrent call
    std::map<cudaStream_t, std::unique_ptr<Workspace>> stream_ws;     // device-pointer API: one per caller stream
    // fast-pass visited tables are sized max_search x degree x vis_scale; the scale doubles (up to 8) when more than
    // 1% of the recent queries overflowed into the retry pass (heavier data distributions visit more nodes)
    std::atomic<uint32_t> vis_scale{1};
    // slow path sizing
    uint32_t slow_ctas = 4;
    uint32_t slow_list_cap = 32768;
    uint32_t slow_vis_slots = 0;
};

namespace {

using Handle = granne_b200_index;

int check_device(int device, int* num_sms, size_t* smem_optin) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(GRANNE_B200_ERR_NO_DEVICE,
                    std::string("no CUDA device available (granne_b200 has no CPU fallback): ") +
                        (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    if (device < 0 || device >= count) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "device ordinal out of range");
    cudaDeviceProp prop{};
    GB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)  // sm_90a code loads on compute capability 9.0 only
        return fail(GRANNE_B200_ERR_NO_DEVICE,
                    std::string("device ") + prop.name + " is not sm_90 (H100 class); this library is built for sm_90a only");
    *num_sms = prop.multiProcessorCount;
    *smem_optin = prop.sharedMemPerBlockOptin;
    return GRANNE_B200_OK;
}

template <class T>
int dev_alloc(Handle* h, T** out, size_t count) {
    void* p = nullptr;
    const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
    GB_CUDA(cudaMalloc(&p, bytes));
    h->allocations.emplace_back(p, [](void* q) { cudaFree(q); });
    h->device_bytes += bytes;
    *out = static_cast<T*>(p);
    return GRANNE_B200_OK;
}

// Uploads `nrows` dense rows in slabs through a temporary device buffer and re-lays them out on the device.
int stage_dense(Handle* h, const uint8_t* host_rows, uint64_t nrows, uint32_t dim, bool is_i8,
                bool device_src = false) {
    gb::DeviceIndex& d = h->dev;
    d.dim = dim;
    d.full = dim / 32;
    d.tail = dim % 32;
    d.num_vectors = nrows;
    if (is_i8) {
        d.vec_group = 1;
        d.row_stride = (dim + 31u) & ~31u;  // rows start on 32-byte sector boundaries (DistI8)
        int8_t* dst = nullptr;
        int rc = dev_alloc(h, &dst, (size_t)nrows * d.row_stride);
        if (rc) return rc;
        d.vectors = dst;
        const uint64_t slab = std::max<uint64_t>(1, (64ull << 20) / dim);
        int8_t* tmp = nullptr;
        if (!device_src) GB_CUDA(cudaMalloc(&tmp, (size_t)std::min(slab, std::max<uint64_t>(nrows, 1)) * dim));
        for (uint64_t r0 = 0; r0 < nrows; r0 += slab) {
            const uint64_t nr = std::min(slab, nrows - r0);
            const int8_t* src = reinterpret_cast<const int8_t*>(host_rows) + r0 * dim;  // device memory if device_src
            if (!device_src) {
                GB_CUDA(cudaMemcpy(tmp, src, (size_t)nr * dim, cudaMemcpyHostToDevice));
                src = tmp;
            }
            gb::pad_rows_i8_kernel<<<h->num_sms * 8, 256>>>(src, dst + r0 * d.row_stride, nr, dim, d.row_stride);
            h->launches++;
            GB_CUDA(cudaGetLastError());
        }
        GB_CUDA(cudaDeviceSynchronize());
        if (tmp) GB_CUDA(cudaFree(tmp));
    } else {
        const uint32_t full = d.full;
        const bool templated = (full <= 4 || full == 6 || full == 8) && h->dev.kind == gb::kAngularF32;
        d.vec_group = !templated || full == 0 ? 1 : (full % 4 == 0 ? 4 : (full % 2 == 0 ? 2 : 1));
        d.row_stride = (dim + 3u) & ~3u;
        float* dst = nullptr;
        int rc = dev_alloc(h, &dst, (size_t)nrows * d.row_stride);
        if (rc) return rc;
        d.vectors = dst;
        const uint64_t slab = std::max<uint64_t>(1, (64ull << 20) / (dim * 4ull));
        float* tmp = nullptr;
        if (!device_src) GB_CUDA(cudaMalloc(&tmp, (size_t)std::min(slab, std::max<uint64_t>(nrows, 1)) * dim * 4));
        const float* src = reinterpret_cast<const float*>(host_rows);  // device memory if device_src
        for (uint64_t r0 = 0; r0 < nrows; r0 += slab) {
            const uint64_t nr = std::min(slab, nrows - r0);
            const float* from = src + r0 * dim;
            if (!device_src) {
                GB_CUDA(cudaMemcpy(tmp, from, (size_t)nr * dim * 4, cudaMemcpyHostToDevice));
                from = tmp;
            }
            gb::permute_rows_f32_kernel<<<h->num_sms * 8, 256>>>(from, dst + r0 * d.row_stride, nr, dim, full,
                                                                 d.vec_group, d.row_stride);
            h->launches++;
            GB_CUDA(cudaGetLastError());
        }
        GB_CUDA(cudaDeviceSynchronize());
        if (tmp) GB_CUDA(cudaFree(tmp));
    }
    return GRANNE_B200_OK;
}

// Stages the element container (vectors / embedding table + element term lists) in HBM.
int stage_elements(Handle* h, int kind, const uint8_t* el, size_t el_len, const uint8_t* emb, size_t emb_len) {
    std::string err;
    int rc;
    gb::DeviceIndex& d = h->dev;
    d.kind = kind;
    if (kind == GRANNE_B200_EMBEDDINGS) {
        gb::DenseView ev;
        if (!gb::parse_dense(emb, emb_len, 4, &ev, &err)) return fail(GRANNE_B200_ERR_FORMAT, "embeddings: " + err);
        gb::SumElements se;
        if (!gb::parse_sum_elements(el, el_len, &se, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        for (uint32_t t : se.terms)
            if (t >= ev.num) return fail(GRANNE_B200_ERR_FORMAT, "element refers to a missing embedding id");
        if (ev.dim > 4096) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "embeddings wider than 4096 are unsupported");
        rc = stage_dense(h, ev.data, ev.num, (uint32_t)ev.dim, false);
        if (rc) return rc;
        d.num_elements = se.offsets.size() - 1;
        unsigned long long* doff = nullptr;
        uint32_t* dterms = nullptr;
        if ((rc = dev_alloc(h, &doff, se.offsets.size()))) return rc;
        if ((rc = dev_alloc(h, &dterms, se.terms.size()))) return rc;
        GB_CUDA(cudaMemcpy(doff, se.offsets.data(), se.offsets.size() * 8, cudaMemcpyHostToDevice));
        if (!se.terms.empty())
            GB_CUDA(cudaMemcpy(dterms, se.terms.data(), se.terms.size() * 4, cudaMemcpyHostToDevice));
        d.sum_offsets = doff;
        d.sum_terms = dterms;
    } else {
        gb::DenseView dv;
        const bool i8 = kind == GRANNE_B200_ANGULAR_INT;
        if (!gb::parse_dense(el, el_len, i8 ? 1 : 4, &dv, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        if (dv.dim > 16384) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "vectors wider than 16384 are unsupported");
        rc = stage_dense(h, dv.data, dv.num, (uint32_t)dv.dim, i8);
        if (rc) return rc;
        d.num_elements = dv.num;
    }
    return GRANNE_B200_OK;
}

// Stages a dense element container whose rows already live in HBM (row-major elements: normalised f32 / i8).
int stage_device_elements(Handle* h, int kind, const void* d_rows, uint64_t n, uint32_t dim) {
    if (kind != GRANNE_B200_ANGULAR && kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "device-resident elements: angular or angular_int only");
    if (!d_rows && n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
    if (dim == 0 || dim > 16384) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "vectors wider than 16384 are unsupported");
    cudaPointerAttributes at{};
    if (n && (cudaPointerGetAttributes(&at, d_rows) != cudaSuccess || at.type != cudaMemoryTypeDevice ||
              at.device != h->device)) {
        cudaGetLastError();
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is not device memory of the requested device");
    }
    h->dev.kind = kind;
    int rc = stage_dense(h, static_cast<const uint8_t*>(d_rows), n, dim, kind == GRANNE_B200_ANGULAR_INT, true);
    if (rc) return rc;
    h->dev.num_elements = n;
    return GRANNE_B200_OK;
}

int check_open_args(const void* el, int kind, const void* emb) {
    if (!el) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements buffer is null");
    if (kind != GRANNE_B200_ANGULAR && kind != GRANNE_B200_ANGULAR_INT && kind != GRANNE_B200_EMBEDDINGS)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "Invalid element type");
    if (kind == GRANNE_B200_EMBEDDINGS && !emb)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "embeddings buffer required for this element type");
    return GRANNE_B200_OK;
}

void finish_handle(Handle* h) {
    h->index_len = h->dev.num_layers ? h->dev.layer_len[h->dev.num_layers - 1] : 0;
    // slow-path visited table: large enough for every node of the bottom layer (capped)
    const uint64_t want = h->index_len + h->index_len / 7 + 1024;
    h->slow_vis_slots = (uint32_t)std::min<uint64_t>(want, 16ull << 20);
}

// `dev_rows` != nullptr: the element container is given as device-resident rows (n_dev x dim_dev) instead of a file image
int open_impl(const uint8_t* index_bytes, size_t index_len, int kind, const uint8_t* el, size_t el_len,
              const uint8_t* emb, size_t emb_len, int device, Handle** out, const void* dev_rows = nullptr,
              uint64_t n_dev = 0, uint32_t dim_dev = 0) {
    if (!out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "out handle pointer is null");
    *out = nullptr;
    if (!index_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index buffer is null");
    int rc = dev_rows ? GRANNE_B200_OK : check_open_args(el, kind, emb);
    if (rc) return rc;

    std::unique_ptr<Handle> h(new Handle());
    rc = check_device(device, &h->num_sms, &h->smem_optin);
    if (rc) return rc;
    h->device = device;
    GB_DEVICE(device);

    std::string err;
    gb::HostGraph graph;
    if (!gb::parse_index(index_bytes, index_len, &graph, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
    if (graph.layers.size() > (size_t)gb::kMaxLayers) return fail(GRANNE_B200_ERR_FORMAT, "too many layers");
    if (dev_rows)
        rc = stage_device_elements(h.get(), kind, dev_rows, n_dev, dim_dev);
    else
        rc = stage_elements(h.get(), kind, el, el_len, emb, emb_len);
    if (rc) return rc;

    gb::DeviceIndex& d = h->dev;
    d.num_layers = (int)graph.layers.size();
    for (int l = 0; l < d.num_layers; ++l) {
        const gb::HostLayer& L = graph.layers[l];
        if (L.num_nodes > d.num_elements)
            return fail(GRANNE_B200_ERR_FORMAT, "index refers to more elements than the container holds");
        uint32_t* rows = nullptr;
        if ((rc = dev_alloc(h.get(), &rows, L.rows.size()))) return rc;
        if (!L.rows.empty()) GB_CUDA(cudaMemcpy(rows, L.rows.data(), L.rows.size() * 4, cudaMemcpyHostToDevice));
        d.layer_rows[l] = rows;
        d.layer_width[l] = L.width;
        d.layer_len[l] = L.num_nodes;
        h->layer_max_degree.push_back(L.max_degree);
    }
    finish_handle(h.get());
    *out = h.release();
    return GRANNE_B200_OK;
}

int read_file(const char* path, std::vector<uint8_t>* out) {
    if (!path) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "path is null");
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) return fail(GRANNE_B200_ERR_IO, std::string("Could not open ") + path);
    const std::streamsize n = f.tellg();
    f.seekg(0);
    out->resize((size_t)n);
    if (n > 0 && !f.read(reinterpret_cast<char*>(out->data()), n))
        return fail(GRANNE_B200_ERR_IO, std::string("Could not read ") + path);
    return GRANNE_B200_OK;
}

// ---- launch configuration -----------------------------------------------------------------------------------------
struct LaunchPlan {
    uint32_t list_cap, vis_slots, vis_upper;
    uint32_t vis_retry;  // visited slots per CTA of the retry pass
    int rows;           // fast list rows R (capacity 32*R), 0 = generic list
    uint32_t stg_rows;  // candidate rows per bulk-copy batch (staged distance engines only)
    uint32_t stg_row_bytes;
    uint32_t tile_rows;  // ordered-sum tile rows: 8 staged f32, 32 generic f32, 0 for i8 / embeddings
    size_t base_smem;   // tile + mbarrier + query (+ embeddings scratch) + staging
    size_t smem;        // fast pass total
    bool staged;
};

bool is_templated_f32(const gb::DeviceIndex& d) {
    // DistF32<FULL> with FULL > 0 (see dispatch_search)
    return d.kind == gb::kAngularF32 && d.full > 0 && !(d.vec_group == 1 && d.full > 4) &&
           (d.full <= 4 || d.full == 6 || d.full == 8);
}
bool is_generic_f32_staged(const gb::DeviceIndex& d) {
    // DistF32Generic stages rows of up to 8 KB (dim < 2080); wider rows load directly
    return d.kind == gb::kAngularF32 && !is_templated_f32(d) && d.full >= 1 && d.full <= 64;
}
bool is_staged_kind(const gb::DeviceIndex& d) {
    return d.kind == gb::kAngularI8 || is_templated_f32(d) || is_generic_f32_staged(d);
}

LaunchPlan make_plan(const Handle* h, uint32_t max_search) {
    const gb::DeviceIndex& d = h->dev;
    LaunchPlan p{};
    // fast list: capacity 32*R with R odd (conflict-free lane-major access); slack >= 16 entries over max_search
    p.rows = 0;
    for (int r : {3, 7, 15, 31})
        if (max_search + 16 <= 32u * r) {
            p.rows = r;
            break;
        }
    p.list_cap = p.rows ? 32u * p.rows : std::max<uint32_t>(32, (max_search + 16 + 31) & ~31u);
    const uint32_t deg = h->layer_max_degree.empty() ? 1 : std::max<uint32_t>(8, h->layer_max_degree.back());
    uint64_t want = std::max<uint64_t>(1024, (uint64_t)max_search * std::min<uint32_t>(deg, 64));
    want = (want + 31) & ~31ull;
    // the retry pass gets 8x the base table, the fast pass base x scale (both capped at 4 MB per warp)
    const uint64_t cap_slots = 1ull << 20;
    p.vis_retry = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(want * 8, want), std::max<uint64_t>(cap_slots, want));
    want = std::min<uint64_t>(want * h->vis_scale.load(), std::max<uint64_t>(cap_slots, want));
    const uint32_t qbytes = (d.kind == gb::kAngularI8) ? d.row_stride : ((d.dim + 3u) & ~3u) * 4u;
    p.staged = is_staged_kind(d);
    p.tile_rows = d.kind == gb::kAngularI8 ? 0u : ((p.staged || d.kind == gb::kSumEmbeddings) ? 8u : 32u);
    const bool generic_staged = is_generic_f32_staged(d);
    if (is_templated_f32(d))  // the ordered-sum tile has one row per staged candidate row of a batch
        p.tile_rows = std::min<uint32_t>(8u, std::max<uint32_t>(4, ((unsigned)GB_STG_BYTES / (d.full * 128u)) & ~3u));
    size_t base = gb::tile_bytes_for_rows(p.tile_rows) + 16 + ((qbytes + 15u) & ~15u) * (d.kind == gb::kSumEmbeddings ? 2 : 1);
    p.stg_rows = 0;
    p.stg_row_bytes = 0;
    if (d.kind == gb::kSumEmbeddings) {
        // staging tile = the summed vectors of a batch of candidates (one row each)
        p.stg_row_bytes = ((d.dim + 3u) & ~3u) * 4u;
        p.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(4, (8192u / p.stg_row_bytes) & ~3u));
        base = ((base + 127) & ~size_t(127)) + (size_t)p.stg_rows * p.stg_row_bytes;
    }
    if (p.staged && d.kind == gb::kAngularI8) {
        // DistI8: the staging tile is a set of 512-byte pass slots (32 lanes x one 16-byte chunk each)
        p.stg_row_bytes = 512;
        p.stg_rows = std::max<uint32_t>(2, (unsigned)GB_STG_BYTES / 512u);
        base = ((base + 127) & ~size_t(127)) + (size_t)p.stg_rows * p.stg_row_bytes;
    } else if (generic_staged) {
        const uint32_t row_bytes = d.full * 128u;
        p.stg_row_bytes = row_bytes;
        p.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(2, (unsigned)(2 * GB_STG_BYTES) / row_bytes));
        base = ((base + 127) & ~size_t(127)) + (size_t)p.stg_rows * row_bytes;
    } else if (p.staged) {
        const uint32_t row_bytes = d.full * 128u;
        p.stg_row_bytes = row_bytes;
        p.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(4, ((unsigned)GB_STG_BYTES / row_bytes) & ~3u));
        base = ((base + 127) & ~size_t(127)) + (size_t)p.stg_rows * row_bytes;
    }
    p.base_smem = base;
    const size_t budget = h->smem_optin;
    if (p.rows) {
        // fast pass: list in shared memory, visited set in global memory
        p.vis_slots = (uint32_t)want;
        p.vis_upper = std::min<uint32_t>(1024, p.vis_slots);
        p.smem = base + gb::fast_list_bytes(p.rows);
        return p;
    }
    const size_t fixed = base + (size_t)p.list_cap * 8;
    if (fixed + 4096 > budget) {  // caller rejects: the candidate list alone does not fit
        p.vis_slots = p.vis_upper = 0;
        p.smem = 0;
        return p;
    }
    if (fixed + want * 4 > budget) want = (budget - fixed) / 4 / 32 * 32;  // huge max_search: overflow -> slow path
    p.vis_slots = (uint32_t)want;
    p.vis_upper = std::min<uint32_t>(1024, p.vis_slots);
    p.smem = fixed + (size_t)p.vis_slots * 4;
    return p;
}

// next longer fast list for the retry pass (0 = none: go straight to the slow pass)
constexpr int retry_rows(int R) { return R == 3 ? 7 : (R == 7 ? 15 : (R == 15 ? 31 : 0)); }

template <class Kern>
int set_smem_attr(Kern kern, Handle* h, std::atomic<bool>* done) {
    if (!done->load()) {
        GB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        done->store(true);
    }
    return GRANNE_B200_OK;
}

template <class Dist, int R>
int launch_kernels(Handle* h, Workspace* w, gb::SearchArgs a, const LaunchPlan& plan, cudaStream_t stream,
                   const gb::DeviceIndex& dv) {
    constexpr int RR = retry_rows(R);
    auto kern = gb::search_kernel<Dist, R>;
    auto retry = gb::search_kernel<Dist, (RR > 0 ? RR : 1)>;
    auto slow = gb::search_kernel<Dist, 0>;
    static std::atomic<bool> attr_set[64][3];  // function attributes are per device
    const int dslot = h->device & 63;
    int rc;
    if ((rc = set_smem_attr(kern, h, &attr_set[dslot][0]))) return rc;
    if (RR > 0 && (rc = set_smem_attr(retry, h, &attr_set[dslot][1]))) return rc;
    if ((rc = set_smem_attr(slow, h, &attr_set[dslot][2]))) return rc;
    // fast pass
    static std::mutex occ_mu;
    static std::map<size_t, int> occ_cache;
    int occ = 0;
    {
        std::lock_guard<std::mutex> g(occ_mu);
        auto it = occ_cache.find(plan.smem);
        if (it == occ_cache.end()) {
            GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 32, plan.smem));
            occ_cache[plan.smem] = occ;
        } else {
            occ = it->second;
        }
    }
    if (occ < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search too large for the shared-memory workspace");
    static const int occ_cap = [] {  // tuning/diagnostic knob: cap the resident one-warp CTAs per SM
        const char* e = std::getenv("GRANNE_B200_MAX_CTAS_PER_SM");
        return e ? std::max(1, std::atoi(e)) : 1 << 20;
    }();
    occ = std::min(occ, occ_cap);
    const unsigned long long slots = (unsigned long long)occ * h->num_sms;
    const unsigned grid = (unsigned)std::min<unsigned long long>(a.nq, slots);
    if (R > 0) {
        // per-CTA visited tables (global memory, L2 resident); sized for a full wave so later calls reuse it
        const size_t need = (size_t)slots * plan.vis_slots;
        if (need > w->vis_cap) {
            GB_CUDA(cudaStreamSynchronize(stream));
            cudaFree(w->d_vis);
            w->d_vis = nullptr;
            w->vis_cap = 0;
            GB_CUDA(cudaMalloc(&w->d_vis, need * sizeof(uint32_t)));
            w->vis_cap = need;
        }
        a.vis_global = w->d_vis;
    }
    const bool have_retry = R > 0 && RR > 0;
    a.pass = 0;
    a.slow_pass = 0;
    a.final_pass = 0;
    a.gate_in = nullptr;
    a.gate_out = w->d_counters + 3;
    kern<<<grid, 32, plan.smem, stream>>>(dv, a);
    h->launches++;
    GB_CUDA(cudaGetLastError());
    if (have_retry) {
        // retry pass: only the queries the fast pass flagged (exits at once if none) on a full-size grid of its own,
        // with the next longer list and 8x larger visited tables — so a batch of heavy queries (e.g. the reference's
        // uniform test distribution before the table scale has adapted) never funnels through the 4-CTA slow pass
        gb::SearchArgs r = a;
        r.pass = 1;
        r.work_counter = w->d_counters + 1;
        r.gate_in = w->d_counters + 3;
        r.gate_out = w->d_counters + 4;
        r.vis_slots = std::max(plan.vis_slots, plan.vis_retry);
        r.vis_slots_upper = plan.vis_upper;
        const unsigned rgrid = (unsigned)std::min<unsigned long long>(a.nq, (unsigned long long)h->num_sms * 4);
        const size_t need = (size_t)h->num_sms * 4 * r.vis_slots;
        if (need > w->vis_retry_cap) {
            GB_CUDA(cudaStreamSynchronize(stream));
            cudaFree(w->d_vis_retry);
            w->d_vis_retry = nullptr;
            w->vis_retry_cap = 0;
            GB_CUDA(cudaMalloc(&w->d_vis_retry, need * sizeof(uint32_t)));
            w->vis_retry_cap = need;
        }
        r.vis_global = w->d_vis_retry;
        const size_t rsmem = plan.base_smem + gb::fast_list_bytes(RR > 0 ? RR : 1);
        retry<<<rgrid, 32, rsmem, stream>>>(dv, r);
        h->launches++;
        GB_CUDA(cudaGetLastError());
    }
    // slow pass: re-runs only the queries that are still flagged (exits immediately if none)
    gb::SearchArgs s = a;
    s.pass = 2;
    s.slow_pass = 1;
    s.final_pass = 1;
    s.work_counter = w->d_counters + 2;
    s.gate_in = w->d_counters + (have_retry ? 4 : 3);
    s.gate_out = nullptr;
    slow<<<h->slow_ctas, 32, plan.base_smem, stream>>>(dv, s);
    h->launches++;
    GB_CUDA(cudaGetLastError());
    return GRANNE_B200_OK;
}

template <class Dist>
int launch_search(Handle* h, Workspace* w, const gb::SearchArgs& a, const LaunchPlan& plan, cudaStream_t stream,
                  const gb::DeviceIndex& dv) {
    switch (plan.rows) {
        case 3: return launch_kernels<Dist, 3>(h, w, a, plan, stream, dv);
        case 7: return launch_kernels<Dist, 7>(h, w, a, plan, stream, dv);
        case 15: return launch_kernels<Dist, 15>(h, w, a, plan, stream, dv);
        case 31: return launch_kernels<Dist, 31>(h, w, a, plan, stream, dv);
        default: return launch_kernels<Dist, 0>(h, w, a, plan, stream, dv);
    }
}

// `d`: the staged index the kernels see — the handle's own, or a private view of it (compute_order searches single
// layers without touching the shared handle)
int dispatch_search(Handle* h, Workspace* w, const gb::SearchArgs& a, const LaunchPlan& plan, cudaStream_t stream,
                    const gb::DeviceIndex& d) {
    switch (d.kind) {
        case gb::kAngularI8:
            return launch_search<gb::DistI8>(h, w, a, plan, stream, d);
        case gb::kSumEmbeddings:
            return launch_search<gb::DistSum>(h, w, a, plan, stream, d);
        default:
            break;
    }
    if (d.vec_group == 1 && d.full > 4) return launch_search<gb::DistF32Generic>(h, w, a, plan, stream, d);
    switch (d.full) {
        case 0: return launch_search<gb::DistF32<0>>(h, w, a, plan, stream, d);
        case 1: return launch_search<gb::DistF32<1>>(h, w, a, plan, stream, d);
        case 2: return launch_search<gb::DistF32<2>>(h, w, a, plan, stream, d);
        case 3: return launch_search<gb::DistF32<3>>(h, w, a, plan, stream, d);
        case 4: return launch_search<gb::DistF32<4>>(h, w, a, plan, stream, d);
        case 6: return launch_search<gb::DistF32<6>>(h, w, a, plan, stream, d);
        case 8: return launch_search<gb::DistF32<8>>(h, w, a, plan, stream, d);
        default: return launch_search<gb::DistF32Generic>(h, w, a, plan, stream, d);
    }
}

// ---- workspace pool -----------------------------------------------------------------------------------------------
int ws_acquire(Handle* h, Workspace** out) {
    {
        std::lock_guard<std::mutex> g(h->pool_mu);
        if (!h->pool.empty()) {
            *out = h->pool.back().release();
            h->pool.pop_back();
            return GRANNE_B200_OK;
        }
    }
    std::unique_ptr<Workspace> w(new Workspace());
    GB_CUDA(cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking));
    GB_CUDA(cudaMalloc(&w->d_counters, 64));
    w->d_error = reinterpret_cast<int*>(w->d_counters + 8);
    GB_CUDA(cudaMalloc(&w->d_retried, 8));
    GB_CUDA(cudaMemset(w->d_retried, 0, 8));
    GB_CUDA(cudaMallocHost(&w->h_retried, 8));
    *w->h_retried = 0;
    GB_CUDA(cudaMalloc(&w->d_slow_list, (size_t)h->slow_ctas * h->slow_list_cap * 8));
    w->slow_vis_cap = (size_t)h->slow_ctas * h->slow_vis_slots;
    GB_CUDA(cudaMalloc(&w->d_slow_vis, w->slow_vis_cap * 4));
    *out = w.release();
    return GRANNE_B200_OK;
}
void ws_release(Handle* h, Workspace* w) {
    std::lock_guard<std::mutex> g(h->pool_mu);
    h->pool.emplace_back(w);
}
void ws_destroy(Workspace* w) {
    if (!w) return;
    cudaFree(w->d_queries);
    cudaFree(w->d_ids);  // ids | dists | counts are one block
    cudaFree(w->d_stats);
    cudaFree(w->d_status);
    cudaFree(w->d_counters);  // d_error lives inside this block
    cudaFree(w->d_retried);
    if (w->h_retried) cudaFreeHost(w->h_retried);
    cudaFree(w->d_vis_retry);
    cudaFree(w->d_slow_list);
    cudaFree(w->d_slow_vis);
    cudaFree(w->d_vis);
    if (w->h_pinned) cudaFreeHost(w->h_pinned);
    if (w->stream) cudaStreamDestroy(w->stream);
}

int ws_reserve(Workspace* w, size_t query_bytes, size_t nq, size_t k) {
    if (query_bytes > w->queries_cap) {
        cudaFree(w->d_queries);
        w->d_queries = nullptr;
        w->queries_cap = 0;
        GB_CUDA(cudaMalloc(&w->d_queries, query_bytes));
        w->queries_cap = query_bytes;
    }
    if (nq * k > w->out_cap_q * w->out_cap_k || nq > w->out_cap_q) {
        cudaFree(w->d_ids);  // one block: ids | dists | counts, so that one copy brings a whole result back
        cudaFree(w->d_stats);
        w->d_ids = nullptr, w->d_dists = nullptr, w->d_counts = nullptr, w->d_stats = nullptr;
        w->out_cap_q = w->out_cap_k = 0;
        GB_CUDA(cudaMalloc(&w->d_ids, (2 * std::max<size_t>(nq * k, 1) + std::max<size_t>(nq, 1)) * 4));
        GB_CUDA(cudaMalloc(&w->d_stats, std::max<size_t>(nq, 1) * 4 * 8));
        w->out_cap_q = nq;
        w->out_cap_k = k;
    }
    w->d_dists = reinterpret_cast<float*>(w->d_ids + nq * k);  // packed for THIS call's nq x k
    w->d_counts = w->d_ids + 2 * nq * k;
    const size_t pinned = query_bytes + nq * k * 8 + nq * 4 + nq * 32 + 128;
    if (pinned > w->pinned_cap) {
        if (w->h_pinned) cudaFreeHost(w->h_pinned);
        w->h_pinned = nullptr;
        w->pinned_cap = 0;
        GB_CUDA(cudaMallocHost(&w->h_pinned, pinned));
        w->pinned_cap = pinned;
    }
    return GRANNE_B200_OK;
}

int ws_reserve_status(Workspace* w, size_t nq) {
    if (nq > w->status_cap) {
        cudaFree(w->d_status);
        w->d_status = nullptr;
        w->status_cap = 0;
        GB_CUDA(cudaMalloc(&w->d_status, std::max<size_t>(nq, 1) * sizeof(int)));
        w->status_cap = nq;
    }
    return GRANNE_B200_OK;
}

int validate_search(const Handle* h, const void* q, size_t nq, int fmt, uint32_t max_search, uint32_t k,
                    const void* ids, const void* dists) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    if (fmt != GRANNE_B200_QUERY_RAW_F32 && fmt != GRANNE_B200_QUERY_ELEMENT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unknown query format");
    if (max_search == 0)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT,
                    "max_search must be >= 1 (the reference panics on 0, src/index/mod.rs:1019)");
    if (nq > 0xFFFFFFF0ull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many queries in one batch");
    if (nq && (!q || (k && (!ids || !dists)))) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null buffer");
    return GRANNE_B200_OK;
}

// Enqueues one batch on `stream` with device pointers.  Needs a workspace for status words / slow path.
int enqueue_search(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, uint32_t max_search,
                   uint32_t k, uint32_t* d_ids, float* d_dists, uint32_t* d_counts, unsigned long long* d_stats,
                   cudaStream_t stream, bool reset_error, const granne_b200_peer_gather* pg = nullptr,
                   const gb::DeviceIndex* view = nullptr) {
    const LaunchPlan plan = make_plan(h, max_search);
    if (plan.smem == 0 || max_search + 64 > h->slow_list_cap)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search exceeds the supported maximum (about 27000)");
    int rc = ws_reserve_status(w, nq);
    if (rc) return rc;
    // the slow-path visited tables follow the index size (a builder's index grows after its workspace was made)
    if ((size_t)h->slow_ctas * h->slow_vis_slots > w->slow_vis_cap) {
        GB_CUDA(cudaStreamSynchronize(stream));
        cudaFree(w->d_slow_vis);
        w->d_slow_vis = nullptr;
        w->slow_vis_cap = 0;
        GB_CUDA(cudaMalloc(&w->d_slow_vis, (size_t)h->slow_ctas * h->slow_vis_slots * 4));
        w->slow_vis_cap = (size_t)h->slow_ctas * h->slow_vis_slots;
    }
    // Adapt the visited-table scale to the data: more than 1% of the recent queries needed the retry pass -> double
    // it (read from the pinned mirror of the device counter, i.e. without synchronising; it lags by a call or two).
    w->total_queries += nq;
    {
        const unsigned long long retried = *reinterpret_cast<volatile unsigned long long*>(w->h_retried);
        const unsigned long long dq = w->total_queries - w->seen_total, dr = retried - w->seen_retried;
        if (dq >= 2048) {
            if (dr * 100 > dq) {
                uint32_t cur = h->vis_scale.load();
                // most of the window overflowed: the data simply visits far more nodes -> straight to the maximum
                const uint32_t next = dr * 2 > dq ? 8u : std::min<uint32_t>(8u, cur * 2);
                if (cur < next) h->vis_scale.compare_exchange_strong(cur, next);
            }
            w->seen_total = w->total_queries;
            w->seen_retried = retried;
        }
    }
    // one memset per call: the work counters / gates of the three passes (and the error word of a host-API call);
    // the per-query status words need no reset: the fast pass writes every one of them
    GB_CUDA(cudaMemsetAsync(w->d_counters, 0, reset_error ? 64 : 32, stream));
    gb::SearchArgs a{};
    a.queries = d_queries;
    a.query_format = fmt;
    a.nq = nq;
    a.max_search = max_search;
    a.num_neighbors = k;
    a.list_cap = plan.list_cap;
    a.vis_slots = plan.vis_slots;
    a.vis_slots_upper = plan.vis_upper;
    a.out_ids = d_ids;
    a.out_dists = d_dists;
    a.out_counts = d_counts;
    a.out_stats = d_stats;
    a.query_status = w->d_status;
    a.work_counter = w->d_counters;
    a.retried = w->d_retried;
    a.error_flag = w->d_error;
    a.slow_list = w->d_slow_list;
    a.slow_visited = w->d_slow_vis;
    a.slow_list_cap = h->slow_list_cap;
    a.slow_vis_slots = h->slow_vis_slots;
    a.pass = a.slow_pass = a.final_pass = 0;
    a.pg = gb::PeerGather{};
    if (pg) {
        a.pg.n_peers = pg->n_peers;
        a.pg.my_rank = pg->my_rank;
        a.pg.row_offset = pg->row_offset;
        a.pg.seq = pg->seq;
        a.pg.done_counter = w->d_counters + 5;
        for (uint32_t p = 0; p < pg->n_peers; ++p) {
            a.pg.ids[p] = static_cast<uint32_t*>(pg->ids[p]);
            a.pg.dists[p] = static_cast<float*>(pg->dists[p]);
            a.pg.flags[p] = static_cast<unsigned int*>(pg->flags[p]);
        }
    }
    a.stg_rows = plan.stg_rows;
    a.stg_row_bytes = plan.stg_row_bytes;
    a.tile_rows = plan.tile_rows;
    a.vis_global = nullptr;
    rc = dispatch_search(h, w, a, plan, stream, view ? *view : h->dev);
    if (rc) return rc;
    GB_CUDA(cudaMemcpyAsync(w->h_retried, w->d_retried, 8, cudaMemcpyDeviceToHost, stream));
    return GRANNE_B200_OK;
}

int error_from_bits(int bits) {
    if (bits & gb::kStatusNotFinite)
        return fail(GRANNE_B200_ERR_NOT_FINITE, "a NaN distance occurred (non-finite query or element)");
    if (bits & gb::kStatusOverflow)
        return fail(GRANNE_B200_ERR_CAPACITY, "exact search workspace exhausted even on the slow path");
    return GRANNE_B200_OK;
}

// ---- GranneBuilder (src/index/mod.rs:295-531, 645-960) on the device ---------------------------------------------
struct DistDispatch {
    // calls f.template run<Dist>() for the distance engine that serves `d` (same mapping as dispatch_search)
    template <class F>
    static int call(const gb::DeviceIndex& d, F&& f) {
        switch (d.kind) {
            case gb::kAngularI8: return f.template run<gb::DistI8>();
            case gb::kSumEmbeddings: return f.template run<gb::DistSum>();
            default: break;
        }
        if (d.vec_group == 1 && d.full > 4) return f.template run<gb::DistF32Generic>();
        switch (d.full) {
            case 0: return f.template run<gb::DistF32<0>>();
            case 1: return f.template run<gb::DistF32<1>>();
            case 2: return f.template run<gb::DistF32<2>>();
            case 3: return f.template run<gb::DistF32<3>>();
            case 4: return f.template run<gb::DistF32<4>>();
            case 6: return f.template run<gb::DistF32<6>>();
            case 8: return f.template run<gb::DistF32<8>>();
            default: return f.template run<gb::DistF32Generic>();
        }
    }
};

struct PairLaunch {
    Handle* h;
    gb::PairArgs a;
    size_t smem;
    unsigned grid;
    cudaStream_t stream;
    template <class Dist>
    int run() {
        auto k = gb::pair_distance_kernel<Dist>;
        GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        k<<<grid, 32, smem, stream>>>(h->dev, a);
        h->launches++;
        GB_CUDA(cudaGetLastError());
        return GRANNE_B200_OK;
    }
};

struct LinkLaunch {
    Handle* h;
    gb::BuildArgs a;
    size_t smem;
    unsigned grid;
    cudaStream_t stream;
    bool prune;
    template <class Dist>
    int run() {
        if (prune) {
            auto k = gb::build_prune_kernel<Dist>;
            GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
            k<<<grid, 32, smem, stream>>>(h->dev, a);
        } else {
            auto k = gb::build_link_kernel<Dist>;
            GB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
            k<<<grid, 32, smem, stream>>>(h->dev, a);
        }
        h->launches++;
        GB_CUDA(cudaGetLastError());
        return GRANNE_B200_OK;
    }
};

}  // namespace

struct granne_b200_builder {
    std::unique_ptr<Handle> h;  // search view over the layers built so far (+ the one under construction)
    granne_b200_build_config cfg{};
    uint32_t stride = 0;  // physical row stride (node_width rounded up to 8)
    std::vector<std::shared_ptr<void>> layer_mem;
    Workspace* ws = nullptr;
    // batch scratch
    uint32_t* d_ids = nullptr;
    uint32_t* d_cand_ids = nullptr;
    float* d_cand_d = nullptr;
    uint32_t* d_cand_cnt = nullptr;
    int* d_locks = nullptr;
    unsigned int* d_counter = nullptr;
    size_t batch_cap = 0, cand_cap = 0, locks_cap = 0;
};

namespace {

using Builder = granne_b200_builder;

int builder_reserve(Builder* b, size_t batch, size_t ef, size_t nodes) {
    if (batch > b->batch_cap || ef > b->cand_cap) {
        cudaFree(b->d_ids);
        cudaFree(b->d_cand_ids);
        cudaFree(b->d_cand_d);
        cudaFree(b->d_cand_cnt);
        b->d_ids = nullptr, b->d_cand_ids = nullptr, b->d_cand_d = nullptr, b->d_cand_cnt = nullptr;
        b->batch_cap = std::max(batch, b->batch_cap);
        b->cand_cap = std::max(ef, b->cand_cap);
        GB_CUDA(cudaMalloc(&b->d_ids, b->batch_cap * 4));
        GB_CUDA(cudaMalloc(&b->d_cand_ids, b->batch_cap * b->cand_cap * 4));
        GB_CUDA(cudaMalloc(&b->d_cand_d, b->batch_cap * b->cand_cap * 4));
        GB_CUDA(cudaMalloc(&b->d_cand_cnt, b->batch_cap * 4));
    }
    if (nodes > b->locks_cap) {
        cudaFree(b->d_locks);
        b->d_locks = nullptr;
        GB_CUDA(cudaMalloc(&b->d_locks, nodes * sizeof(int)));
        b->locks_cap = nodes;
    }
    if (!b->d_counter) GB_CUDA(cudaMalloc(&b->d_counter, 16));
    return GRANNE_B200_OK;
}

// index_elements (:716-802) for the layer at dev.layer_rows[num_layers-1]
int builder_index_elements(Builder* b, uint32_t layer_m, uint32_t ef, uint64_t already, uint64_t num, bool reinsert) {
    Handle* h = b->h.get();
    gb::DeviceIndex& d = h->dev;
    const int cur = d.num_layers - 1;
    uint32_t* rows = const_cast<uint32_t*>(d.layer_rows[cur]);
    cudaStream_t stream = b->ws->stream;
    const LaunchPlan plan = make_plan(h, ef);
    if (plan.smem == 0) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search too large");
    const uint64_t first = reinsert ? 0 : already;
    const uint64_t total = num - first;
    // test knob: GRANNE_B200_BUILD_MAX_BATCH=1 makes every insertion see all earlier links, i.e. the reference's
    // `singlethreaded` build order (read on every call so that one process can switch it)
    size_t max_batch = 4096;
    if (const char* e = std::getenv("GRANNE_B200_BUILD_MAX_BATCH")) max_batch = (size_t)std::max(1, std::atoi(e));
    // test knob: GRANNE_B200_BUILD_LINK_WARPS caps the warps that link a batch in (default num_sms x 8).  At 1 the work
    // counter hands out the members in batch order, so a batched build is deterministic.  The prune pass needs no cap:
    // each warp there writes only its own node's row.
    uint64_t link_warps = (uint64_t)h->num_sms * 8;
    if (const char* e = std::getenv("GRANNE_B200_BUILD_LINK_WARPS"))
        link_warps = std::min<uint64_t>(link_warps, (uint64_t)std::max(1, std::atoi(e)));
    int rc = builder_reserve(b, max_batch, ef, num);
    if (rc) return rc;
    GB_CUDA(cudaMemsetAsync(b->d_locks, 0, num * sizeof(int), stream));
    const size_t link_smem = plan.base_smem + gb::link_scratch_bytes(gb::link_cand_cap(ef, b->cfg.num_neighbors),
                                                                      b->cfg.num_neighbors) + 64;
    uint64_t pos = 0;
    while (pos < total) {
        // nodes already linked into this layer: a batch never exceeds 1/16 of them (its members do not see each other)
        const uint64_t present = reinsert ? num : first + pos;
        const uint64_t bsz = std::min<uint64_t>(std::min<uint64_t>(max_batch, std::max<uint64_t>(1, present / 16)), total - pos);
        const uint32_t start = reinsert ? (uint32_t)(num - 1 - pos) : (uint32_t)(first + pos);
        gb::iota_kernel<<<(unsigned)((bsz + 255) / 256), 256, 0, stream>>>(b->d_ids, (uint32_t)bsz, start, reinsert ? -1 : 1);
        h->launches++;
        // candidates = search_for_neighbors(layer, prev_layers.search(e,1,1), e, max_search) (:819-820)
        rc = enqueue_search(h, b->ws, b->d_ids, bsz, gb::kQueryById, ef, ef, b->d_cand_ids, b->d_cand_d, b->d_cand_cnt,
                            nullptr, stream, false);
        if (rc) return rc;
        GB_CUDA(cudaMemsetAsync(b->d_counter, 0, 16, stream));
        LinkLaunch L{h, {}, link_smem, 0, stream, false};
        L.a.ids = b->d_ids;
        L.a.n_batch = (uint32_t)bsz;
        L.a.cand_ids = b->d_cand_ids;
        L.a.cand_dists = b->d_cand_d;
        L.a.cand_counts = b->d_cand_cnt;
        L.a.cand_stride = ef;
        L.a.rows = rows;
        L.a.stride = b->stride;
        L.a.node_width = b->cfg.num_neighbors;
        L.a.max_neighbors = layer_m;
        L.a.locks = b->d_locks;
        L.a.stg_rows = plan.stg_rows;
        L.a.stg_row_bytes = plan.stg_row_bytes;
        L.a.tile_rows = plan.tile_rows;
        L.a.work_counter = b->d_counter;
        L.a.num_nodes = (uint32_t)num;
        L.grid = (unsigned)std::min<uint64_t>(bsz, link_warps);
        if ((rc = DistDispatch::call(d, L))) return rc;
        pos += bsz;
    }
    // limit number of neighbors (:794-797)
    GB_CUDA(cudaMemsetAsync(b->d_counter, 0, 16, stream));
    LinkLaunch P{h, {}, plan.base_smem + gb::link_scratch_bytes(gb::link_cand_cap(0, b->cfg.num_neighbors),
                                                               b->cfg.num_neighbors) + 64, 0, stream, true};
    P.a.rows = rows;
    P.a.stride = b->stride;
    P.a.node_width = b->cfg.num_neighbors;
    P.a.max_neighbors = layer_m;
    P.a.stg_rows = plan.stg_rows;
    P.a.stg_row_bytes = plan.stg_row_bytes;
    P.a.tile_rows = plan.tile_rows;
    P.a.work_counter = b->d_counter;
    P.a.num_nodes = (uint32_t)num;
    P.grid = (unsigned)std::min<uint64_t>(num, (uint64_t)h->num_sms * 8);
    if ((rc = DistDispatch::call(d, P))) return rc;
    GB_CUDA(cudaStreamSynchronize(stream));
    int herr[4] = {0, 0, 0, 0};
    GB_CUDA(cudaMemcpy(herr, b->ws->d_error, sizeof(herr), cudaMemcpyDeviceToHost));
    GB_CUDA(cudaMemset(b->ws->d_error, 0, sizeof(herr)));
    return error_from_bits(herr[0]);
}

// index_elements_in_last_layer (:646-713)
int builder_index_last_layer(Builder* b, uint64_t max_num_elements) {
    Handle* h = b->h.get();
    gb::DeviceIndex& d = h->dev;
    const int cur = d.num_layers - 1;
    const uint64_t total = b->cfg.expected_num_elements >= 0 ? (uint64_t)b->cfg.expected_num_elements : d.num_elements;
    const uint64_t ideal =
        gb::num_elements_in_layer(std::max<uint64_t>(total, d.num_elements), b->cfg.layer_multiplier, (uint64_t)cur);
    const uint64_t have = d.layer_len[cur];
    if (ideal <= have) return GRANNE_B200_OK;  // nothing to index in this layer
    const uint64_t num = std::min<uint64_t>(max_num_elements, ideal);
    uint32_t layer_m = b->cfg.num_neighbors;
    if (ideal < total) layer_m = std::max<uint32_t>(1, layer_m / 2);  // half num_neighbors on upper layers
    // the layer grows: fresh allocation (snapshots handed out by get_index keep the old one alive)
    uint32_t* grown = nullptr;
    GB_CUDA(cudaMalloc(&grown, std::max<size_t>((size_t)num * b->stride * 4, 16)));
    std::shared_ptr<void> mem(grown, [](void* q) { cudaFree(q); });
    cudaStream_t stream = b->ws->stream;
    gb::fill_u32_kernel<<<h->num_sms * 4, 256, 0, stream>>>(grown, (unsigned long long)num * b->stride, gb::kUnusedId);
    h->launches++;
    if (have) GB_CUDA(cudaMemcpyAsync(grown, d.layer_rows[cur], (size_t)have * b->stride * 4, cudaMemcpyDeviceToDevice, stream));
    b->layer_mem[cur] = mem;
    d.layer_rows[cur] = grown;
    d.layer_len[cur] = num;
    h->layer_max_degree[cur] = b->cfg.num_neighbors;
    finish_handle(h);
    int rc = builder_index_elements(b, layer_m, b->cfg.max_search, have, num, false);
    if (rc) return rc;
    if (b->cfg.reinsert_elements) {
        // use half max_search when reindexing (:698-699)
        rc = builder_index_elements(b, layer_m, std::max<uint32_t>(1, b->cfg.max_search / 2), 0, num, true);
        if (rc) return rc;
    }
    return GRANNE_B200_OK;
}

// build_partial (:374-402)
int builder_build_partial(Builder* b, uint64_t num_elements) {
    Handle* h = b->h.get();
    gb::DeviceIndex& d = h->dev;
    if (num_elements == 0) return GRANNE_B200_OK;
    if (num_elements < h->index_len)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "Cannot index fewer elements than already in index.");
    if (num_elements > d.num_elements)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "Cannot index more elements than exist.");
    GB_DEVICE(h->device);
    int rc;
    if (d.num_layers > 0 && (rc = builder_index_last_layer(b, num_elements))) return rc;
    while (h->index_len < num_elements) {
        if (d.num_layers >= gb::kMaxLayers) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many layers");
        // new layer = clone of the previous one (:392-398)
        const int l = d.num_layers;
        d.layer_rows[l] = l ? d.layer_rows[l - 1] : nullptr;
        d.layer_len[l] = l ? d.layer_len[l - 1] : 0;
        d.layer_width[l] = b->stride;
        d.num_layers = l + 1;
        b->layer_mem.push_back(l ? b->layer_mem[l - 1] : std::shared_ptr<void>());
        h->layer_max_degree.push_back(b->cfg.num_neighbors);
        finish_handle(h);
        if ((rc = builder_index_last_layer(b, num_elements))) return rc;
    }
    return GRANNE_B200_OK;
}

}  // namespace

// =================================================================================================================
// C ABI
// =================================================================================================================
extern "C" {

int granne_b200_abi_version(void) { return GRANNE_B200_ABI_VERSION; }

const char* granne_b200_last_error(void) { return g_last_error.c_str(); }

int granne_b200_open(const void* index_bytes, size_t index_len, int element_kind, const void* elements_bytes,
                     size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                     granne_b200_index** out) {
    try {
        return open_impl(static_cast<const uint8_t*>(index_bytes), index_len, element_kind,
                         static_cast<const uint8_t*>(elements_bytes), elements_len,
                         static_cast<const uint8_t*>(embeddings_bytes), embeddings_len, device, out);
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_open_device_elements(const void* index_bytes, size_t index_len, int element_kind,
                                     const void* d_element_rows, uint64_t num_elements, uint32_t dim, int device,
                                     granne_b200_index** out) {
    try {
        if (!d_element_rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
        return open_impl(static_cast<const uint8_t*>(index_bytes), index_len, element_kind, nullptr, 0, nullptr, 0,
                         device, out, d_element_rows, num_elements, dim);
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_open_files(const char* index_path, int element_kind, const char* elements_path,
                           const char* embeddings_path, int device, granne_b200_index** out) {
    try {
        std::vector<uint8_t> ib, eb, mb;
        int rc;
        if ((rc = read_file(index_path, &ib))) return rc;
        if ((rc = read_file(elements_path, &eb))) return rc;
        if (element_kind == GRANNE_B200_EMBEDDINGS) {
            if (!embeddings_path)
                return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "embeddings_path required for this element type!");
            if ((rc = read_file(embeddings_path, &mb))) return rc;
        }
        return open_impl(ib.data(), ib.size(), element_kind, eb.data(), eb.size(), mb.empty() ? nullptr : mb.data(),
                         mb.size(), device, out);
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

void granne_b200_close(granne_b200_index* h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    for (auto& w : h->pool) ws_destroy(w.get());
    h->pool.clear();
    for (auto& kv : h->stream_ws) ws_destroy(kv.second.get());
    h->stream_ws.clear();
    h->allocations.clear();
    delete h;
}

uint64_t granne_b200_len(const granne_b200_index* h) { return h ? h->index_len : 0; }
uint64_t granne_b200_num_layers(const granne_b200_index* h) { return h ? (uint64_t)h->dev.num_layers : 0; }
uint64_t granne_b200_layer_len(const granne_b200_index* h, uint64_t layer) {
    if (!h || layer >= (uint64_t)h->dev.num_layers) return 0;
    return h->dev.layer_len[layer];
}
uint64_t granne_b200_num_elements(const granne_b200_index* h) { return h ? h->dev.num_elements : 0; }
uint64_t granne_b200_dim(const granne_b200_index* h) { return h ? h->dev.dim : 0; }
int granne_b200_element_kind(const granne_b200_index* h) { return h ? h->dev.kind : -1; }
uint64_t granne_b200_launch_count(const granne_b200_index* h) { return h ? h->launches.load() : 0; }
uint64_t granne_b200_device_bytes(const granne_b200_index* h) { return h ? h->device_bytes : 0; }

int granne_b200_get_neighbors(const granne_b200_index* h, uint64_t idx, uint64_t layer, uint32_t* out, size_t cap,
                              size_t* out_n) {
    if (!h || !out_n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (layer >= (uint64_t)h->dev.num_layers || idx >= h->dev.layer_len[layer])
        return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "node or layer out of range");
    GB_DEVICE(h->device);
    const uint32_t w = h->dev.layer_width[layer];
    std::vector<uint32_t> row(w);
    GB_CUDA(cudaMemcpy(row.data(), h->dev.layer_rows[layer] + idx * w, w * 4, cudaMemcpyDeviceToHost));
    size_t n = 0;
    while (n < w && row[n] != gb::kUnusedId) ++n;
    *out_n = n;
    for (size_t i = 0; i < n && i < cap && out; ++i) out[i] = row[i];
    return GRANNE_B200_OK;
}

int granne_b200_get_element(const granne_b200_index* hc, uint64_t idx, void* out) {
    granne_b200_index* h = const_cast<granne_b200_index*>(hc);
    if (!h || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (idx >= h->dev.num_elements) return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "element index out of range");
    GB_DEVICE(h->device);
    const size_t bytes = h->dev.kind == gb::kAngularI8 ? h->dev.dim : (size_t)h->dev.dim * 4;
    void* d = nullptr;
    GB_CUDA(cudaMalloc(&d, bytes));
    gb::get_element_kernel<<<1, 32>>>(h->dev, idx, d);
    h->launches++;
    cudaError_t e = cudaMemcpy(out, d, bytes, cudaMemcpyDeviceToHost);
    cudaFree(d);
    GB_CUDA(e);
    return GRANNE_B200_OK;
}

static int search_device_impl(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                              uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                              uint32_t* d_out_counts, uint64_t* d_out_stats, void* cuda_stream,
                              const granne_b200_peer_gather* pg) {
    int rc = validate_search(h, d_queries, nq, query_format, max_search, num_neighbors, pg ? (void*)pg : d_out_ids,
                             pg ? (void*)pg : d_out_dists);
    if (rc) return rc;
    if (pg) {
        if (pg->n_peers < 1 || pg->n_peers > GRANNE_B200_MAX_PEERS || pg->my_rank >= pg->n_peers)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "peer gather: n_peers must be 1..8 and my_rank < n_peers");
        for (uint32_t p = 0; p < pg->n_peers; ++p)
            if (!pg->ids[p] || !pg->dists[p] || !pg->flags[p])
                return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "peer gather: null peer pointer");
    }
    if (nq == 0) return GRANNE_B200_OK;
    GB_DEVICE(h->device);
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    // One workspace per caller stream: calls on the same stream are serialised by the stream itself, so the status
    // words / slow-path buffers can be reused; the error word stays sticky until granne_b200_stream_status().
    Workspace* w = nullptr;
    {
        std::lock_guard<std::mutex> g(h->pool_mu);
        auto it = h->stream_ws.find(stream);
        if (it != h->stream_ws.end()) w = it->second.get();
    }
    if (!w) {
        Workspace* fresh = nullptr;
        if ((rc = ws_acquire(h, &fresh))) return rc;
        cudaError_t e = cudaMemset(fresh->d_error, 0, 4 * sizeof(int));
        bool lost_race = false;
        {
            std::lock_guard<std::mutex> g(h->pool_mu);
            auto it = h->stream_ws.find(stream);  // two threads may meet here on the first use of a stream
            if (it != h->stream_ws.end()) {
                w = it->second.get();
                lost_race = true;
            } else {
                h->stream_ws[stream] = std::unique_ptr<Workspace>(fresh);
                w = fresh;
            }
        }
        if (lost_race) ws_release(h, fresh);  // back to the pool, nothing is leaked
        GB_CUDA(e);
    }
    return enqueue_search(h, w, d_queries, nq, query_format, max_search, num_neighbors, d_out_ids, d_out_dists,
                          d_out_counts, reinterpret_cast<unsigned long long*>(d_out_stats), stream, false, pg);
}

int granne_b200_search_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                    uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids,
                                    float* d_out_dists, uint32_t* d_out_counts, uint64_t* d_out_stats,
                                    void* cuda_stream) {
    return search_device_impl(h, d_queries, nq, query_format, max_search, num_neighbors, d_out_ids, d_out_dists,
                              d_out_counts, d_out_stats, cuda_stream, nullptr);
}

int granne_b200_search_batch_device_gather(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_neighbors,
                                           const granne_b200_peer_gather* gather, uint32_t* d_out_counts,
                                           uint64_t* d_out_stats, void* cuda_stream) {
    if (!gather) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "peer gather descriptor is null");
    return search_device_impl(h, d_queries, nq, query_format, max_search, num_neighbors, nullptr, nullptr,
                              d_out_counts, d_out_stats, cuda_stream, gather);
}

// The device-pointer API keeps one workspace per distinct caller stream (status words, visited tables: up to
// ~1 GB at large max_search).  A caller that retires a stream hands its workspace back with this call (it synchronises
// the stream first); granne_b200_close releases everything anyway.
int granne_b200_release_stream(granne_b200_index* h, void* cuda_stream) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    GB_DEVICE(h->device);
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    std::unique_ptr<Workspace> w;
    {
        std::lock_guard<std::mutex> g(h->pool_mu);
        auto it = h->stream_ws.find(stream);
        if (it == h->stream_ws.end()) return GRANNE_B200_OK;
        w = std::move(it->second);
        h->stream_ws.erase(it);
    }
    GB_CUDA(cudaStreamSynchronize(stream));
    int e[4] = {0, 0, 0, 0};
    GB_CUDA(cudaMemcpy(e, w->d_error, sizeof(e), cudaMemcpyDeviceToHost));
    h->sticky_error.fetch_or(e[0]);  // reported by the next granne_b200_stream_status
    ws_destroy(w.get());
    return GRANNE_B200_OK;
}

int granne_b200_stream_status(granne_b200_index* h) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    GB_DEVICE(h->device);
    GB_CUDA(cudaDeviceSynchronize());
    int bits = h->sticky_error.exchange(0);
    std::lock_guard<std::mutex> g(h->pool_mu);
    for (auto& kv : h->stream_ws) {
        int e[4] = {0, 0, 0, 0};
        GB_CUDA(cudaMemcpy(e, kv.second->d_error, sizeof(e), cudaMemcpyDeviceToHost));
        bits |= e[0];
        GB_CUDA(cudaMemset(kv.second->d_error, 0, sizeof(e)));
    }
    return error_from_bits(bits);
}

int granne_b200_search_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                             uint32_t max_search, uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                             uint32_t* out_counts, uint64_t* out_stats) {
    int rc = validate_search(h, queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    GB_DEVICE(h->device);
    const size_t k = num_neighbors;
    const bool i8q = h->dev.kind == gb::kAngularI8 && query_format == GRANNE_B200_QUERY_ELEMENT;
    const size_t qbytes = nq * h->dev.dim * (i8q ? 1 : 4);
    Workspace* w = nullptr;
    if ((rc = ws_acquire(h, &w))) return rc;
    struct Releaser {
        Handle* h;
        Workspace* w;
        ~Releaser() { ws_release(h, w); }
    } rel{h, w};
    if ((rc = ws_reserve(w, qbytes, nq, k))) return rc;
    // pinned staging layout: queries | ids | dists | counts | stats | error
    uint8_t* hp = static_cast<uint8_t*>(w->h_pinned);
    uint8_t* hq = hp;
    uint32_t* hids = reinterpret_cast<uint32_t*>(hp + ((qbytes + 15) & ~size_t(15)));
    float* hd = reinterpret_cast<float*>(hids + nq * k);
    uint32_t* hc = reinterpret_cast<uint32_t*>(hd + nq * k);
    int* herr = reinterpret_cast<int*>(hc + nq);
    unsigned long long* hstats = reinterpret_cast<unsigned long long*>(
        reinterpret_cast<uint8_t*>(hp) + ((reinterpret_cast<uint8_t*>(herr + 4) - hp + 15) & ~size_t(15)));
    // (pinned_cap was sized with slack for the alignment above)
    std::memcpy(hq, queries, qbytes);
    GB_CUDA(cudaMemcpyAsync(w->d_queries, hq, qbytes, cudaMemcpyHostToDevice, w->stream));
    rc = enqueue_search(h, w, w->d_queries, nq, query_format, max_search, num_neighbors, w->d_ids, w->d_dists,
                        w->d_counts, out_stats ? w->d_stats : nullptr, w->stream, true);
    if (rc) return rc;
    // one packed copy: ids | dists | counts (device and pinned layouts match), then the 16-byte error word
    GB_CUDA(cudaMemcpyAsync(hids, w->d_ids, (2 * nq * k + nq) * 4, cudaMemcpyDeviceToHost, w->stream));
    GB_CUDA(cudaMemcpyAsync(herr, w->d_error, 4 * sizeof(int), cudaMemcpyDeviceToHost, w->stream));
    if (out_stats) GB_CUDA(cudaMemcpyAsync(hstats, w->d_stats, nq * 32, cudaMemcpyDeviceToHost, w->stream));
    GB_CUDA(cudaStreamSynchronize(w->stream));
    if (out_stats) std::memcpy(out_stats, hstats, nq * 32);
    if (k) {
        std::memcpy(out_ids, hids, nq * k * 4);
        std::memcpy(out_dists, hd, nq * k * 4);
    }
    if (out_counts) std::memcpy(out_counts, hc, nq * 4);
    return error_from_bits(herr[0]);
}

int granne_b200_inspect_index(const void* index_bytes, size_t index_len, uint64_t* out_num_layers,
                              uint64_t* out_layer_len, uint32_t* out_max_degree, uint32_t* out_row_width, size_t cap) {
    if (!index_bytes || !out_num_layers) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        *out_num_layers = graph.layers.size();
        for (size_t l = 0; l < graph.layers.size() && l < cap; ++l) {
            if (out_layer_len) out_layer_len[l] = graph.layers[l].num_nodes;
            if (out_max_degree) out_max_degree[l] = graph.layers[l].max_degree;
            if (out_row_width) out_row_width[l] = graph.layers[l].width;
        }
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_decode_layer(const void* index_bytes, size_t index_len, uint64_t layer, uint32_t* rows,
                             size_t rows_cap_u32) {
    if (!index_bytes || !rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        if (layer >= graph.layers.size()) return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "layer out of range");
        const gb::HostLayer& L = graph.layers[layer];
        if (L.rows.size() > rows_cap_u32) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "rows buffer too small");
        std::memcpy(rows, L.rows.data(), L.rows.size() * 4);
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

// ---- GranneBuilder ------------------------------------------------------------------------------------------------
void granne_b200_build_config_default(granne_b200_build_config* cfg) {
    if (!cfg) return;
    cfg->layer_multiplier = 15.0f;
    cfg->expected_num_elements = -1;
    cfg->num_neighbors = 30;
    cfg->max_search = 200;
    cfg->reinsert_elements = 1;
    cfg->show_progress = 0;
}

static int builder_new_impl(const granne_b200_build_config* cfg, int element_kind, const void* elements_bytes,
                            size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                            granne_b200_builder** out, const void* dev_rows, uint64_t n_dev, uint32_t dim_dev) {
    try {
        if (!out || !cfg) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
        *out = nullptr;
        int rc = dev_rows ? GRANNE_B200_OK : check_open_args(elements_bytes, element_kind, embeddings_bytes);
        if (rc) return rc;
        // the on-disk format counts a list's entries in one byte (set_vector.rs:91-99): 255 is the format's limit
        if (cfg->num_neighbors < 1 || cfg->num_neighbors > 255)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "num_neighbors must be in 1..255");
        if (cfg->max_search < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search must be >= 1");
        if (!(cfg->layer_multiplier > 1.0f))
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "layer_multiplier must be > 1");
        std::unique_ptr<granne_b200_builder> b(new granne_b200_builder());
        b->cfg = *cfg;
        b->stride = (cfg->num_neighbors + 7u) & ~7u;
        b->h.reset(new Handle());
        Handle* h = b->h.get();
        rc = check_device(device, &h->num_sms, &h->smem_optin);
        if (rc) return rc;
        h->device = device;
        GB_DEVICE(device);
        if (dev_rows)
            rc = stage_device_elements(h, element_kind, dev_rows, n_dev, dim_dev);
        else
            rc = stage_elements(h, element_kind, static_cast<const uint8_t*>(elements_bytes), elements_len,
                                static_cast<const uint8_t*>(embeddings_bytes), embeddings_len);
        if (rc) return rc;
        if (h->dev.num_elements >= 0xFFFFFFFFull)  // assert!(elements.len() < UNUSED) (:420)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many elements");
        h->dev.num_layers = 0;
        finish_handle(h);
        if ((rc = ws_acquire(h, &b->ws))) return rc;
        GB_CUDA(cudaMemset(b->ws->d_error, 0, 4 * sizeof(int)));
        *out = b.release();
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_builder_new(const granne_b200_build_config* cfg, int element_kind, const void* elements_bytes,
                            size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                            granne_b200_builder** out) {
    return builder_new_impl(cfg, element_kind, elements_bytes, elements_len, embeddings_bytes, embeddings_len, device,
                            out, nullptr, 0, 0);
}

int granne_b200_builder_new_device_elements(const granne_b200_build_config* cfg, int element_kind,
                                            const void* d_element_rows, uint64_t num_elements, uint32_t dim,
                                            int device, granne_b200_builder** out) {
    if (!d_element_rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
    return builder_new_impl(cfg, element_kind, nullptr, 0, nullptr, 0, device, out, d_element_rows, num_elements, dim);
}

// GranneBuilder::push for the dense containers (ExtendableElementContainer::push, src/index/mod.rs:512-531;
// src/elements/dense_vector.rs:120-136): `elements_bytes` is an elements file image of the same width whose rows are
// appended to the staged container.  The appended elements are indexed by the next build() / build_partial().
int granne_b200_builder_append(granne_b200_builder* b, const void* elements_bytes, size_t elements_len) {
    if (!b || !elements_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        Handle* h = b->h.get();
        gb::DeviceIndex& d = h->dev;
        if (d.kind == gb::kSumEmbeddings) {
            // ExtendableElementContainer for SumEmbeddings (src/elements/embeddings/mod.rs:97-100,177-189): the image
            // holds the new elements' term lists (VariableWidthSliceVector, src/slice_vector/mod.rs:660-676); they
            // are appended behind the staged ones, the embedding table is unchanged
            gb::SumElements se;
            std::string err;
            if (!gb::parse_sum_elements(static_cast<const uint8_t*>(elements_bytes), elements_len, &se, &err))
                return fail(GRANNE_B200_ERR_FORMAT, err);
            const uint64_t add = se.offsets.size() - 1;
            if (add == 0) return GRANNE_B200_OK;
            for (uint32_t t : se.terms)
                if (t >= d.num_vectors) return fail(GRANNE_B200_ERR_FORMAT, "element refers to a missing embedding id");
            const uint64_t old_n = d.num_elements, new_n = old_n + add;
            if (new_n >= 0xFFFFFFFFull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many elements");  // :420
            GB_DEVICE(h->device);
            GB_CUDA(cudaStreamSynchronize(b->ws->stream));
            unsigned long long old_terms = 0;
            if (old_n)
                GB_CUDA(cudaMemcpy(&old_terms, d.sum_offsets + old_n, 8, cudaMemcpyDeviceToHost));
            std::vector<unsigned long long> off(add + 1);
            for (uint64_t i = 0; i <= add; ++i) off[i] = old_terms + se.offsets[i];
            unsigned long long* doff = nullptr;
            uint32_t* dterms = nullptr;
            int rc;
            if ((rc = dev_alloc(h, &doff, new_n + 1))) return rc;
            if ((rc = dev_alloc(h, &dterms, (size_t)old_terms + se.terms.size()))) return rc;
            if (old_n) {
                GB_CUDA(cudaMemcpy(doff, d.sum_offsets, (size_t)old_n * 8, cudaMemcpyDeviceToDevice));
                if (old_terms) GB_CUDA(cudaMemcpy(dterms, d.sum_terms, (size_t)old_terms * 4, cudaMemcpyDeviceToDevice));
            }
            GB_CUDA(cudaMemcpy(doff + old_n, off.data(), (add + 1) * 8, cudaMemcpyHostToDevice));
            if (!se.terms.empty())
                GB_CUDA(cudaMemcpy(dterms + old_terms, se.terms.data(), se.terms.size() * 4, cudaMemcpyHostToDevice));
            // (the old arrays stay alive in h->allocations: snapshots handed out by get_index may still read them)
            d.sum_offsets = doff;
            d.sum_terms = dterms;
            d.num_elements = new_n;
            return GRANNE_B200_OK;
        }
        if (d.kind != gb::kAngularF32 && d.kind != gb::kAngularI8)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unknown element kind");
        const bool i8 = d.kind == gb::kAngularI8;
        const size_t esz = i8 ? 1 : 4;
        gb::DenseView dv;
        std::string err;
        if (!gb::parse_dense(static_cast<const uint8_t*>(elements_bytes), elements_len, esz, &dv, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        if (dv.dim != d.dim) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "appended elements have a different width");
        if (dv.num == 0) return GRANNE_B200_OK;
        const uint64_t old_n = d.num_vectors, new_n = old_n + dv.num;
        if (new_n >= 0xFFFFFFFFull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many elements");  // :420
        GB_DEVICE(h->device);
        GB_CUDA(cudaStreamSynchronize(b->ws->stream));
        const size_t row_bytes = (size_t)d.row_stride * esz;
        uint8_t* dst = nullptr;
        GB_CUDA(cudaMalloc(&dst, std::max<size_t>((size_t)new_n * row_bytes, 16)));
        std::shared_ptr<void> owner(dst, [](void* q) { cudaFree(q); });
        if (old_n) GB_CUDA(cudaMemcpy(dst, d.vectors, (size_t)old_n * row_bytes, cudaMemcpyDeviceToDevice));
        // new rows: upload in slabs, then the same re-layout kernels as the loader
        const uint64_t slab = std::max<uint64_t>(1, (64ull << 20) / ((size_t)d.dim * esz));
        uint8_t* tmp = nullptr;
        GB_CUDA(cudaMalloc(&tmp, (size_t)std::min<uint64_t>(slab, dv.num) * d.dim * esz));
        std::shared_ptr<void> tmp_owner(tmp, [](void* q) { cudaFree(q); });
        for (uint64_t r0 = 0; r0 < dv.num; r0 += slab) {
            const uint64_t nr = std::min<uint64_t>(slab, dv.num - r0);
            GB_CUDA(cudaMemcpy(tmp, dv.data + r0 * d.dim * esz, (size_t)nr * d.dim * esz, cudaMemcpyHostToDevice));
            uint8_t* out_rows = dst + (size_t)(old_n + r0) * row_bytes;
            if (i8)
                gb::pad_rows_i8_kernel<<<h->num_sms * 8, 256>>>(reinterpret_cast<const int8_t*>(tmp),
                                                                reinterpret_cast<int8_t*>(out_rows), nr, d.dim,
                                                                d.row_stride);
            else
                gb::permute_rows_f32_kernel<<<h->num_sms * 8, 256>>>(reinterpret_cast<const float*>(tmp),
                                                                     reinterpret_cast<float*>(out_rows), nr, d.dim,
                                                                     d.full, d.vec_group, d.row_stride);
            h->launches++;
            GB_CUDA(cudaGetLastError());
        }
        GB_CUDA(cudaDeviceSynchronize());
        // swap the container; snapshots handed out by get_index keep the old buffer alive through their own reference
        for (auto it = h->allocations.begin(); it != h->allocations.end(); ++it)
            if (it->get() == d.vectors) {
                h->device_bytes -= std::min<uint64_t>(h->device_bytes, std::max<size_t>((size_t)old_n * row_bytes, 16));
                h->allocations.erase(it);
                break;
            }
        h->allocations.push_back(owner);
        h->device_bytes += std::max<size_t>((size_t)new_n * row_bytes, 16);
        d.vectors = dst;
        d.num_vectors = new_n;
        d.num_elements = new_n;
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_builder_build(granne_b200_builder* b, uint64_t num_elements) {
    if (!b) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "builder is null");
    try {
        return builder_build_partial(b, num_elements ? num_elements : b->h->dev.num_elements);
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

uint64_t granne_b200_builder_len(const granne_b200_builder* b) { return b ? b->h->index_len : 0; }
uint64_t granne_b200_builder_num_layers(const granne_b200_builder* b) { return b ? (uint64_t)b->h->dev.num_layers : 0; }
uint64_t granne_b200_builder_layer_len(const granne_b200_builder* b, uint64_t layer) {
    if (!b || layer >= (uint64_t)b->h->dev.num_layers) return 0;
    return b->h->dev.layer_len[layer];
}
uint64_t granne_b200_builder_num_elements(const granne_b200_builder* b) { return b ? b->h->dev.num_elements : 0; }
int granne_b200_builder_get_neighbors(const granne_b200_builder* b, uint64_t idx, uint64_t layer, uint32_t* out,
                                      size_t cap, size_t* n_out) {
    if (!b) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null builder");
    return granne_b200_get_neighbors(b->h.get(), idx, layer, out, cap, n_out);
}

// Index::write_index (src/index/io.rs:11-70) from the staged fixed-width rows of any handle.
int granne_b200_write_index(const granne_b200_index* h, void* out, size_t cap, size_t* out_len) {
    if (!h || !out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        GB_DEVICE(h->device);
        std::vector<std::vector<uint32_t>> host(h->dev.num_layers);
        std::vector<gb::LayerView> views;
        for (int l = 0; l < h->dev.num_layers; ++l) {
            const uint32_t stride = h->dev.layer_width[l];
            const size_t n = (size_t)h->dev.layer_len[l] * stride;
            host[l].resize(n);
            if (n) GB_CUDA(cudaMemcpy(host[l].data(), h->dev.layer_rows[l], n * 4, cudaMemcpyDeviceToHost));
            views.push_back({host[l].data(), h->dev.layer_len[l], stride});
        }
        std::vector<uint8_t> image;
        std::string err;
        if (!gb::encode_index(views, &image, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        *out_len = image.size();
        if (!out) return GRANNE_B200_OK;
        if (cap < image.size()) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
        std::memcpy(out, image.data(), image.size());
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_builder_write_index(granne_b200_builder* b, void* out, size_t cap, size_t* out_len) {
    if (!b) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return granne_b200_write_index(b->h.get(), out, cap, out_len);
}

int granne_b200_builder_get_index(granne_b200_builder* b, granne_b200_index** out) {
    if (!b || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        const Handle* src = b->h.get();
        std::unique_ptr<Handle> h(new Handle());
        h->device = src->device;
        h->num_sms = src->num_sms;
        h->smem_optin = src->smem_optin;
        h->dev = src->dev;
        h->allocations = src->allocations;  // shared ownership of the staged elements
        for (const auto& m : b->layer_mem)
            if (m) h->allocations.push_back(m);
        h->device_bytes = src->device_bytes;
        h->layer_max_degree = src->layer_max_degree;
        finish_handle(h.get());
        *out = h.release();
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

void granne_b200_builder_free(granne_b200_builder* b) {
    if (!b) return;
    DeviceGuard guard(b->h->device);
    cudaDeviceSynchronize();
    cudaFree(b->d_ids);
    cudaFree(b->d_cand_ids);
    cudaFree(b->d_cand_d);
    cudaFree(b->d_cand_cnt);
    cudaFree(b->d_locks);
    cudaFree(b->d_counter);
    if (b->ws) {
        ws_destroy(b->ws);
        delete b->ws;
    }
    delete b;
}

int granne_b200_elements_from_raw(int element_kind, const float* raw, uint64_t n, uint32_t dim, int device, void* out,
                                  size_t cap, size_t* out_len) {
    if (!out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (element_kind != GRANNE_B200_ANGULAR && element_kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements_from_raw builds angular or angular_int vectors");
    if (dim == 0 || dim > 8192) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "dim must be in 1..8192");
    const size_t esz = element_kind == GRANNE_B200_ANGULAR ? 4 : 1;
    const size_t need = 8 + (size_t)n * dim * esz;
    *out_len = need;
    if (!out) return GRANNE_B200_OK;
    if (cap < need) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
    if (n && !raw) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    int sms = 0;
    size_t optin = 0;
    int rc = check_device(device, &sms, &optin);
    if (rc) return rc;
    GB_DEVICE(device);
    uint8_t* o = static_cast<uint8_t*>(out);
    for (int b8 = 0; b8 < 8; ++b8) o[b8] = (uint8_t)((uint64_t)dim >> (8 * b8));
    const uint64_t slab = std::max<uint64_t>(1, (256ull << 20) / ((size_t)dim * 4));
    float* d_raw = nullptr;
    void* d_out = nullptr;
    const uint64_t rows_alloc = std::min<uint64_t>(slab, std::max<uint64_t>(n, 1));
    GB_CUDA(cudaMalloc(&d_raw, rows_alloc * dim * 4));
    cudaError_t e = cudaMalloc(&d_out, rows_alloc * dim * esz);
    if (e != cudaSuccess) {
        cudaFree(d_raw);
        GB_CUDA(e);
    }
    for (uint64_t r0 = 0; r0 < n && rc == GRANNE_B200_OK; r0 += slab) {
        const uint64_t nr = std::min(slab, n - r0);
        e = cudaMemcpy(d_raw, raw + r0 * dim, (size_t)nr * dim * 4, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            gb::make_elements_kernel<<<(unsigned)std::min<uint64_t>(nr, (uint64_t)sms * 32), 32, (size_t)dim * 4>>>(
                d_raw, nr, dim, element_kind, d_out);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess)
            e = cudaMemcpy(o + 8 + (size_t)r0 * dim * esz, d_out, (size_t)nr * dim * esz, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(GRANNE_B200_ERR_CUDA, cudaGetErrorString(e));
    }
    cudaFree(d_raw);
    cudaFree(d_out);
    return rc;
}

// Vector::from per row (angular.rs:55-61 / angular_int.rs:28-45), device to device: d_raw = n x dim f32 rows in HBM,
// d_out = n x dim elements (f32 or i8), both on `device`; runs on `cuda_stream` (asynchronous).
int granne_b200_elements_from_raw_device(int element_kind, const float* d_raw, uint64_t n, uint32_t dim, int device,
                                         void* d_out, void* cuda_stream) {
    if (element_kind != GRANNE_B200_ANGULAR && element_kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements_from_raw supports angular and angular_int");
    if (dim == 0 || dim > 12000) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unsupported dimension");
    if (n == 0) return GRANNE_B200_OK;
    if (!d_raw || !d_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    int sms = 0;
    size_t optin = 0;
    int rc = check_device(device, &sms, &optin);
    if (rc) return rc;
    GB_DEVICE(device);
    gb::make_elements_kernel<<<(unsigned)std::min<uint64_t>(n, (uint64_t)sms * 32), 32, (size_t)dim * 4,
                               static_cast<cudaStream_t>(cuda_stream)>>>(d_raw, n, dim, element_kind, d_out);
    GB_CUDA(cudaGetLastError());
    return GRANNE_B200_OK;
}

// ---- compute_distance (py/src/lib.rs:71-89) -----------------------------------------------------------------------
int granne_b200_compute_distances(int element_kind, const float* a, const float* b, uint64_t n, uint32_t dim, int device,
                                  float* out) {
    if (n == 0) return GRANNE_B200_OK;
    if (!a || !b || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (n > 0xFFFFFFFFull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many pairs for one call");
    try {
        // the b vectors become an element container (Vector::from per row, on the device) ...
        size_t need = 0;
        int rc = granne_b200_elements_from_raw(element_kind, nullptr, n, dim, device, nullptr, 0, &need);
        if (rc) return rc;
        std::vector<uint8_t> elements(need);
        if ((rc = granne_b200_elements_from_raw(element_kind, b, n, dim, device, elements.data(), need, &need))) return rc;
        // ... behind an index without layers
        std::vector<uint8_t> image;
        std::string err;
        if (!gb::encode_index({}, &image, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        Handle* raw_h = nullptr;
        if ((rc = open_impl(image.data(), image.size(), element_kind, elements.data(), elements.size(), nullptr, 0, device,
                            &raw_h)))
            return rc;
        std::unique_ptr<Handle, void (*)(Handle*)> h(raw_h, [](Handle* p) { granne_b200_close(p); });
        const LaunchPlan plan = make_plan(h.get(), 1);
        float *d_a = nullptr, *d_out = nullptr;
        int* d_err = nullptr;
        struct Free {
            float **a, **o;
            int** e;
            ~Free() {
                cudaFree(*a);
                cudaFree(*o);
                cudaFree(*e);
            }
        } guard{&d_a, &d_out, &d_err};
        GB_CUDA(cudaMalloc(&d_a, (size_t)n * dim * 4));
        GB_CUDA(cudaMalloc(&d_out, (size_t)n * 4));
        GB_CUDA(cudaMalloc(&d_err, 4));
        GB_CUDA(cudaMemcpy(d_a, a, (size_t)n * dim * 4, cudaMemcpyHostToDevice));
        GB_CUDA(cudaMemset(d_err, 0, 4));
        PairLaunch L{h.get(), {}, plan.base_smem + gb::link_scratch_bytes(8, 32) + 64, 0, nullptr};
        L.a.queries = d_a;
        L.a.n = (uint32_t)n;
        L.a.out = d_out;
        L.a.error_flag = d_err;
        L.a.stg_rows = plan.stg_rows;
        L.a.stg_row_bytes = plan.stg_row_bytes;
        L.a.tile_rows = plan.tile_rows;
        L.grid = (unsigned)std::min<uint64_t>(n, (uint64_t)h->num_sms * 16);
        if ((rc = DistDispatch::call(h->dev, L))) return rc;
        GB_CUDA(cudaDeviceSynchronize());
        int herr = 0;
        GB_CUDA(cudaMemcpy(&herr, d_err, 4, cudaMemcpyDeviceToHost));
        GB_CUDA(cudaMemcpy(out, d_out, (size_t)n * 4, cudaMemcpyDeviceToHost));
        return error_from_bits(herr);
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_reencode_index(const void* index_bytes, size_t index_len, void* out, size_t cap, size_t* out_len) {
    if (!index_bytes || !out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        std::vector<gb::LayerView> views;
        for (const gb::HostLayer& L : graph.layers) views.push_back({L.rows.data(), L.num_nodes, L.width});
        std::vector<uint8_t> image;
        if (!gb::encode_index(views, &image, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        *out_len = image.size();
        if (!out) return GRANNE_B200_OK;
        if (cap < image.size()) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
        std::memcpy(out, image.data(), image.size());
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

// ---- reorder (src/index/reorder.rs) -----------------------------------------------------------------------------------

// Granne::compute_order (reorder.rs:126-174).  The trail of element idx (find_entrypoint_trail, reorder.rs:180-207) is
// one max_search = 1 search_for_neighbors from node 0 in each of the first min(8, layer) layers: here, per trail layer,
// ONE batch of the search kernel over a single-layer view of the staged graph, queries given by element id.
int granne_b200_compute_order(granne_b200_index* h, uint64_t* order_out, uint64_t cap) {
    if (!h || !order_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    const uint64_t n = h->index_len;
    if (cap < n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "order buffer shorter than Index::len");
    const int nl = h->dev.num_layers;
    if (nl == 0) return GRANNE_B200_OK;
    try {
        GB_DEVICE(h->device);
        std::vector<uint64_t> layer_lens(nl);
        for (int l = 0; l < nl; ++l) layer_lens[l] = h->dev.layer_len[l];
        const size_t trail_layers = std::min<size_t>(gb::kTrailLayers, (size_t)nl - 1);
        std::vector<std::vector<uint32_t>> eps(trail_layers);
        Workspace* w = nullptr;
        int rc = ws_acquire(h, &w);
        if (rc) return rc;
        const size_t batch = (size_t)std::min<uint64_t>(std::max<uint64_t>(n, 1), 1u << 20);
        uint32_t *d_q = nullptr, *d_ids = nullptr, *d_cnt = nullptr;
        float* d_d = nullptr;
        // the trail searches run over a PRIVATE single-layer view of the staged index: the shared handle is never
        // modified, so concurrent searches on it stay correct
        gb::DeviceIndex view = h->dev;
        struct Cleanup {
            Handle* h;
            Workspace* w;
            uint32_t **q, **ids, **cnt;
            float** d;
            ~Cleanup() {
                cudaFree(*q);
                cudaFree(*ids);
                cudaFree(*cnt);
                cudaFree(*d);
                ws_release(h, w);
            }
        } cleanup{h, w, &d_q, &d_ids, &d_cnt, &d_d};
        GB_CUDA(cudaMalloc(&d_q, batch * 4));
        GB_CUDA(cudaMalloc(&d_ids, batch * 4));
        GB_CUDA(cudaMalloc(&d_cnt, batch * 4));
        GB_CUDA(cudaMalloc(&d_d, batch * 4));
        for (size_t j = 0; j < trail_layers; ++j) {
            eps[j].resize(n - layer_lens[j]);
            view.num_layers = 1;
            view.layer_rows[0] = h->dev.layer_rows[j];
            view.layer_width[0] = h->dev.layer_width[j];
            view.layer_len[0] = h->dev.layer_len[j];
            for (uint64_t base = layer_lens[j]; base < n; base += batch) {
                const uint64_t bsz = std::min<uint64_t>(batch, n - base);
                gb::iota_kernel<<<(unsigned)((bsz + 255) / 256), 256, 0, w->stream>>>(d_q, (uint32_t)bsz, (uint32_t)base, 1);
                h->launches++;
                rc = enqueue_search(h, w, d_q, bsz, gb::kQueryById, 1, 1, d_ids, d_d, d_cnt, nullptr, w->stream, true,
                                    nullptr, &view);
                if (rc) return rc;
                GB_CUDA(cudaMemcpyAsync(eps[j].data() + (base - layer_lens[j]), d_ids, bsz * 4, cudaMemcpyDeviceToHost,
                                        w->stream));
                int herr[4] = {0, 0, 0, 0};
                GB_CUDA(cudaMemcpyAsync(herr, w->d_error, sizeof(herr), cudaMemcpyDeviceToHost, w->stream));
                GB_CUDA(cudaStreamSynchronize(w->stream));
                if ((rc = error_from_bits(herr[0]))) return rc;
            }
        }
        gb::order_from_trails(layer_lens, eps, order_out);
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_order_from_trails(const uint64_t* layer_lens, uint32_t num_layers, const uint32_t* trails, uint64_t n,
                                  uint64_t* order_out) {
    if (!layer_lens || !trails || !order_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        std::vector<uint64_t> lens(layer_lens, layer_lens + num_layers);
        if (num_layers == 0 || lens.back() != n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "n must equal the last layer's length");
        for (uint32_t l = 1; l < num_layers; ++l)
            if (lens[l] < lens[l - 1]) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "layer lengths must not decrease");
        const size_t trail_layers = std::min<size_t>(gb::kTrailLayers, (size_t)num_layers - 1);
        std::vector<std::vector<uint32_t>> eps(trail_layers);
        for (size_t j = 0; j < trail_layers; ++j) {
            eps[j].resize(n - lens[j]);
            for (uint64_t idx = lens[j]; idx < n; ++idx) {
                const uint32_t v = trails[idx * gb::kTrailLayers + j];
                if (v >= lens[j]) return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "trail entry outside its layer");
                eps[j][idx - lens[j]] = v;
            }
        }
        gb::order_from_trails(lens, eps, order_out);
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_order_by_keys(const void* index_bytes, size_t index_len, const uint64_t* keys, uint64_t num_keys,
                              uint32_t key_width, uint64_t* order_out) {
    if (!index_bytes || !keys || !order_out || key_width == 0)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        std::vector<uint64_t> layer_lens;
        for (const gb::HostLayer& L : graph.layers) layer_lens.push_back(L.num_nodes);
        if (num_keys != (layer_lens.empty() ? 0 : layer_lens.back()))  // assert_eq!(self.len(), keys.len())
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "number of keys must equal Index::len");
        gb::order_by_keys(layer_lens, keys, key_width, order_out);
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_embedding_reorder_keys(const void* elements_bytes, size_t elements_len, const void* embeddings_bytes,
                                       size_t embeddings_len, uint64_t* keys_out) {
    if (!elements_bytes || !embeddings_bytes || !keys_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        std::string err;
        if (!gb::embedding_reorder_keys(static_cast<const uint8_t*>(elements_bytes), elements_len,
                                        static_cast<const uint8_t*>(embeddings_bytes), embeddings_len, keys_out, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_apply_order(const void* index_bytes, size_t index_len, int element_kind, const void* elements_bytes,
                            size_t elements_len, const uint64_t* order, uint64_t n, void* out_index, size_t index_cap,
                            size_t* index_out_len, void* out_elements, size_t elements_cap, size_t* elements_out_len) {
    if (!index_bytes || !elements_bytes || !order || !index_out_len || !elements_out_len)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    try {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        std::vector<uint8_t> image, elements;
        if (!gb::reorder_graph(graph, order, n, &image, &err)) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, err);
        const uint8_t* eb = static_cast<const uint8_t*>(elements_bytes);
        bool ok;
        switch (element_kind) {
            case GRANNE_B200_ANGULAR: ok = gb::permute_dense(eb, elements_len, 4, order, n, &elements, &err); break;
            case GRANNE_B200_ANGULAR_INT: ok = gb::permute_dense(eb, elements_len, 1, order, n, &elements, &err); break;
            case GRANNE_B200_EMBEDDINGS: ok = gb::permute_sum_elements(eb, elements_len, order, n, &elements, &err); break;
            default: return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unknown element kind");
        }
        if (!ok) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, err);
        *index_out_len = image.size();
        *elements_out_len = elements.size();
        if (!out_index && !out_elements) return GRANNE_B200_OK;
        if (!out_index || !out_elements || index_cap < image.size() || elements_cap < elements.size())
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
        std::memcpy(out_index, image.data(), image.size());
        std::memcpy(out_elements, elements.data(), elements.size());
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

int granne_b200_merge_topk_device(int device, const uint32_t* d_part_ids, const float* d_part_dists,
                                  const uint64_t* part_base, size_t num_parts, size_t nq, uint32_t k,
                                  uint64_t* d_out_ids, float* d_out_dists, void* cuda_stream) {
    if (!d_part_ids || !d_part_dists || !part_base || !d_out_ids || !d_out_dists)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (num_parts == 0 || num_parts > 64) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "num_parts must be 1..64");
    if (nq == 0 || k == 0) return GRANNE_B200_OK;
    GB_DEVICE(device);
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    unsigned long long* d_base = nullptr;
    GB_CUDA(cudaMallocAsync(&d_base, num_parts * 8, stream));
    GB_CUDA(cudaMemcpyAsync(d_base, part_base, num_parts * 8, cudaMemcpyHostToDevice, stream));
    const unsigned block = 128, grid = (unsigned)((nq + block - 1) / block);
    gb::merge_topk_kernel<<<grid, block, 0, stream>>>(d_part_ids, d_part_dists, d_base, (uint32_t)num_parts, nq, k,
                                                      reinterpret_cast<unsigned long long*>(d_out_ids), d_out_dists);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaFreeAsync(d_base, stream));
    return GRANNE_B200_OK;
}

// ---- several GPUs behind one handle ------------------------------------------------------------------------------------
}  // extern "C"

struct granne_b200_multi {
    int mode = GRANNE_B200_MODE_REPLICATED;
    std::vector<granne_b200_index*> parts;  // one single-device handle per device (replicated) or per shard
    std::vector<uint64_t> base;              // global id of each part's element 0
    uint64_t total_len = 0;
    uint32_t dim = 0;
    int kind = 0;
};

namespace {

// runs fn(i) for i in [0, n) on n threads (one per device: every call blocks on its own stream) and returns the
// first non-zero status together with its message
template <class F>
int for_each_part(size_t n, F&& fn) {
    std::vector<int> rc(n, 0);
    std::vector<std::string> msg(n);
    std::vector<std::thread> th;
    for (size_t i = 1; i < n; ++i)
        th.emplace_back([&, i] {
            rc[i] = fn(i);
            if (rc[i]) msg[i] = g_last_error;  // thread_local: carry it to the caller's thread
        });
    rc[0] = fn(0);
    if (rc[0]) msg[0] = g_last_error;
    for (auto& t : th) t.join();
    for (size_t i = 0; i < n; ++i)
        if (rc[i]) return fail(rc[i], msg[i]);
    return GRANNE_B200_OK;
}

}  // namespace

extern "C" {

int granne_b200_multi_open(int mode, const int* devices, size_t num_devices, int element_kind,
                           const void* const* index_bytes, const size_t* index_len,
                           const void* const* elements_bytes, const size_t* elements_len, size_t num_shards,
                           const void* embeddings_bytes, size_t embeddings_len, granne_b200_multi** out) {
    if (!out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "out handle pointer is null");
    *out = nullptr;
    if (mode != GRANNE_B200_MODE_REPLICATED && mode != GRANNE_B200_MODE_RANGE_PARTITIONED)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unknown multi-GPU mode");
    if (!devices || num_devices == 0 || num_devices > 64)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "device list must name 1..64 devices");
    if (!index_bytes || !index_len || !elements_bytes || !elements_len || num_shards == 0)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (mode == GRANNE_B200_MODE_REPLICATED && num_shards != 1)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "replicated mode takes exactly one index image");
    try {
        std::unique_ptr<granne_b200_multi> m(new granne_b200_multi());
        m->mode = mode;
        m->kind = element_kind;
        const size_t n = mode == GRANNE_B200_MODE_REPLICATED ? num_devices : num_shards;
        m->parts.assign(n, nullptr);
        m->base.assign(n, 0);
        int rc = for_each_part(n, [&](size_t i) {
            const size_t s = mode == GRANNE_B200_MODE_REPLICATED ? 0 : i;
            return granne_b200_open(index_bytes[s], index_len[s], element_kind, elements_bytes[s], elements_len[s],
                                    embeddings_bytes, embeddings_len, devices[i % num_devices], &m->parts[i]);
        });
        if (rc) {
            const std::string keep = g_last_error;
            for (auto* p : m->parts) granne_b200_close(p);
            return fail(rc, keep);
        }
        m->dim = m->parts[0]->dev.dim;
        uint64_t acc = 0;
        for (size_t i = 0; i < n; ++i) {
            if (m->parts[i]->dev.dim != m->dim) {
                for (auto* p : m->parts) granne_b200_close(p);
                return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "shards have different dimensions");
            }
            if (mode == GRANNE_B200_MODE_RANGE_PARTITIONED) {
                m->base[i] = acc;
                acc += m->parts[i]->dev.num_elements;  // ids continue across shards over the ELEMENT ranges
            }
        }
        m->total_len = 0;
        if (mode == GRANNE_B200_MODE_REPLICATED)
            m->total_len = m->parts[0]->index_len;
        else
            for (auto* p : m->parts) m->total_len += p->index_len;
        *out = m.release();
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

void granne_b200_multi_close(granne_b200_multi* m) {
    if (!m) return;
    for (auto* p : m->parts) granne_b200_close(p);
    delete m;
}

uint64_t granne_b200_multi_len(const granne_b200_multi* m) { return m ? m->total_len : 0; }
size_t granne_b200_multi_num_parts(const granne_b200_multi* m) { return m ? m->parts.size() : 0; }
uint64_t granne_b200_multi_shard_base(const granne_b200_multi* m, size_t s) {
    return (m && s < m->base.size()) ? m->base[s] : 0;
}

int granne_b200_multi_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                   uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                   uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    if (nq == 0) return GRANNE_B200_OK;
    if (!queries || (num_neighbors && (!out_ids || !out_dists)))
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null buffer");
    try {
        const size_t n = m->parts.size(), k = num_neighbors;
        const bool i8q = m->kind == GRANNE_B200_ANGULAR_INT && query_format == GRANNE_B200_QUERY_ELEMENT;
        const size_t qrow = (size_t)m->dim * (i8q ? 1 : 4);
        const uint8_t* q = static_cast<const uint8_t*>(queries);
        if (m->mode == GRANNE_B200_MODE_REPLICATED) {
            // contiguous, balanced query slices (the first nq % n devices take one more)
            std::vector<uint32_t> ids(nq * k);
            std::vector<uint32_t> cnt(nq);
            const size_t per = nq / n, extra = nq % n;
            int rc = for_each_part(n, [&](size_t i) {
                const size_t b = i * per + std::min(i, extra), cntq = per + (i < extra ? 1 : 0);
                if (cntq == 0) return (int)GRANNE_B200_OK;
                return granne_b200_search_batch(m->parts[i], q + b * qrow, cntq, query_format, max_search, num_neighbors,
                                                ids.data() + b * k, out_dists + b * k, cnt.data() + b, nullptr);
            });
            if (rc) return rc;
            for (size_t i = 0; i < nq * k; ++i) out_ids[i] = ids[i] == gb::kUnusedId ? ~0ull : (uint64_t)ids[i];
            if (out_counts) std::memcpy(out_counts, cnt.data(), nq * 4);
            return GRANNE_B200_OK;
        }
        // range-partitioned: every shard searches all queries; k-way merge by (distance, global id) on the host
        std::vector<uint32_t> ids(n * nq * k);
        std::vector<float> ds(n * nq * k);
        int rc = for_each_part(n, [&](size_t i) {
            return granne_b200_search_batch(m->parts[i], q, nq, query_format, max_search, num_neighbors,
                                            ids.data() + i * nq * k, ds.data() + i * nq * k, nullptr, nullptr);
        });
        if (rc) return rc;
        std::vector<size_t> cur(n);
        for (size_t qi = 0; qi < nq; ++qi) {
            std::fill(cur.begin(), cur.end(), 0);
            uint32_t found = 0;
            for (size_t r = 0; r < k; ++r) {
                int best = -1;
                float bd = 0.0f;
                uint64_t bid = 0;
                for (size_t p = 0; p < n; ++p) {
                    if (cur[p] >= k) continue;
                    const size_t o = (p * nq + qi) * k + cur[p];
                    if (ids[o] == gb::kUnusedId) continue;  // each tile is sorted and padded at the end
                    const uint64_t gid = m->base[p] + ids[o];
                    if (best < 0 || ds[o] < bd || (ds[o] == bd && gid < bid)) {
                        best = (int)p;
                        bd = ds[o];
                        bid = gid;
                    }
                }
                if (best < 0) {
                    out_ids[qi * k + r] = ~0ull;
                    out_dists[qi * k + r] = std::numeric_limits<float>::infinity();
                } else {
                    out_ids[qi * k + r] = bid;
                    out_dists[qi * k + r] = bd;
                    cur[best] += 1;
                    found += 1;
                }
            }
            if (out_counts) out_counts[qi] = found;
        }
        return GRANNE_B200_OK;
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

}  // extern "C"
