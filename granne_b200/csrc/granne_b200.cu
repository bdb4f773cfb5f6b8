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
#include <type_traits>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "formats.hpp"
#include "reorder.hpp"
#include "build_kernels.cuh"
#include "search_kernels.cuh"
#include "exact_kernels.cuh"
#include "rerank_kernels.cuh"
#include "diverse_kernels.cuh"
#include "within_kernels.cuh"
#include "ids_kernels.cuh"
#include "range_kernels.cuh"

namespace gb = granne_b200;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

// The exception boundary of the C ABI: every entry point that can allocate or throw runs its body through this, so
// that no C++ exception (std::bad_alloc from a container, ...) escapes into a C, C++ or Rust caller.
template <class F>
int guarded(F&& body) {
    try {
        return body();
    } catch (const std::exception& e) {
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, std::string("exception: ") + e.what());
    }
}

#define GB_CUDA(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess) {                                                                        \
            return fail(GRANNE_B200_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));      \
        }                                                                                               \
    } while (0)

// Launches Kern over (grid, block) with `smem` bytes of dynamic shared memory on `stream`, adds it to `launches` (null
// for a call without a handle) and returns the launch's error, so that a failed launch is reported by the call that made
// it rather than left behind as the thread's last error.
template <auto Kern, class... Args>
int launch(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, std::atomic<uint64_t>* launches, Args&&... args) {
    Kern<<<grid, block, smem, stream>>>(std::forward<Args>(args)...);
    if (launches) ++*launches;
    GB_CUDA(cudaGetLastError());
    return GRANNE_B200_OK;
}

// Every entry point runs on its handle's device and leaves the caller's current device as it found it (a host
// application — e.g. one torch process per GPU — must not see its default device change under it).  A guard is
// declared before anything that owns device memory, so that the memory is also freed on that device.
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    DeviceGuard() = default;
    explicit DeviceGuard(int device) : err(enter(device)) {}
    cudaError_t enter(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        return cudaSetDevice(device);
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

// The owners of the host layer's CUDA resources; nothing else frees them.
struct DeviceFree {
    void operator()(void* p) const { cudaFree(p); }
};
struct HostFree {
    void operator()(void* p) const { cudaFreeHost(p); }
};
struct StreamDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;

// `cap` elements of T in device memory (PINNED: pinned host memory).
template <class T, bool PINNED = false>
struct Buffer {
    std::unique_ptr<T, std::conditional_t<PINNED, HostFree, DeviceFree>> p;
    size_t cap = 0;
    T* get() const { return p.get(); }
    // Makes room for `count` elements.  Reallocates only when `count` exceeds the capacity; the old buffer may still
    // be in use by work queued on `stream`, so the stream is synchronised before it is freed.
    int grow(size_t count, cudaStream_t stream) {
        if (count <= cap) return GRANNE_B200_OK;
        if (p) GB_CUDA(cudaStreamSynchronize(stream));
        p.reset();
        cap = 0;
        void* q = nullptr;
        if constexpr (PINNED)
            GB_CUDA(cudaMallocHost(&q, count * sizeof(T)));
        else
            GB_CUDA(cudaMalloc(&q, count * sizeof(T)));
        p.reset(static_cast<T*>(q));
        cap = count;
        return GRANNE_B200_OK;
    }
};
template <class T>
using Pinned = Buffer<T, true>;

constexpr size_t kSearchCounterBytes = 32, kHostCallBytes = 64;  // the start-of-call words (Workspace::d_counters)

// Per-call scratch: device copies of queries/results, status words, stream.  Pooled per handle so that several host
// threads can search concurrently (the reference's `search` is `&self` and reentrant).
struct Workspace {
    Stream stream;  // declared first: destroyed after the buffers
    Buffer<uint8_t> d_queries;
    Buffer<uint32_t> d_ids;  // one block: ids | dists | counts, so that one copy brings a whole result back
    float* d_dists = nullptr;    // inside d_ids, packed for the current call's nq x k
    uint32_t* d_counts = nullptr;
    Buffer<unsigned long long> d_stats;
    Buffer<int> d_status;  // nq ints
    // one 64-byte block: [0..2] work counters of the three passes, [3] fast pass flagged something, [4] retry pass
    // flagged something, [5] done counter (fused gather), [6] work counter of the re-rank kernel, [7] work counter of
    // the diverse selection; d_error = words [8..11].  A call zeroes its words with one memset before its kernels: a
    // host call the whole block, since it reports the errors of its own kernels only (kHostCallBytes, host_batch); a
    // device call or a builder batch the counters when it searches, leaving the error word sticky
    // (kSearchCounterBytes).
    Buffer<unsigned int> d_counters;
    int* d_error = nullptr;              // [0]=sticky error bits of this call (inside the counters block)
    Buffer<unsigned long long> d_retried;  // cumulative: queries that needed more than the fast pass
    Pinned<unsigned long long> h_retried;  // pinned mirror (copied at the end of every call, read without a sync)
    unsigned long long seen_retried = 0, seen_total = 0, total_queries = 0;
    Pinned<uint8_t> h_pinned;            // staging for host<->device copies
    // slow path
    Buffer<unsigned long long> d_slow_list;
    Buffer<uint32_t> d_slow_vis;
    // fast pass: per-CTA visited tables in global memory
    Buffer<uint32_t> d_vis;
    // retry pass: fewer CTAs, larger tables
    Buffer<uint32_t> d_vis_retry;
    // exact search: prepared queries of a chunk, their dy (i8), a slab's distances, the running top-k lists, and for
    // EMBEDDINGS a window of materialised rows (and a dense copy of the table when its staged rows are padded)
    Buffer<uint8_t> d_exact_q;
    Buffer<int> d_exact_qnorm;
    Buffer<float> d_exact_dists;
    Buffer<unsigned long long> d_exact_lists;
    Buffer<float> d_exact_rows;
    Buffer<float> d_exact_table;
    // exact filtered search: a list of admitted ids | the chunk's filters | the counts [ids, filters, list cursor];
    // the queries' prepare statuses
    Buffer<uint32_t> d_exact_ids;
    Buffer<int> d_exact_qstat;
    // two-stage and diverse search: stage 1's candidates, one block ids | dists | counts for the current call's nq x C
    Buffer<uint32_t> d_rerank;
    // exact search within lists: a chunk's running lists | segment prefix; its locks | query flags
    Buffer<unsigned long long> d_within;
    Buffer<int> d_within_flags;
    // queries by element id: the elements' rows, the bad-id flags, and (QUERY_ID_EXCLUDING) the k + 1 column block
    // ids | dists | counts
    Buffer<uint8_t> d_id_rows;
    Buffer<int> d_id_bad;
    Buffer<uint32_t> d_id_res;
    // exact range fill: a chunk's per-query cursors into the caller's segments
    Buffer<unsigned long long> d_range_cursor;
};

// The owners of the arrays a DeviceIndex points to, one slot per pointer: the memory and the bytes allocated for it.
// A copy shares the memory (get_index snapshots), which is freed once no slot holds it.
struct Staged {
    struct Slot {
        std::shared_ptr<void> mem;
        uint64_t bytes = 0;
    };
    Slot vectors, sum_offsets, sum_terms, layer_rows[gb::kMaxLayers];
};

}  // namespace

struct granne_b200_index {
    int device = 0;
    int num_sms = 0;
    size_t smem_optin = 0;
    gb::DeviceIndex dev{};
    Staged dev_mem;
    // the container that re-ranks the candidates of an angular_int index: angular f32 rows
    // (granne_b200_set_rerank_elements*) or a SumEmbeddings container (granne_b200_set_rerank_embeddings);
    // vectors == nullptr until one is attached
    gb::DeviceIndex rerank{};
    Staged rerank_mem;
    uint64_t index_len = 0;  // Index::len
    std::vector<uint32_t> layer_max_degree;
    std::atomic<uint64_t> launches{0};
    std::atomic<int> sticky_error{0};
    std::mutex pool_mu;
    mutable std::mutex rerank_mu;  // serialises the re-rank attaches (granne_b200_set_rerank_*) and device_bytes
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

// Device memory for staged data (elements, layers): `count` T, at least 16 bytes so that every buffer has an address
// of its own.
template <class T>
int dev_alloc(Buffer<T>* mem, size_t count) {
    return mem->grow(std::max<size_t>(count, 16 / sizeof(T)), nullptr);
}

// Puts the filled buffer `mem` into `slot`, replacing whatever the slot held, and returns its address.
template <class T>
T* stage(Staged::Slot* slot, Buffer<T> mem) {
    T* p = mem.get();
    slot->bytes = mem.cap * sizeof(T);
    slot->mem = std::shared_ptr<void>(std::move(mem.p));
    return p;
}

// Stages layer l of h's index: `num_nodes` rows of `width` u32 from host memory.
int stage_layer(Handle* h, int l, const uint32_t* rows, uint64_t num_nodes, uint32_t width) {
    const size_t n = (size_t)num_nodes * width;
    Buffer<uint32_t> mem;
    int rc = dev_alloc(&mem, n);
    if (rc) return rc;
    if (n) GB_CUDA(cudaMemcpy(mem.get(), rows, n * 4, cudaMemcpyHostToDevice));
    h->dev.layer_rows[l] = stage(&h->dev_mem.layer_rows[l], std::move(mem));
    h->dev.layer_width[l] = width;
    h->dev.layer_len[l] = num_nodes;
    return GRANNE_B200_OK;
}

// The type tag DistDispatch passes: Engine<Dist>::type is the engine.
template <class Dist>
struct Engine {
    using type = Dist;
};

// Which distance engine serves an index: returns f(Engine<Dist>{}) for the engine of `d`'s element kind and chunk
// count (d.full = dim / 32) — DistF32<full> for the chunk counts it is compiled for, DistF32Generic for every other
// f32 width.  This is the only place that decides it; the row layout (stage_dense) and the tiles (engine_tiles)
// follow from the engine it picks (fixed_f32_chunks).
struct DistDispatch {
    template <class F>
    static int call(const gb::DeviceIndex& d, F&& f) {
        switch (d.kind) {
            case gb::kAngularI8: return f(Engine<gb::DistI8>{});
            case gb::kSumEmbeddings: return f(Engine<gb::DistSum>{});
            default: break;
        }
        switch (d.full) {
            case 0: return f(Engine<gb::DistF32<0>>{});
            case 1: return f(Engine<gb::DistF32<1>>{});
            case 2: return f(Engine<gb::DistF32<2>>{});
            case 3: return f(Engine<gb::DistF32<3>>{});
            case 4: return f(Engine<gb::DistF32<4>>{});
            case 6: return f(Engine<gb::DistF32<6>>{});
            case 8: return f(Engine<gb::DistF32<8>>{});
            default: return f(Engine<gb::DistF32Generic>{});
        }
    }
};

// FULL of the DistF32<FULL> engine that serves `d`, or -1 when an engine for any width does (DistF32Generic, DistI8,
// DistSum).
template <class Dist>
constexpr int kFixedChunks = -1;
template <int FULL>
constexpr int kFixedChunks<gb::DistF32<FULL>> = FULL;
int fixed_f32_chunks(const gb::DeviceIndex& d) {
    return DistDispatch::call(d, [](auto e) { return kFixedChunks<typename decltype(e)::type>; });
}

// Writes `nrows` dense rows of d's kind and width from `src` (host memory, or device memory if `device_src`) to the
// staged rows at `dst`: in 64 MB slabs through a temporary device buffer, re-laid out on the device by
// pad_rows_i8_kernel / permute_rows_f32_kernel.
int upload_rows(Handle* h, const gb::DeviceIndex& d, const uint8_t* src, uint64_t nrows, bool device_src,
                uint8_t* dst) {
    const bool i8 = d.kind == gb::kAngularI8;
    const size_t esz = i8 ? 1 : 4, src_row = (size_t)d.dim * esz;
    const uint64_t slab = std::max<uint64_t>(1, (64ull << 20) / src_row);
    Buffer<uint8_t> tmp;
    int rc;
    if (!device_src && (rc = tmp.grow((size_t)std::min(slab, std::max<uint64_t>(nrows, 1)) * src_row, nullptr)))
        return rc;
    for (uint64_t r0 = 0; r0 < nrows; r0 += slab) {
        const uint64_t nr = std::min(slab, nrows - r0);
        const uint8_t* from = src + r0 * src_row;
        if (!device_src) {
            GB_CUDA(cudaMemcpy(tmp.get(), from, (size_t)nr * src_row, cudaMemcpyHostToDevice));
            from = tmp.get();
        }
        uint8_t* to = dst + r0 * d.row_stride * esz;
        rc = i8 ? launch<gb::pad_rows_i8_kernel>(h->num_sms * 8, 256, 0, nullptr, &h->launches,
                                                 reinterpret_cast<const int8_t*>(from), reinterpret_cast<int8_t*>(to),
                                                 nr, d.dim, d.row_stride)
                : launch<gb::permute_rows_f32_kernel>(h->num_sms * 8, 256, 0, nullptr, &h->launches,
                                                      reinterpret_cast<const float*>(from), reinterpret_cast<float*>(to),
                                                      nr, d.dim, d.full, d.vec_group, d.row_stride);
        if (rc) return rc;
    }
    GB_CUDA(cudaDeviceSynchronize());
    return GRANNE_B200_OK;
}

// Stages `nrows` dense rows of d's kind (host memory, or device memory if `device_src`) as d's vectors, owned by
// `mem`: the handle's own container (h->dev) or the re-rank rows (h->rerank).
int stage_dense(Handle* h, gb::DeviceIndex& d, Staged& mem, const uint8_t* rows, uint64_t nrows, uint32_t dim,
                bool device_src = false) {
    d.dim = dim;
    d.full = dim / 32;
    d.tail = dim % 32;
    d.num_vectors = nrows;
    const bool i8 = d.kind == gb::kAngularI8;
    if (i8) {
        d.vec_group = 1;
        d.row_stride = (dim + 31u) & ~31u;  // rows start on 32-byte sector boundaries (DistI8)
    } else {
        const uint32_t full = d.full;
        // DistF32<full> reads rows lane-permuted in groups of V = DistF32<full>::V chunks; the other engines read the
        // natural layout (V = 1 permutes nothing)
        d.vec_group = fixed_f32_chunks(d) > 0 ? (full % 4 == 0 ? 4 : (full % 2 == 0 ? 2 : 1)) : 1;
        d.row_stride = (dim + 3u) & ~3u;
    }
    Buffer<uint8_t> dst;
    int rc;
    if ((rc = dev_alloc(&dst, (size_t)nrows * d.row_stride * (i8 ? 1 : 4)))) return rc;
    if ((rc = upload_rows(h, d, rows, nrows, device_src, dst.get()))) return rc;
    d.vectors = stage(&mem.vectors, std::move(dst));
    return GRANNE_B200_OK;
}

// SumEmbeddings::from_bytes (embeddings/mod.rs:56-61) on the host: the embedding table and the element term lists,
// every term id checked against the table.
int parse_sum_container(const uint8_t* el, size_t el_len, const uint8_t* emb, size_t emb_len, gb::DenseView* ev,
                        gb::SumElements* se) {
    std::string err;
    if (!gb::parse_dense(emb, emb_len, 4, ev, &err)) return fail(GRANNE_B200_ERR_FORMAT, "embeddings: " + err);
    if (!gb::parse_sum_elements(el, el_len, se, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
    for (uint32_t t : se->terms)
        if (t >= ev->num) return fail(GRANNE_B200_ERR_FORMAT, "element refers to a missing embedding id");
    if (ev->dim > 4096) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "embeddings wider than 4096 are unsupported");
    return GRANNE_B200_OK;
}

// Stages a parsed SumEmbeddings container (parse_sum_container) as d's embedding table, element offsets and term ids,
// owned by `mem`: the handle's own container (h->dev) or its re-rank container (h->rerank).
int stage_sum(Handle* h, gb::DeviceIndex& d, Staged& mem, const gb::DenseView& ev, const gb::SumElements& se) {
    d.kind = gb::kSumEmbeddings;
    int rc = stage_dense(h, d, mem, ev.data, ev.num, (uint32_t)ev.dim);
    if (rc) return rc;
    d.num_elements = se.offsets.size() - 1;
    Buffer<unsigned long long> doff;
    Buffer<uint32_t> dterms;
    if ((rc = dev_alloc(&doff, se.offsets.size())) || (rc = dev_alloc(&dterms, se.terms.size()))) return rc;
    GB_CUDA(cudaMemcpy(doff.get(), se.offsets.data(), se.offsets.size() * 8, cudaMemcpyHostToDevice));
    if (!se.terms.empty())
        GB_CUDA(cudaMemcpy(dterms.get(), se.terms.data(), se.terms.size() * 4, cudaMemcpyHostToDevice));
    d.sum_offsets = stage(&mem.sum_offsets, std::move(doff));
    d.sum_terms = stage(&mem.sum_terms, std::move(dterms));
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
        gb::SumElements se;
        if ((rc = parse_sum_container(el, el_len, emb, emb_len, &ev, &se))) return rc;
        if ((rc = stage_sum(h, d, h->dev_mem, ev, se))) return rc;
    } else {
        gb::DenseView dv;
        const bool i8 = kind == GRANNE_B200_ANGULAR_INT;
        if (!gb::parse_dense(el, el_len, i8 ? 1 : 4, &dv, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        if (dv.dim > 16384) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "vectors wider than 16384 are unsupported");
        rc = stage_dense(h, d, h->dev_mem, dv.data, dv.num, (uint32_t)dv.dim);
        if (rc) return rc;
        d.num_elements = dv.num;
    }
    return GRANNE_B200_OK;
}

// ---- compute_embeddings_and_save_to_disk (embeddings/parsing.rs:102-152) -------------------------------------------
// The rows are made in windows of elements, so that the device holds the embedding table plus a constant window
// (the reference makes them in 100 chunks for the same reason): at most kEmbWindowBytes of raw f32 rows and
// kEmbWindowMaxRows rows, and at most kEmbWindowTerms term ids unless a single element holds more.
constexpr uint64_t kEmbWindowBytes = 64ull << 20;
constexpr uint64_t kEmbWindowMaxRows = 1ull << 20;
constexpr uint64_t kEmbWindowTerms = 1ull << 24;

struct EmbeddingsInput {
    gb::DenseView table;
    gb::SumElements el;
    uint64_t n = 0;
    uint32_t dim = 0;  // width of the output rows; 0 when there is no row to write (n == 0, or a table without rows)
};

// Every argument and image check of the compute_embeddings calls; runs on the host, before any device call.
int check_embeddings_input(int kind, const void* el, size_t el_len, const void* emb, size_t emb_len,
                           EmbeddingsInput* in) {
    if (!el || !emb) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (kind != GRANNE_B200_ANGULAR && kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "compute_embeddings writes angular or angular_int vectors");
    const int rc = parse_sum_container(static_cast<const uint8_t*>(el), el_len, static_cast<const uint8_t*>(emb),
                                       emb_len, &in->table, &in->el);
    if (rc) return rc;
    in->n = in->el.offsets.size() - 1;
    // an element without terms over a table without rows is the empty vector (embeddings/mod.rs:127-132), and a
    // FixedWidthSliceVector of empty vectors keeps width 0
    in->dim = in->n > 0 && in->table.num > 0 ? (uint32_t)in->table.dim : 0;
    return GRANNE_B200_OK;
}

uint64_t emb_window_rows(uint32_t dim) {
    return std::min(kEmbWindowMaxRows, std::max<uint64_t>(1, kEmbWindowBytes / ((uint64_t)dim * 4)));
}

// End of the window that starts at element r0.
uint64_t emb_window_end(const EmbeddingsInput& in, uint64_t r0) {
    const uint64_t* off = in.el.offsets.data();
    uint64_t r1 = std::min(in.n, r0 + emb_window_rows(in.dim));
    if (off[r1] - off[r0] > kEmbWindowTerms)
        r1 = std::max<uint64_t>(r0 + 1, std::upper_bound(off + r0 + 1, off + r1 + 1, off[r0] + kEmbWindowTerms) - off - 1);
    return r1;
}

// The two kernels for `nr` elements on `stream`: raw rows into d_raw, then Vector::from per row into d_out.  d_out may
// be d_raw (ANGULAR): make_elements_kernel holds a row in shared memory before it writes the row back.  Both are
// counted on `launches` (null: not counted).
int launch_embeddings(const EmbeddingsInput& in, int kind, int num_sms, const float* d_table,
                      const unsigned long long* d_off, uint64_t term_base, const uint32_t* d_terms, uint64_t nr,
                      float* d_raw, void* d_out, int* d_status, cudaStream_t stream, std::atomic<uint64_t>* launches) {
    const gb::SumRowsArgs a{d_table, d_off, term_base, d_terms, nr, in.dim, kind, d_raw, d_status};
    const int rc = launch<gb::sum_embeddings_kernel>((unsigned)std::min<uint64_t>((nr + 7) / 8, (uint64_t)num_sms * 4),
                                                     256, 0, stream, launches, a);
    return rc ? rc
              : launch<gb::make_elements_kernel>((unsigned)std::min<uint64_t>(nr, (uint64_t)num_sms * 32), 32,
                                                 (size_t)in.dim * 4, stream, launches, d_raw, nr, in.dim, kind, d_out);
}

int embeddings_status(int* d_status) {
    int bits = 0;
    GB_CUDA(cudaMemcpy(&bits, d_status, 4, cudaMemcpyDeviceToHost));
    if (bits & gb::kStatusNotFinite)
        return fail(GRANNE_B200_ERR_NOT_FINITE,
                    "an element's sum of embeddings is not finite (angular) or holds NaN (angular_int)");
    return GRANNE_B200_OK;
}

// A pointer the caller says is device memory must be memory of `device`: the kernels would fault on anything else.
int check_device_pointer(const void* p, int device, const char* what) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != device) {
        cudaGetLastError();  // a failed query must not stay behind as the thread's last error
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT,
                    std::string(what) + " is not device memory of device " + std::to_string(device));
    }
    return GRANNE_B200_OK;
}

// Stages a dense element container whose rows already live in HBM (row-major elements: normalised f32 / i8).
int stage_device_elements(Handle* h, int kind, const void* d_rows, uint64_t n, uint32_t dim) {
    if (kind != GRANNE_B200_ANGULAR && kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "device-resident elements: angular or angular_int only");
    if (!d_rows && n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
    if (dim == 0 || dim > 16384) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "vectors wider than 16384 are unsupported");
    int rc;
    if (n && (rc = check_device_pointer(d_rows, h->device, "elements pointer"))) return rc;
    h->dev.kind = kind;
    rc = stage_dense(h, h->dev, h->dev_mem, static_cast<const uint8_t*>(d_rows), n, dim, true);
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

// Makes a handle on `device` with its elements staged: from a file image (el, emb) or, when `dev_rows` is given, from
// n_dev x dim_dev rows already in that device's memory.  `guard` is the caller's, declared before whatever will own
// the handle: it makes the device current here and keeps it current while the caller finishes the handle, so that
// every error path frees the handle's memory on its device.
int new_handle(DeviceGuard* guard, int device, int kind, const uint8_t* el, size_t el_len, const uint8_t* emb,
               size_t emb_len, const void* dev_rows, uint64_t n_dev, uint32_t dim_dev, std::unique_ptr<Handle>* out) {
    int rc = dev_rows ? GRANNE_B200_OK : check_open_args(el, kind, emb);
    if (rc) return rc;
    int num_sms = 0;
    size_t smem_optin = 0;
    if ((rc = check_device(device, &num_sms, &smem_optin))) return rc;
    GB_CUDA(guard->enter(device));
    out->reset(new Handle());
    Handle* h = out->get();
    h->device = device;
    h->num_sms = num_sms;
    h->smem_optin = smem_optin;
    if (dev_rows) return stage_device_elements(h, kind, dev_rows, n_dev, dim_dev);
    return stage_elements(h, kind, el, el_len, emb, emb_len);
}

// `dev_rows` != nullptr: the element container is given as device-resident rows (n_dev x dim_dev) instead of a file image
int open_impl(const uint8_t* index_bytes, size_t index_len, int kind, const uint8_t* el, size_t el_len,
              const uint8_t* emb, size_t emb_len, int device, Handle** out, const void* dev_rows = nullptr,
              uint64_t n_dev = 0, uint32_t dim_dev = 0) {
    if (!out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "out handle pointer is null");
    *out = nullptr;
    if (!index_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index buffer is null");
    DeviceGuard guard;
    std::unique_ptr<Handle> h;
    int rc = new_handle(&guard, device, kind, el, el_len, emb, emb_len, dev_rows, n_dev, dim_dev, &h);
    if (rc) return rc;

    std::string err;
    gb::HostGraph graph;
    if (!gb::parse_index(index_bytes, index_len, &graph, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
    if (graph.layers.size() > (size_t)gb::kMaxLayers) return fail(GRANNE_B200_ERR_FORMAT, "too many layers");
    gb::DeviceIndex& d = h->dev;
    d.num_layers = (int)graph.layers.size();
    for (int l = 0; l < d.num_layers; ++l) {
        const gb::HostLayer& L = graph.layers[l];
        if (L.num_nodes > d.num_elements)
            return fail(GRANNE_B200_ERR_FORMAT, "index refers to more elements than the container holds");
        if ((rc = stage_layer(h.get(), l, L.rows.data(), L.num_nodes, L.width))) return rc;
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

// Hands an encoded image to the caller: always its size; its bytes when there is a buffer, which must hold them.
int copy_image_out(const std::vector<uint8_t>& image, void* out, size_t cap, size_t* out_len) {
    *out_len = image.size();
    if (!out) return GRANNE_B200_OK;
    if (cap < image.size()) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
    std::memcpy(out, image.data(), image.size());
    return GRANNE_B200_OK;
}

// The header of a dense elements image: the rows' width as a little-endian u64 (FixedWidthSliceVector::write).
void write_width_header(uint8_t* image, uint64_t dim) {
    for (int b = 0; b < 8; ++b) image[b] = (uint8_t)(dim >> (8 * b));
}

// ---- launch configuration -----------------------------------------------------------------------------------------
// What every one-warp kernel over a container places first in its shared window: the tiles of the engine that serves
// it, and where its SmemLayout ends.  Behind that the search kernels put their list (and visited set), rerank_kernel
// its keys, the build kernels their link scratch.
struct EngineTiles {
    gb::WarpTiles tiles;
    size_t base_smem;  // gb::SmemLayout::end: tile + id scratch + reserved + query (+ embeddings scratch) + staging
};

EngineTiles engine_tiles(const gb::DeviceIndex& d) {
    EngineTiles e{};
    gb::WarpTiles& t = e.tiles;
    const int fixed_chunks = fixed_f32_chunks(d);
    if (d.kind == gb::kAngularI8) {
        // DistI8: no ordered sums; the staging tile is a set of 512-byte pass slots (32 lanes x one 16-byte chunk each)
        t.tile_rows = 0;
        t.stg_row_bytes = 512;
        t.stg_rows = std::max<uint32_t>(2, (unsigned)GB_STG_BYTES / 512u);
    } else if (d.kind == gb::kSumEmbeddings) {
        // DistSum: the staging tile holds the summed vectors of a batch of candidates (one row each)
        t.tile_rows = 8;
        t.stg_row_bytes = ((d.dim + 3u) & ~3u) * 4u;
        t.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(4, (8192u / t.stg_row_bytes) & ~3u));
    } else if (fixed_chunks > 0) {
        // DistF32<full>: the ordered-sum tile has one row per staged candidate row of a batch
        t.stg_row_bytes = d.full * 128u;
        t.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(4, ((unsigned)GB_STG_BYTES / t.stg_row_bytes) & ~3u));
        t.tile_rows = t.stg_rows;
    } else if (fixed_chunks < 0 && d.full <= 64) {
        // DistF32Generic stages rows of up to 8 KB (dim < 2080), at most 8 (the tile rows) per batch
        t.tile_rows = 8;
        t.stg_row_bytes = d.full * 128u;
        t.stg_rows = std::min<uint32_t>(8u, std::max<uint32_t>(2, (unsigned)(2 * GB_STG_BYTES) / t.stg_row_bytes));
    } else {
        // DistF32<0> (dim < 32) and DistF32Generic on wider rows load directly; the generic engine then parks the lane
        // partials of up to 32 candidates in the tile
        t.tile_rows = 32;
    }
    e.base_smem = gb::SmemLayout<size_t>(0, d.kind, d.dim, d.row_stride, t).end;
    return e;
}

// The search passes' sizes for h's own container.
struct LaunchPlan {
    uint32_t list_cap, vis_slots, vis_upper;
    uint32_t vis_retry;  // visited slots per CTA of the retry pass
    int rows;           // fast list rows R (capacity 32*R), 0 = generic list
    EngineTiles engine;
    size_t smem;        // fast pass total
    size_t extra;       // bytes every pass appends behind its own shared memory (a filtered search's admitted list)
};

// extra: shared memory a pass needs behind its own (0 for an unfiltered search); the generic pass's visited set
// shrinks to leave room for it.
LaunchPlan make_plan(const Handle* h, uint32_t max_search, size_t extra = 0) {
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
    p.engine = engine_tiles(h->dev);
    p.extra = extra;
    const size_t base = p.engine.base_smem;
    const size_t budget = h->smem_optin - extra;
    if (p.rows) {
        // fast pass: list in shared memory, visited set in global memory
        p.vis_slots = (uint32_t)want;
        p.vis_upper = std::min<uint32_t>(1024, p.vis_slots);
        p.smem = base + gb::fast_list_bytes(p.rows) + extra;
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
    p.smem = fixed + (size_t)p.vis_slots * 4 + extra;
    return p;
}

// next longer fast list for the retry pass (0 = none: go straight to the slow pass)
constexpr int retry_rows(int R) { return R == 3 ? 7 : (R == 7 ? 15 : (R == 15 ? 31 : 0)); }

// Raises Kern's dynamic shared-memory limit to the device's opt-in maximum, once per (kernel, device): function
// attributes are per device.  One flag per device ordinal (every handle's device is one, check_device), so the check
// takes no lock.
template <auto Kern>
int raise_smem_limit(const Handle* h) {
    static std::vector<std::atomic<bool>> raised([] {
        int n = 0;
        cudaGetDeviceCount(&n);
        return (size_t)n;
    }());
    std::atomic<bool>& done = raised[h->device];
    if (!done.load()) {
        GB_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        done.store(true);
    }
    return GRANNE_B200_OK;
}

// Launches the one-warp kernel Kern(d, a) over the staged container d, grid CTAs of 32 threads with `smem` bytes of
// dynamic shared memory, and counts it.
template <auto Kern, class Args>
int launch_warps(Handle* h, unsigned grid, size_t smem, cudaStream_t stream, const gb::DeviceIndex& d, const Args& a) {
    const int rc = raise_smem_limit<Kern>(h);
    return rc ? rc : launch<Kern>(grid, 32, smem, stream, &h->launches, d, a);
}

// Resident one-warp CTAs per SM of Kern with `smem` bytes of dynamic shared memory, queried once per (kernel, smem).
template <auto Kern>
int resident_ctas(const Handle* h, size_t smem, int* occ) {
    const int rc = raise_smem_limit<Kern>(h);  // the query counts the CTAs the raised limit admits
    if (rc) return rc;
    static std::mutex mu;
    static std::map<size_t, int> cache;
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(smem);
    if (it == cache.end()) {
        GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, Kern, 32, smem));
        cache[smem] = *occ;
    } else {
        *occ = it->second;
    }
    return GRANNE_B200_OK;
}

template <class Dist, int R, bool FILT>
int launch_kernels(Handle* h, Workspace* w, gb::SearchArgs a, const LaunchPlan& plan, cudaStream_t stream,
                   const gb::DeviceIndex& dv) {
    constexpr int RR = retry_rows(R);
    constexpr auto kern = gb::search_kernel<Dist, R, FILT>;
    constexpr auto retry = gb::search_kernel<Dist, (RR > 0 ? RR : 1), FILT>;
    constexpr auto slow = gb::search_kernel<Dist, 0, FILT>;
    // fast pass
    int occ = 0;
    int rc = resident_ctas<kern>(h, plan.smem, &occ);
    if (rc) return rc;
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
        if ((rc = w->d_vis.grow((size_t)slots * plan.vis_slots, stream))) return rc;
        a.vis_global = w->d_vis.get();
    }
    const bool have_retry = R > 0 && RR > 0;
    a.pass = 0;
    a.slow_pass = 0;
    a.final_pass = 0;
    a.gate_in = nullptr;
    a.gate_out = w->d_counters.get() + 3;
    if ((rc = launch_warps<kern>(h, grid, plan.smem, stream, dv, a))) return rc;
    if (have_retry) {
        // retry pass: only the queries the fast pass flagged (exits at once if none) on a full-size grid of its own,
        // with the next longer list and 8x larger visited tables — so a batch of heavy queries (e.g. the reference's
        // uniform test distribution before the table scale has adapted) never funnels through the 4-CTA slow pass
        gb::SearchArgs r = a;
        r.pass = 1;
        r.work_counter = w->d_counters.get() + 1;
        r.gate_in = w->d_counters.get() + 3;
        r.gate_out = w->d_counters.get() + 4;
        r.vis_slots = std::max(plan.vis_slots, plan.vis_retry);
        r.vis_slots_upper = plan.vis_upper;
        const unsigned rgrid = (unsigned)std::min<unsigned long long>(a.nq, (unsigned long long)h->num_sms * 4);
        if ((rc = w->d_vis_retry.grow((size_t)h->num_sms * 4 * r.vis_slots, stream))) return rc;
        r.vis_global = w->d_vis_retry.get();
        const size_t rsmem = plan.engine.base_smem + gb::fast_list_bytes(RR > 0 ? RR : 1) + plan.extra;
        if ((rc = launch_warps<retry>(h, rgrid, rsmem, stream, dv, r))) return rc;
    }
    // slow pass: re-runs only the queries that are still flagged (exits immediately if none)
    gb::SearchArgs s = a;
    s.pass = 2;
    s.slow_pass = 1;
    s.final_pass = 1;
    s.work_counter = w->d_counters.get() + 2;
    s.gate_in = w->d_counters.get() + (have_retry ? 4 : 3);
    s.gate_out = nullptr;
    return launch_warps<slow>(h, h->slow_ctas, plan.engine.base_smem + plan.extra, stream, dv, s);
}

// ---- workspace pool -----------------------------------------------------------------------------------------------
int ws_acquire(Handle* h, std::unique_ptr<Workspace>* out) {
    {
        std::lock_guard<std::mutex> g(h->pool_mu);
        if (!h->pool.empty()) {
            *out = std::move(h->pool.back());
            h->pool.pop_back();
            return GRANNE_B200_OK;
        }
    }
    std::unique_ptr<Workspace> w(new Workspace());
    cudaStream_t s = nullptr;
    GB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    w->stream.reset(s);
    int rc;
    if ((rc = w->d_counters.grow(16, s))) return rc;
    w->d_error = reinterpret_cast<int*>(w->d_counters.get() + 8);
    if ((rc = w->d_retried.grow(1, s))) return rc;
    GB_CUDA(cudaMemset(w->d_retried.get(), 0, 8));
    if ((rc = w->h_retried.grow(1, s))) return rc;
    *w->h_retried.get() = 0;
    if ((rc = w->d_slow_list.grow((size_t)h->slow_ctas * h->slow_list_cap, s))) return rc;
    if ((rc = w->d_slow_vis.grow((size_t)h->slow_ctas * h->slow_vis_slots, s))) return rc;
    *out = std::move(w);
    return GRANNE_B200_OK;
}
void ws_release(Handle* h, std::unique_ptr<Workspace> w) {
    std::lock_guard<std::mutex> g(h->pool_mu);
    h->pool.push_back(std::move(w));
}

// A host call's buffers for nq queries and m result entries (ids | dists | counts: m, m and nq words).
int ws_reserve(Workspace* w, size_t query_bytes, size_t nq, size_t m) {
    cudaStream_t s = w->stream.get();
    int rc;
    if ((rc = w->d_queries.grow(query_bytes, s)) || (rc = w->d_ids.grow(2 * m + nq, s)) ||
        (rc = w->d_stats.grow(nq * 4, s)))
        return rc;
    w->d_dists = reinterpret_cast<float*>(w->d_ids.get() + m);
    w->d_counts = w->d_ids.get() + 2 * m;
    return w->h_pinned.grow(query_bytes + m * 8 + nq * 4 + nq * 32 + 128, s);
}

// One workspace per caller stream: calls on the same stream are serialised by the stream itself, so the status words /
// slow-path buffers can be reused; the error word stays sticky until granne_b200_stream_status().
int stream_workspace(Handle* h, cudaStream_t stream, Workspace** out) {
    Workspace* w = nullptr;
    {
        std::lock_guard<std::mutex> g(h->pool_mu);
        auto it = h->stream_ws.find(stream);
        if (it != h->stream_ws.end()) w = it->second.get();
    }
    if (!w) {
        std::unique_ptr<Workspace> fresh;
        int rc;
        if ((rc = ws_acquire(h, &fresh))) return rc;
        cudaError_t e = cudaMemset(fresh->d_error, 0, 4 * sizeof(int));
        {
            std::lock_guard<std::mutex> g(h->pool_mu);
            auto it = h->stream_ws.find(stream);  // two threads may meet here on the first use of a stream
            if (it == h->stream_ws.end()) it = h->stream_ws.emplace(stream, std::move(fresh)).first;
            w = it->second.get();
        }
        if (fresh) ws_release(h, std::move(fresh));  // lost that race: back to the pool
        GB_CUDA(e);
    }
    *out = w;
    return GRANNE_B200_OK;
}

bool by_id(int fmt) { return fmt == GRANNE_B200_QUERY_ID || fmt == GRANNE_B200_QUERY_ID_EXCLUDING; }

// The argument rules every query call shares, in the order they are reported.  None of them reads the handle, so bad
// arguments are reported before anything touches a device.  `own_rule`: the message of the call's own rule on its
// sizes when the arguments break it, else nullptr.  `id_formats`: the call also takes queries by element id.
int validate_batch(const Handle* h, const void* q, size_t nq, int fmt, uint32_t k, const void* ids, const void* dists,
                   const char* own_rule, bool id_formats = true) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    if (fmt != GRANNE_B200_QUERY_RAW_F32 && fmt != GRANNE_B200_QUERY_ELEMENT && !(id_formats && by_id(fmt)))
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "unknown query format");
    if (own_rule) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, own_rule);
    if (nq > 0xFFFFFFF0ull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many queries in one batch");
    if (nq && (!q || (k && (!ids || !dists)))) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null buffer");
    return GRANNE_B200_OK;
}

constexpr const char* kMaxSearchRule = "max_search must be >= 1 (the reference panics on 0, src/index/mod.rs:1019)";
constexpr const char* kExactKRule = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)";
constexpr const char* kBadCandidatesRule =
    "a candidate list is longer than its stride, not ascending by distance, or holds an id >= Index::len";

int validate_search(const Handle* h, const void* q, size_t nq, int fmt, uint32_t max_search, uint32_t k,
                    const void* ids, const void* dists, bool id_formats = true) {
    return validate_batch(h, q, nq, fmt, k, ids, dists, max_search == 0 ? kMaxSearchRule : nullptr, id_formats);
}

int validate_exact(const Handle* h, const void* q, size_t nq, int fmt, uint32_t k, const void* ids,
                   const void* dists) {
    return validate_batch(h, q, nq, fmt, k, ids, dists, k > GRANNE_B200_EXACT_MAX_K ? kExactKRule : nullptr);
}

// The rule QUERY_ID_EXCLUDING adds, reported after a call's other rules: the call runs with k + 1 columns, so k + 1
// must be within the call's cap (GRANNE_B200_EXACT_MAX_K, or the u32 range for search_batch).
int check_exclude_k(int fmt, uint32_t k, uint64_t cap) {
    if (fmt == GRANNE_B200_QUERY_ID_EXCLUDING && (uint64_t)k + 1 > cap)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT,
                    cap == GRANNE_B200_EXACT_MAX_K
                        ? "num_neighbors exceeds 1023 with GRANNE_B200_QUERY_ID_EXCLUDING (the call runs k + 1)"
                        : "num_neighbors + 1 exceeds u32 with GRANNE_B200_QUERY_ID_EXCLUDING");
    return GRANNE_B200_OK;
}

// The host check of n element ids in host memory: each < granne_b200_num_elements(h).
int check_element_ids(const Handle* h, const uint32_t* ids, size_t n) {
    for (size_t i = 0; i < n; ++i)
        if (ids[i] >= h->dev.num_elements)
            return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "element id >= granne_b200_num_elements");
    return GRANNE_B200_OK;
}

// The host check of a host call's queries: its ids when the call is by id, else nothing.
int check_host_query_ids(const Handle* h, const void* queries, size_t nq, int fmt) {
    return by_id(fmt) ? check_element_ids(h, static_cast<const uint32_t*>(queries), nq) : GRANNE_B200_OK;
}

gb::PeerGather device_gather(const granne_b200_peer_gather& pg, unsigned int* done_counter) {
    gb::PeerGather d{};
    d.n_peers = pg.n_peers;
    d.my_rank = pg.my_rank;
    d.row_offset = pg.row_offset;
    d.seq = pg.seq;
    d.done_counter = done_counter;
    for (uint32_t p = 0; p < pg.n_peers; ++p) {
        d.ids[p] = static_cast<uint32_t*>(pg.ids[p]);
        d.dists[p] = static_cast<float*>(pg.dists[p]);
        d.flags[p] = static_cast<unsigned int*>(pg.flags[p]);
    }
    return d;
}

// The filters of a filtered search, in device memory (granne_b200_search_filtered_batch_device's arguments).
struct DeviceFilters {
    const uint32_t* words;         // num_filters x filter_words u32
    const uint32_t* query_filter;  // nq entries, or null (every query uses filter 0)
    uint64_t filter_words;
    uint32_t num_filters;
    uint64_t bit_base;             // bit of element 0 (a shard's base in a range-partitioned multi handle)
};

// The device outputs of a query call, in search_batch's layout: nq x k ids and distances, nq counts, nq x 4 stats (a
// null pointer: not wanted, where the call allows it).
struct QueryOut {
    uint32_t* ids;
    float* dists;
    uint32_t* counts;
    uint64_t* stats;
};

// Enqueues one batch on `stream` with device pointers.  Needs a workspace for status words / slow path, whose counters
// the caller has zeroed on `stream` (Workspace::d_counters; the per-query status words need no reset: the fast pass
// writes every one of them).  `filt`: a filtered search (search_kernel<Dist, R, true>), whose passes each append
// round_up(k, 32) keys of shared memory.
int enqueue_search(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, uint32_t max_search,
                   uint32_t k, const QueryOut& out, cudaStream_t stream, const granne_b200_peer_gather* pg = nullptr,
                   const gb::DeviceIndex* view = nullptr, const DeviceFilters* filt = nullptr) {
    const uint32_t filter_cap = (k + 31u) & ~31u;
    const LaunchPlan plan = make_plan(h, max_search, filt ? (size_t)filter_cap * 8 : 0);
    if (plan.smem == 0 || max_search + 64 > h->slow_list_cap)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search exceeds the supported maximum (about 27000)");
    int rc = w->d_status.grow(nq, stream);
    if (rc) return rc;
    // the slow-path visited tables follow the index size (a builder's index grows after its workspace was made)
    if ((rc = w->d_slow_vis.grow((size_t)h->slow_ctas * h->slow_vis_slots, stream))) return rc;
    // Adapt the visited-table scale to the data: more than 1% of the recent queries needed the retry pass -> double
    // it (read from the pinned mirror of the device counter, i.e. without synchronising; it lags by a call or two).
    w->total_queries += nq;
    {
        const unsigned long long retried = *reinterpret_cast<volatile unsigned long long*>(w->h_retried.get());
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
    gb::SearchArgs a{};
    a.queries = d_queries;
    a.query_format = fmt;
    a.nq = nq;
    a.max_search = max_search;
    a.num_neighbors = k;
    a.list_cap = plan.list_cap;
    a.vis_slots = plan.vis_slots;
    a.vis_slots_upper = plan.vis_upper;
    a.out_ids = out.ids;
    a.out_dists = out.dists;
    a.out_counts = out.counts;
    a.out_stats = reinterpret_cast<unsigned long long*>(out.stats);
    a.query_status = w->d_status.get();
    a.work_counter = w->d_counters.get();
    a.retried = w->d_retried.get();
    a.error_flag = w->d_error;
    a.slow_list = w->d_slow_list.get();
    a.slow_visited = w->d_slow_vis.get();
    a.slow_list_cap = h->slow_list_cap;
    a.slow_vis_slots = h->slow_vis_slots;
    a.pass = a.slow_pass = a.final_pass = 0;
    a.pg = pg ? device_gather(*pg, w->d_counters.get() + 5) : gb::PeerGather{};
    a.tiles = plan.engine.tiles;
    a.vis_global = nullptr;
    if (filt) {
        a.filters = filt->words;
        a.query_filter = filt->query_filter;
        a.filter_words = filt->filter_words;
        a.filter_bit_base = filt->bit_base;
        a.num_filters = filt->num_filters;
        a.filter_cap = filter_cap;
    }
    // the staged index the kernels see: the handle's own, or a private view of it (compute_order searches single
    // layers without touching the shared handle)
    const gb::DeviceIndex& dv = view ? *view : h->dev;
    auto launch = [&](auto filtered) {
        constexpr bool FILT = decltype(filtered)::value;
        return DistDispatch::call(dv, [&](auto e) {
            using Dist = typename decltype(e)::type;
            switch (plan.rows) {
                case 3: return launch_kernels<Dist, 3, FILT>(h, w, a, plan, stream, dv);
                case 7: return launch_kernels<Dist, 7, FILT>(h, w, a, plan, stream, dv);
                case 15: return launch_kernels<Dist, 15, FILT>(h, w, a, plan, stream, dv);
                case 31: return launch_kernels<Dist, 31, FILT>(h, w, a, plan, stream, dv);
                default: return launch_kernels<Dist, 0, FILT>(h, w, a, plan, stream, dv);
            }
        });
    };
    rc = filt ? launch(std::true_type{}) : launch(std::false_type{});
    if (rc) return rc;
    GB_CUDA(cudaMemcpyAsync(w->h_retried.get(), w->d_retried.get(), 8, cudaMemcpyDeviceToHost, stream));
    return GRANNE_B200_OK;
}

int error_from_bits(int bits) {
    if (bits & gb::kStatusNotFinite)
        return fail(GRANNE_B200_ERR_NOT_FINITE, "a NaN distance occurred (non-finite query or element)");
    if (bits & gb::kStatusOverflow)
        return fail(GRANNE_B200_ERR_CAPACITY, "exact search workspace exhausted even on the slow path");
    if (bits & gb::kStatusBadList)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "a candidate list has bad offsets or an id >= Index::len");
    if (bits & gb::kStatusBadFilter)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "a query_filter entry is >= num_filters");
    if (bits & gb::kStatusBadId)
        return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "an element id is >= granne_b200_num_elements");
    if (bits & gb::kStatusBadSegment)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT,
                    "a range search segment's length differs from its query's count (it is padded)");
    if (bits & gb::kStatusBadCandidates)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, kBadCandidatesRule);
    return GRANNE_B200_OK;
}

// Bytes of one query row in `fmt` for an index of `kind` (gb::ElementKind) and width `dim`: a u32 id for the id
// formats, i8 when the queries already are elements of an angular_int index, f32 otherwise.
size_t query_row_bytes(int kind, uint32_t dim, int fmt) {
    if (by_id(fmt)) return 4;
    return (size_t)dim * (kind == gb::kAngularI8 && fmt == GRANNE_B200_QUERY_ELEMENT ? 1 : 4);
}

// The host-pointer form of a query call (arguments validated, nq > 0), on a pooled workspace and its stream: the
// queries go up through pinned memory, the call's words are zeroed (Workspace::d_counters), `enqueue(w, stream, out)`
// queues the call's kernels from w->d_queries into the workspace's result block (w->d_ids | w->d_dists | w->d_counts:
// m ids, m dists, nq counts; out.stats is null when the caller wants no stats), and one synchronise brings the results
// and the error word back.  host_batch: the k columns of search_batch's layout, m = nq * k.
template <class Enqueue>
int host_batch_entries(Handle* h, const void* queries, size_t nq, int fmt, size_t m, uint32_t* out_ids,
                       float* out_dists, uint32_t* out_counts, uint64_t* out_stats, Enqueue&& enqueue) {
    return guarded([&] {
        GB_DEVICE(h->device);
        std::unique_ptr<Workspace> ws;
        int rc = ws_acquire(h, &ws);
        if (rc) return rc;
        Workspace* w = ws.get();
        const size_t qbytes = nq * query_row_bytes(h->dev.kind, h->dev.dim, fmt);
        const int status = [&] {
            if ((rc = ws_reserve(w, qbytes, nq, m))) return rc;
            cudaStream_t stream = w->stream.get();
            // pinned staging layout: queries | ids | dists | counts | error | stats, the blocks behind the queries and
            // behind the error word on 16-byte boundaries (ws_reserve sizes the buffer with slack for both)
            uint8_t* hp = w->h_pinned.get();
            uint32_t* hids = reinterpret_cast<uint32_t*>(hp + ((qbytes + 15) & ~size_t(15)));
            float* hd = reinterpret_cast<float*>(hids + m);
            uint32_t* hc = reinterpret_cast<uint32_t*>(hd + m);
            int* herr = reinterpret_cast<int*>(hc + nq);
            unsigned long long* hstats = reinterpret_cast<unsigned long long*>(
                hp + ((reinterpret_cast<uint8_t*>(herr + 4) - hp + 15) & ~size_t(15)));
            std::memcpy(hp, queries, qbytes);
            GB_CUDA(cudaMemcpyAsync(w->d_queries.get(), hp, qbytes, cudaMemcpyHostToDevice, stream));
            GB_CUDA(cudaMemsetAsync(w->d_counters.get(), 0, kHostCallBytes, stream));
            uint64_t* d_stats = out_stats ? reinterpret_cast<uint64_t*>(w->d_stats.get()) : nullptr;
            if ((rc = enqueue(w, stream, QueryOut{w->d_ids.get(), w->d_dists, w->d_counts, d_stats}))) return rc;
            // one packed copy: ids | dists | counts (device and pinned layouts match), then the 16-byte error word
            GB_CUDA(cudaMemcpyAsync(hids, w->d_ids.get(), (2 * m + nq) * 4, cudaMemcpyDeviceToHost, stream));
            GB_CUDA(cudaMemcpyAsync(herr, w->d_error, 4 * sizeof(int), cudaMemcpyDeviceToHost, stream));
            if (out_stats) GB_CUDA(cudaMemcpyAsync(hstats, w->d_stats.get(), nq * 32, cudaMemcpyDeviceToHost, stream));
            GB_CUDA(cudaStreamSynchronize(stream));
            if (out_stats) std::memcpy(out_stats, hstats, nq * 32);
            if (m) {
                std::memcpy(out_ids, hids, m * 4);
                std::memcpy(out_dists, hd, m * 4);
            }
            if (out_counts) std::memcpy(out_counts, hc, nq * 4);
            return error_from_bits(herr[0]);
        }();
        ws_release(h, std::move(ws));  // back to the pool on every path
        return status;
    });
}
template <class Enqueue>
int host_batch(Handle* h, const void* queries, size_t nq, int fmt, size_t k, uint32_t* out_ids, float* out_dists,
               uint32_t* out_counts, uint64_t* out_stats, Enqueue&& enqueue) {
    return host_batch_entries(h, queries, nq, fmt, nq * k, out_ids, out_dists, out_counts, out_stats,
                              std::forward<Enqueue>(enqueue));
}

// The device-pointer form of a query call (arguments validated, nq > 0): `enqueue(w, stream)` queues the call's
// kernels on the caller's stream with that stream's workspace, after zeroing its search counters when the call
// `searches` (Workspace::d_counters).  Asynchronous; errors stay in the workspace's error word until
// granne_b200_stream_status().
template <class Enqueue>
int device_batch(Handle* h, void* cuda_stream, bool searches, Enqueue&& enqueue) {
    return guarded([&] {
        GB_DEVICE(h->device);
        cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
        Workspace* w = nullptr;
        int rc = stream_workspace(h, stream, &w);
        if (rc) return rc;
        if (searches) GB_CUDA(cudaMemsetAsync(w->d_counters.get(), 0, kSearchCounterBytes, stream));
        return enqueue(w, stream);
    });
}

struct HostInput { const void* data; size_t bytes; };  // a caller's array that a host call copies to the device

// Runs `enqueue(d)` with the arrays `in` copied up on `stream`, d[i] the device copy of in[i], all in one stream-ordered
// allocation freed behind the call's kernels: they are the caller's inputs, not workspace, so that long lists or large
// bitmaps leave no device memory held by the pooled workspace.  An error of the enqueue is reported before one of the
// free.
template <size_t N, class Enqueue>
int with_call_inputs(cudaStream_t stream, const HostInput (&in)[N], Enqueue&& enqueue) {
    size_t total = 0;
    for (const HostInput& a : in) total += a.bytes;
    void* mem = nullptr;
    GB_CUDA(cudaMallocAsync(&mem, total, stream));
    const int rc = [&] {
        const void* d[N];
        uint8_t* p = static_cast<uint8_t*>(mem);
        for (size_t i = 0; i < N; p += in[i].bytes, ++i) {
            d[i] = p;
            if (in[i].bytes) GB_CUDA(cudaMemcpyAsync(p, in[i].data, in[i].bytes, cudaMemcpyHostToDevice, stream));
        }
        return enqueue(d);
    }();
    const cudaError_t fe = cudaFreeAsync(mem, stream);
    if (rc) return rc;
    GB_CUDA(fe);
    return GRANNE_B200_OK;
}

// ---- queries by element id (ids_kernels.cuh) ------------------------------------------------------------------------
// Enqueues a query call on `stream` whatever its format: `call(q, fmt, k, out)` queues the call's kernels for device
// query rows q.  RAW_F32 and ELEMENT queries go straight to it.  Ids (nq u32 in device memory at d_q) are read as
// elements first: get_elements_kernel writes their rows into the workspace (a bad id reads nothing and flags its
// query), the call runs on those rows as ELEMENT queries, and id_results_kernel writes the caller's columns.
// QUERY_ID runs the call into the caller's output; only a device call, whose ids no host has checked
// (`host_checked`), needs the pass that blanks flagged queries.  QUERY_ID_EXCLUDING runs it with k + 1 columns into
// the workspace (stats straight into the caller's: they do not depend on k) and drops each query's own id.
// The rows of nq ids (device memory) as ELEMENT queries in w->d_id_rows, their bad-id flags in w->d_id_bad.
int enqueue_id_rows(Handle* h, Workspace* w, const uint32_t* ids, size_t nq, cudaStream_t stream) {
    const gb::DeviceIndex& d = h->dev;
    const size_t row = query_row_bytes(d.kind, d.dim, GRANNE_B200_QUERY_ELEMENT);
    int rc;
    if ((rc = w->d_id_rows.grow(std::max<size_t>(nq * row, 16), stream)) || (rc = w->d_id_bad.grow(nq, stream)))
        return rc;
    const size_t smem = d.kind == gb::kSumEmbeddings ? (size_t)d.dim * 4 : 0;
    return launch<gb::get_elements_kernel>((unsigned)std::min<uint64_t>(nq, (uint64_t)h->num_sms * 32), 32, smem, stream,
                                           &h->launches, d, ids, nq, d.num_elements, w->d_id_rows.get(),
                                           w->d_id_bad.get(), w->d_error);
}

template <class Call>
int enqueue_query(Handle* h, Workspace* w, const void* d_q, size_t nq, int fmt, uint32_t k, const QueryOut& out,
                  bool host_checked, cudaStream_t stream, Call&& call) {
    if (!by_id(fmt)) return call(d_q, fmt, k, out);
    const bool exclude = fmt == GRANNE_B200_QUERY_ID_EXCLUDING;
    const uint32_t* ids = static_cast<const uint32_t*>(d_q);
    int rc = enqueue_id_rows(h, w, ids, nq, stream);
    if (rc) return rc;
    QueryOut res = out;
    const uint32_t kk = exclude ? k + 1 : k;
    if (exclude) {
        if ((rc = w->d_id_res.grow(2 * nq * kk + nq, stream))) return rc;
        uint32_t* r = w->d_id_res.get();
        res = {r, reinterpret_cast<float*>(r + nq * kk), r + 2 * nq * kk, out.stats};
    }
    if ((rc = call(w->d_id_rows.get(), (int)GRANNE_B200_QUERY_ELEMENT, kk, res))) return rc;
    if (!exclude && host_checked) return GRANNE_B200_OK;
    return launch<gb::id_results_kernel>((unsigned)std::min<uint64_t>((nq + 3) / 4, (uint64_t)h->num_sms * 16), 128, 0,
                                         stream, &h->launches, res.ids, res.dists, res.counts, kk, ids,
                                         w->d_id_bad.get(), exclude, nq, k, out.ids, out.dists, out.counts,
                                         reinterpret_cast<unsigned long long*>(out.stats));
}

// ---- exact k-NN (exact_kernels.cuh) -------------------------------------------------------------------------------
// The slab buffer holds at most kExactSlabFloats distances (256 MB) and a slab at most kExactMaxSlabRows rows, so the
// workspace of a call is bounded whatever nq and n are.
constexpr uint64_t kExactSlabFloats = 64ull << 20;
constexpr uint64_t kExactMaxSlabRows = 1ull << 20;

// Distances of the prepared query chunk (qc queries in w->d_exact_q) to `nrows` rows, slab by slab into
// w->d_exact_dists (qc rows of `slab` floats), each slab then handed to step(ns, id_base): the ns distances of row r
// belong to element id_base + r.
template <class Step>
int exact_scan_rows(Handle* h, Workspace* w, uint32_t qc, const void* rows, uint64_t nrows, uint32_t row_stride,
                    uint32_t vec_group, uint64_t base, uint64_t slab, cudaStream_t stream, Step& step) {
    const gb::DeviceIndex& d = h->dev;
    for (uint64_t s0 = 0; s0 < nrows; s0 += slab) {
        const uint64_t ns = std::min(slab, nrows - s0);
        gb::ExactScanArgs a{};
        a.row_stride = row_stride;
        a.vec_group = vec_group;
        a.nrows = ns;
        a.dim = d.dim;
        a.full = d.full;
        a.tail = d.tail;
        a.queries = w->d_exact_q.get();
        a.qnorm = w->d_exact_qnorm.get();
        a.nq = qc;
        a.dists = w->d_exact_dists.get();
        a.ld = slab;
        a.error = w->d_error;
        const dim3 grid((unsigned)((ns + gb::kExactRB - 1) / gb::kExactRB), (qc + gb::kExactQB - 1) / gb::kExactQB);
        int rc;
        if (d.kind == gb::kAngularI8) {
            a.rows = static_cast<const int8_t*>(rows) + s0 * row_stride;
            rc = launch<gb::exact_scan_i8_kernel<false>>(grid, 256, 0, stream, &h->launches, a);
        } else {
            a.rows = static_cast<const float*>(rows) + s0 * row_stride;
            rc = launch<gb::exact_scan_f32_kernel<false>>(grid, 256, 0, stream, &h->launches, a);
        }
        if (rc || (rc = step(ns, base + s0))) return rc;
    }
    return GRANNE_B200_OK;
}

// Distances of the prepared query chunk to the rows of a list (LISTED): row r of w->d_exact_dists is element ids[r] of
// `rows` (ids null: row r), for r < count[0] (device memory; at most `cap`).  The host does not know the count, so the
// grid is one wave of the scan's blocks (at most the list's capacity in row tiles) and the blocks stride over the
// tiles: a short list costs a small launch, not the slab grid, and an empty one a launch whose blocks return.  (The
// slab-shaped grid, its blocks past the count returning, measured 0.9 ms slower at 0.1 % and 15 % slower on full f32
// lists over 10M x 128 on an H100, though 6 % faster on i8 rows.)
int exact_scan_listed(Handle* h, Workspace* w, uint32_t qc, const void* rows, uint32_t row_stride, uint32_t vec_group,
                      const uint32_t* ids, const uint32_t* count, uint64_t cap, uint64_t ld, cudaStream_t stream) {
    const gb::DeviceIndex& d = h->dev;
    gb::ExactScanArgs a{};
    a.rows = rows;
    a.row_stride = row_stride;
    a.vec_group = vec_group;
    a.dim = d.dim;
    a.full = d.full;
    a.tail = d.tail;
    a.queries = w->d_exact_q.get();
    a.qnorm = w->d_exact_qnorm.get();
    a.nq = qc;
    a.dists = w->d_exact_dists.get();
    a.ld = ld;
    a.row_ids = ids;
    a.row_count = count;
    const unsigned gy = (qc + gb::kExactQB - 1) / gb::kExactQB;
    // two 256-thread blocks per SM are resident: no more than fit, so that no block waits for a whole list's tiles
    const uint64_t wave = std::max<uint64_t>(1, (uint64_t)h->num_sms * 2 / gy);
    const dim3 grid((unsigned)std::max<uint64_t>(1, std::min(wave, (cap + gb::kExactRB - 1) / gb::kExactRB)), gy);
    return d.kind == gb::kAngularI8 ? launch<gb::exact_scan_i8_kernel<true>>(grid, 256, 0, stream, &h->launches, a)
                                    : launch<gb::exact_scan_f32_kernel<true>>(grid, 256, 0, stream, &h->launches, a);
}

// Ids per list of a filtered scan: a slab, and for EMBEDDINGS at most a window of materialised rows; at least 32, so
// that a word of the bitmaps always fits (exact_list_ids_kernel).
uint64_t list_cap(uint64_t slab, uint64_t wrows, bool emb) {
    return emb ? std::min(slab, std::max<uint64_t>(wrows, 32)) : slab;
}

// The ExactList of query chunk c0 of a filtered scan (exact_scan with filters): its id buffer holds `slab` ids, the
// chunk's filters, then the three counts (exact_list_ids_kernel).
gb::ExactList exact_list(Workspace* w, const DeviceFilters& f, size_t c0, uint64_t slab) {
    gb::ExactList l{};
    l.ids = w->d_exact_ids.get();
    l.count = l.ids + slab + gb::kExactMaxChunk;
    l.filters = f.words;
    l.query_filter = f.query_filter ? f.query_filter + c0 : nullptr;
    l.filter_words = f.filter_words;
    l.bit_base = f.bit_base;
    l.num_filters = f.num_filters;
    l.qstatus = w->d_exact_qstat.get();
    l.error = w->d_error;
    return l;
}

// The exact scan of nq queries (device memory, the caller's format) against [0, Index::len), the loop the exact and
// range calls share: query chunks of at most kExactMaxChunk, and per chunk begin(c0, qc), the queries prepared as
// elements, every slab of rows (EMBEDDINGS: of every window of materialised rows) scanned and handed to
// slab_step(c0, qc, ns, id_base, ld) with its distances in w->d_exact_dists (qc rows of ld floats), then end(c0, qc).
// Without `scan` (no rows, or nothing to rank) only begin and end run.  A NaN distance or query sets kStatusNotFinite
// in w->d_error.
//
// With `filt` (the exact filtered call) the rows scanned are the ids the chunk's filters admit (exact_list): they are
// listed on the device, up to list_cap ids at a time from a cursor that stays on the device, only their rows are
// scanned (exact_scan_listed), and slab_step(c0, qc, slab, 0, slab) finds the ids and their count in the chunk's
// ExactList.  The host issues as many lists as the densest filter could need; those past the end are empty.  A NaN is
// left for that step to flag (exact_select_kernel<true>), with each query's prepare status in w->d_exact_qstat.  No
// host synchronisation: the counts stay on the device.
template <class Begin, class Slab, class End>
int exact_scan(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, bool scan, cudaStream_t stream,
               Begin&& begin, Slab&& slab_step, End&& end, const DeviceFilters* filt = nullptr) {
    const gb::DeviceIndex& d = h->dev;
    const uint64_t n = h->index_len;
    const bool i8 = d.kind == gb::kAngularI8, emb = d.kind == gb::kSumEmbeddings;
    const size_t in_row = query_row_bytes(d.kind, d.dim, fmt);
    const size_t qc_max = std::min<size_t>(nq, gb::kExactMaxChunk);
    uint64_t slab = 0;
    const float* table = static_cast<const float*>(d.vectors);
    uint64_t wrows = 0;
    int rc;
    if (scan) {
        slab = std::min<uint64_t>(kExactMaxSlabRows, kExactSlabFloats / qc_max) / gb::kExactRB * gb::kExactRB;
        slab = std::min<uint64_t>(slab, (n + gb::kExactRB - 1) / gb::kExactRB * gb::kExactRB);
        const size_t qrow = i8 ? d.row_stride : (size_t)d.dim * 4;
        if ((rc = w->d_exact_q.grow(std::max<size_t>(qc_max * qrow, 16), stream)) ||
            (rc = w->d_exact_qnorm.grow(qc_max, stream)) || (rc = w->d_exact_dists.grow(qc_max * slab, stream)))
            return rc;
        if (emb) {
            // SumEmbeddings::get rows, window by window (compute_embeddings' ANGULAR rows, which search exactly like
            // the container); the staged table's rows are padded to a multiple of 4 floats, the sum kernel reads
            // dense rows
            wrows = std::min<uint64_t>(n, emb_window_rows(std::max<uint32_t>(d.dim, 1)));
            const uint64_t rows_cap = filt ? std::max(wrows, list_cap(slab, wrows, emb)) : wrows;
            if ((rc = w->d_exact_rows.grow(std::max<size_t>(rows_cap * d.dim, 16), stream))) return rc;
            if (d.row_stride != d.dim && d.num_vectors) {
                if ((rc = w->d_exact_table.grow((size_t)d.num_vectors * d.dim, stream))) return rc;
                GB_CUDA(cudaMemcpy2DAsync(w->d_exact_table.get(), (size_t)d.dim * 4, d.vectors,
                                          (size_t)d.row_stride * 4, (size_t)d.dim * 4, d.num_vectors,
                                          cudaMemcpyDeviceToDevice, stream));
                table = w->d_exact_table.get();
            }
        }
        if (filt && ((rc = w->d_exact_ids.grow(slab + gb::kExactMaxChunk + 3, stream)) ||
                     (rc = w->d_exact_qstat.grow(qc_max, stream))))
            return rc;
    }
    for (size_t c0 = 0; c0 < nq; c0 += gb::kExactMaxChunk) {
        const uint32_t qc = (uint32_t)std::min<size_t>(gb::kExactMaxChunk, nq - c0);
        if ((rc = begin(c0, qc))) return rc;
        if (scan) {
            if ((rc = launch<gb::exact_prepare_kernel>((unsigned)std::min<uint64_t>(qc, (uint64_t)h->num_sms * 32), 32, 0,
                                                       stream, &h->launches, d,
                                                       static_cast<const uint8_t*>(d_queries) + c0 * in_row, fmt, qc,
                                                       w->d_exact_q.get(), w->d_exact_qnorm.get(), w->d_error,
                                                       filt ? w->d_exact_qstat.get() : nullptr)))
                return rc;
            auto step = [&](uint64_t ns, uint64_t id_base) { return slab_step(c0, qc, ns, id_base, slab); };
            if (filt) {
                const gb::ExactList l = exact_list(w, *filt, c0, slab);
                uint32_t* count = const_cast<uint32_t*>(l.count);
                uint32_t* ids = w->d_exact_ids.get();
                if ((rc = launch<gb::exact_chunk_filters_kernel>(1, gb::kExactListThreads, 0, stream, &h->launches,
                                                                 l.query_filter, qc, filt->num_filters, ids + slab,
                                                                 count)))
                    return rc;
                // lists of at most `cap` ids, each but the last fuller than cap - 32 (exact_list_ids_kernel)
                const uint64_t cap = list_cap(slab, wrows, emb);
                const uint64_t lists = (n + cap - 32) / (cap - 31);
                for (uint64_t li = 0; li < lists; ++li) {
                    if ((rc = launch<gb::exact_list_ids_kernel>(1, gb::kExactListThreads, 0, stream, &h->launches,
                                                                filt->words, filt->filter_words, filt->bit_base,
                                                                ids + slab, count, n, (uint32_t)cap, ids)))
                        return rc;
                    if (emb) {
                        if ((rc = launch<gb::exact_listed_rows_kernel>(
                                 (unsigned)std::min<uint64_t>(cap, (uint64_t)h->num_sms * 32), 32, (size_t)d.dim * 4,
                                 stream, &h->launches, d, ids, count, w->d_exact_rows.get())))
                            return rc;
                        rc = exact_scan_listed(h, w, qc, w->d_exact_rows.get(), d.dim, 1, nullptr, count, cap, slab,
                                               stream);
                    } else {
                        rc = exact_scan_listed(h, w, qc, d.vectors, d.row_stride, d.vec_group, ids, count, cap, slab,
                                               stream);
                    }
                    if (rc || (rc = step(slab, 0))) return rc;
                }
            } else if (emb) {
                EmbeddingsInput in;
                in.dim = d.dim;
                for (uint64_t r0 = 0; r0 < n; r0 += wrows) {
                    const uint64_t nr = std::min(wrows, n - r0);
                    if ((rc = launch_embeddings(in, gb::kAngularF32, h->num_sms, table, d.sum_offsets + r0, 0,
                                                d.sum_terms, nr, w->d_exact_rows.get(), w->d_exact_rows.get(),
                                                w->d_error, stream, &h->launches)))
                        return rc;
                    if ((rc = exact_scan_rows(h, w, qc, w->d_exact_rows.get(), nr, d.dim, 1, r0, slab, stream, step)))
                        return rc;
                }
            } else if ((rc = exact_scan_rows(h, w, qc, d.vectors, n, d.row_stride, d.vec_group, 0, slab, stream,
                                             step))) {
                return rc;
            }
        }
        if ((rc = end(c0, qc))) return rc;
    }
    return GRANNE_B200_OK;
}

// Enqueues one exact search on `stream`: nq queries (device memory, the caller's format) against [0, Index::len),
// results in search_batch's layout.  A NaN distance or query sets kStatusNotFinite in w->d_error.  With `filt` (the
// exact filtered call) query q ranks the ids its filter admits only: the LISTED scan, select and write (exact_scan);
// a query whose query_filter entry is >= num_filters gets count 0 and padding and sets kStatusBadFilter.
int enqueue_exact(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, uint32_t k, const QueryOut& out,
                  cudaStream_t stream, const DeviceFilters* filt = nullptr) {
    const uint64_t n = h->index_len;
    const uint32_t count = (uint32_t)std::min<uint64_t>(k, n);
    const bool scan = k > 0 && n > 0;
    int rc;
    if (scan && (rc = w->d_exact_lists.grow(std::min<size_t>(nq, gb::kExactMaxChunk) * gb::kExactMaxK, stream)))
        return rc;
    return exact_scan(
        h, w, d_queries, nq, fmt, scan, stream,
        [&](size_t, uint32_t qc) {
            if (scan) GB_CUDA(cudaMemsetAsync(w->d_exact_lists.get(), 0xFF, (size_t)qc * gb::kExactMaxK * 8, stream));
            return (int)GRANNE_B200_OK;
        },
        [&](size_t c0, uint32_t qc, uint64_t ns, uint64_t id_base, uint64_t ld) {
            if (filt)
                return launch<gb::exact_select_kernel<true>>(qc, gb::kExactSelThreads, 0, stream, &h->launches,
                                                             w->d_exact_dists.get(), ld, ns, 0, k,
                                                             w->d_exact_lists.get(), exact_list(w, *filt, c0, ld));
            return launch<gb::exact_select_kernel<false>>(qc, gb::kExactSelThreads, 0, stream, &h->launches,
                                                          w->d_exact_dists.get(), ld, ns, (uint32_t)id_base, k,
                                                          w->d_exact_lists.get(), gb::ExactList{});
        },
        [&](size_t c0, uint32_t qc) {
            // a filtered call always writes: its kernel also checks the chunk's query_filter entries
            const uint64_t outs = std::max<uint64_t>((uint64_t)qc * k, out.counts || filt ? qc : 0);
            if (outs == 0) return (int)GRANNE_B200_OK;
            uint32_t* ids = out.ids ? out.ids + c0 * k : nullptr;
            float* dists = out.dists ? out.dists + c0 * k : nullptr;
            uint32_t* counts = out.counts ? out.counts + c0 : nullptr;
            const unsigned grid = (unsigned)((outs + 255) / 256);
            if (filt) {
                gb::ExactList l{};
                l.query_filter = filt->query_filter ? filt->query_filter + c0 : nullptr;
                l.num_filters = filt->num_filters;
                l.error = w->d_error;
                return launch<gb::exact_write_kernel<true>>(grid, 256, 0, stream, &h->launches,
                                                            scan ? w->d_exact_lists.get() : nullptr, qc, k, 0, ids,
                                                            dists, counts, l);
            }
            return launch<gb::exact_write_kernel<false>>(grid, 256, 0, stream, &h->launches, w->d_exact_lists.get(), qc,
                                                         k, count, ids, dists, counts, gb::ExactList{});
        },
        filt);
}

// ---- exact range search (range_kernels.cuh) -----------------------------------------------------------------------
// The per-query inputs of a range call by id: skip (QUERY_ID_EXCLUDING: the query's own id, removed from its range in
// the count and the fill alike) and bad (a device call: the bad-id flags, whose queries count 0).
struct RangeIds {
    const uint32_t* skip;
    const int* bad;
};

// Enqueues a range call whatever its format: `call(q, fmt, ids)` queues its kernels for device query rows q.  Ids are
// read as elements first (enqueue_id_rows) and the call runs on those rows as ELEMENT queries; only a device call, whose
// ids no host has checked (`host_checked`), passes the bad-id flags.
template <class Call>
int enqueue_range_query(Handle* h, Workspace* w, const void* d_q, size_t nq, int fmt, bool host_checked,
                        cudaStream_t stream, Call&& call) {
    if (!by_id(fmt)) return call(d_q, fmt, RangeIds{nullptr, nullptr});
    const uint32_t* ids = static_cast<const uint32_t*>(d_q);
    const int rc = enqueue_id_rows(h, w, ids, nq, stream);
    if (rc) return rc;
    return call(w->d_id_rows.get(), (int)GRANNE_B200_QUERY_ELEMENT,
                RangeIds{fmt == GRANNE_B200_QUERY_ID_EXCLUDING ? ids : nullptr, host_checked ? nullptr : w->d_id_bad.get()});
}

gb::RangeArgs range_args(Workspace* w, size_t c0, uint64_t ns, uint64_t id_base, uint64_t ld, float radius,
                         const RangeIds& ri) {
    gb::RangeArgs a{};
    a.dists = w->d_exact_dists.get();
    a.ld = ld;
    a.nrows = ns;
    a.base = (uint32_t)id_base;
    a.radius = radius;
    a.skip = ri.skip ? ri.skip + c0 : nullptr;
    a.bad = ri.bad ? ri.bad + c0 : nullptr;
    return a;
}

dim3 range_grid(uint64_t ns, uint32_t qc) {
    const uint64_t rows = (uint64_t)gb::kRangeThreads * gb::kRangeRowsPerThread;
    return dim3((unsigned)((ns + rows - 1) / rows), qc);
}

// Enqueues the count of a range call: counts[q] = |R(q)| (u64, device memory) for nq queries (device memory, ELEMENT
// or RAW_F32).  With n > 0 the scan always runs, so a NaN distance sets kStatusNotFinite whatever the radius.
int enqueue_range_count(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, float radius,
                        const RangeIds& ri, uint64_t* counts, cudaStream_t stream) {
    GB_CUDA(cudaMemsetAsync(counts, 0, nq * 8, stream));
    auto none = [](size_t, uint32_t) { return (int)GRANNE_B200_OK; };
    return exact_scan(h, w, d_queries, nq, fmt, h->index_len > 0, stream, none,
                      [&](size_t c0, uint32_t qc, uint64_t ns, uint64_t id_base, uint64_t ld) {
                          return launch<gb::range_count_kernel>(range_grid(ns, qc), gb::kRangeThreads, 0, stream,
                                                                &h->launches,
                                                                range_args(w, c0, ns, id_base, ld, radius, ri),
                                                                reinterpret_cast<unsigned long long*>(counts) + c0);
                      },
                      none);
}

// Enqueues the fill of a range call: R(q) into the caller's segment [offsets[q], offsets[q + 1]) of ids / dists (device
// memory), sorted by (distance, id).  Per chunk the cursors start at the chunk's offsets, every slab's entries in range
// are emitted at them, and range_finish_kernel sorts each segment in place, or pads it and sets kStatusBadSegment when
// its length is not the query's count.
int enqueue_range_fill(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, float radius,
                       const RangeIds& ri, const uint64_t* d_offsets, uint32_t* ids, float* dists,
                       cudaStream_t stream) {
    const unsigned long long* offsets = reinterpret_cast<const unsigned long long*>(d_offsets);
    int rc = w->d_range_cursor.grow(std::min<size_t>(nq, gb::kExactMaxChunk), stream);
    if (rc) return rc;
    unsigned long long* cursor = w->d_range_cursor.get();
    return exact_scan(
        h, w, d_queries, nq, fmt, h->index_len > 0, stream,
        [&](size_t c0, uint32_t qc) {
            GB_CUDA(cudaMemcpyAsync(cursor, offsets + c0, (size_t)qc * 8, cudaMemcpyDeviceToDevice, stream));
            return (int)GRANNE_B200_OK;
        },
        [&](size_t c0, uint32_t qc, uint64_t ns, uint64_t id_base, uint64_t ld) {
            return launch<gb::range_emit_kernel>(range_grid(ns, qc), gb::kRangeThreads, 0, stream, &h->launches,
                                                 range_args(w, c0, ns, id_base, ld, radius, ri), cursor, offsets + c0,
                                                 ids, dists);
        },
        [&](size_t c0, uint32_t qc) {
            return launch<gb::range_finish_kernel>(qc, gb::kRangeSortThreads, 0, stream, &h->launches, offsets + c0,
                                                   cursor, ids, dists, w->d_error);
        });
}

// ---- two-stage search: angular_int traversal, exact re-rank (rerank_kernels.cuh) ---------------------------------
// The re-rank container is angular f32 rows (DistF32 engines) or a SumEmbeddings container (DistSum); one per handle.
// The checks on the handle before any container is read: an angular_int index without a re-rank container.
int check_rerank_target(const Handle* h) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    if (h->dev.kind != gb::kAngularI8)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "a re-rank container is attached to an angular_int index only");
    if (h->rerank.vectors)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "a re-rank container is already attached to this index");
    return GRANNE_B200_OK;
}

// The checks on the container: the index's width, and an element for every element of [0, Index::len).
int check_rerank_shape(const Handle* h, uint64_t n, uint64_t dim) {
    if (dim != h->dev.dim)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "the re-rank container must have the index's width");
    if (n < h->index_len)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "the re-rank container must cover every element of the index");
    return GRANNE_B200_OK;
}

// Stages h's re-rank container with stage_into(r, mem) (stage_dense or stage_sum into an empty view r and its owners
// mem).  It becomes visible to searches only once fully staged; a container that fails part-way frees its memory
// when mem goes out of scope.  The target check is repeated under the handle's attach lock, so that of two concurrent
// attaches one stages its container and the other fails.
template <class StageInto>
int stage_rerank(Handle* h, StageInto&& stage_into) {
    std::lock_guard<std::mutex> g(h->rerank_mu);
    int rc = check_rerank_target(h);
    if (rc) return rc;
    gb::DeviceIndex r{};
    Staged mem;
    if ((rc = stage_into(r, mem))) return rc;
    h->rerank = r;
    h->rerank_mem = std::move(mem);
    return GRANNE_B200_OK;
}

// Stages n angular f32 element rows as h's re-rank rows, laid out for the engine DistDispatch picks for their width.
int stage_rerank_rows(Handle* h, const uint8_t* rows, uint64_t n, uint32_t dim, bool device_src) {
    return stage_rerank(h, [&](gb::DeviceIndex& r, Staged& mem) {
        r.kind = gb::kAngularF32;
        const int rc = stage_dense(h, r, mem, rows, n, dim, device_src);
        r.num_elements = n;
        return rc;
    });
}

// Every host check of a SumEmbeddings re-rank container against h (h itself passed check_rerank_target): the images
// parse, every term id is a row of the table, the table is at most 4096 wide (parse_sum_container), it has the index's
// width, and there is an element for every element of the index.
int check_rerank_sum(const Handle* h, const void* el, size_t el_len, const void* emb, size_t emb_len,
                     gb::DenseView* ev, gb::SumElements* se) {
    if (!el || !emb) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements or embeddings buffer is null");
    const int rc = parse_sum_container(static_cast<const uint8_t*>(el), el_len, static_cast<const uint8_t*>(emb),
                                       emb_len, ev, se);
    if (rc) return rc;
    return check_rerank_shape(h, se->offsets.size() - 1, ev->dim);
}

// Drops h's re-rank container and its memory (the multi handle's attach undoes a partial attach with it).  The caller
// makes h's device current.
void release_rerank(Handle* h) {
    std::lock_guard<std::mutex> g(h->rerank_mu);
    h->rerank = gb::DeviceIndex{};
    h->rerank_mem = Staged{};
}

// validate_search's rules (raw or element queries only) plus the two-stage ones.
int validate_rerank(const Handle* h, const void* q, size_t nq, int fmt, uint32_t max_search, uint32_t c,
                    uint32_t k, const void* ids, const void* dists) {
    int rc = validate_search(h, q, nq, fmt, max_search, k, ids, dists, false);
    if (rc) return rc;
    if (fmt != GRANNE_B200_QUERY_RAW_F32)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "the two-stage search takes raw f32 queries");
    if (!h->rerank.vectors)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "no re-rank container is attached to this index");
    if (c == 0 || c > GRANNE_B200_RERANK_MAX_CANDIDATES)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "num_candidates must be in 1..1024");
    if (k > c) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "num_neighbors exceeds num_candidates");
    return GRANNE_B200_OK;
}

// Enqueues one two-stage search on `stream`: stage 1 is enqueue_search with k = C into the workspace's candidate
// block, stage 2 is rerank_kernel over h->rerank into the caller's outputs.  Stage 1 writes out.stats as search does.
int enqueue_rerank(Handle* h, Workspace* w, const void* d_queries, size_t nq, uint32_t max_search, uint32_t c,
                   uint32_t k, const QueryOut& out, cudaStream_t stream) {
    int rc = w->d_rerank.grow(2 * nq * c + nq, stream);
    if (rc) return rc;
    uint32_t* cand_ids = w->d_rerank.get();
    uint32_t* cand_counts = cand_ids + 2 * nq * c;
    if ((rc = enqueue_search(h, w, d_queries, nq, GRANNE_B200_QUERY_RAW_F32, max_search, c,
                             {cand_ids, reinterpret_cast<float*>(cand_ids + nq * c), cand_counts, out.stats}, stream)))
        return rc;
    const EngineTiles eng = engine_tiles(h->rerank);
    gb::RerankArgs a{};
    a.queries = static_cast<const float*>(d_queries);
    a.nq = nq;
    a.cand_ids = cand_ids;
    a.cand_counts = cand_counts;
    a.cand_stride = c;
    a.num_neighbors = k;
    a.out_ids = out.ids;
    a.out_dists = out.dists;
    a.out_counts = out.counts;
    a.work_counter = w->d_counters.get() + 6;  // zeroed with the search counters before stage 1, on this stream
    a.error_flag = w->d_error;
    a.tiles = eng.tiles;
    const size_t smem = gb::rerank_keys_offset(eng.base_smem) + (size_t)gb::rerank_key_slots(c) * 8;
    // the f32 engine for the width of angular rows, DistSum for a SumEmbeddings container (never the i8 engine: no
    // container is staged as angular_int)
    return DistDispatch::call(h->rerank, [&](auto e) {
        using Dist = typename decltype(e)::type;
        if constexpr (std::is_same<Dist, gb::DistI8>::value) {
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "re-rank container must be angular f32 rows or SumEmbeddings");
        } else {
            int occ = 0;
            const int err = resident_ctas<gb::rerank_kernel<Dist>>(h, smem, &occ);
            if (err) return err;
            if (occ < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "re-rank workspace exceeds shared memory");
            const unsigned grid = (unsigned)std::min<unsigned long long>(a.nq, (unsigned long long)occ * h->num_sms);
            return launch_warps<gb::rerank_kernel<Dist>>(h, grid, smem, stream, h->rerank, a);
        }
    });
}

// ---- diverse search: select_neighbors over candidate lists (diverse_kernels.cuh) ----------------------------------
constexpr const char* kDiverseStrideRule = "the candidate stride exceeds GRANNE_B200_DIVERSE_MAX_CANDIDATES (1024)";

// validate_search's rules with max_search <= GRANNE_B200_DIVERSE_MAX_CANDIDATES as part of the call's own rule.
int validate_diverse(const Handle* h, const void* q, size_t nq, int fmt, uint32_t max_search, uint32_t k,
                     const void* ids, const void* dists) {
    const char* rule = max_search == 0 ? kMaxSearchRule
                       : max_search > GRANNE_B200_DIVERSE_MAX_CANDIDATES
                           ? "max_search exceeds GRANNE_B200_DIVERSE_MAX_CANDIDATES (1024)"
                           : nullptr;
    return validate_batch(h, q, nq, fmt, k, ids, dists, rule);
}

// The rules of the standalone selection that read no handle, in the order they are reported: the handle is null;
// stride > GRANNE_B200_DIVERSE_MAX_CANDIDATES; nq above the batch limit; with nq > 0, a null candidate array (ids and
// distances only when stride > 0) or a null output (when k > 0).
int validate_select(const Handle* h, const void* ids, const void* dists, const void* counts, size_t nq,
                    uint32_t stride, uint32_t k, const void* out_ids, const void* out_dists) {
    int rc = validate_batch(h, counts, nq, GRANNE_B200_QUERY_RAW_F32, k, out_ids, out_dists,
                            stride > GRANNE_B200_DIVERSE_MAX_CANDIDATES ? kDiverseStrideRule : nullptr);
    if (rc) return rc;
    if (nq > 0 && stride > 0 && (!ids || !dists)) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null buffer");
    return GRANNE_B200_OK;
}

// The host check of nq caller lists in host memory: each count <= stride, its ids < Index::len and its distances
// ascending (no NaN).
int check_candidate_lists(const Handle* h, const uint32_t* ids, const float* dists, const uint32_t* counts, size_t nq,
                          uint32_t stride) {
    for (size_t q = 0; q < nq; ++q) {
        if (counts[q] > stride) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, kBadCandidatesRule);
        const uint32_t* id = ids + q * stride;
        const float* d = dists + q * stride;
        for (uint32_t t = 0; t < counts[q]; ++t)
            if (id[t] >= h->index_len || d[t] != d[t] || (t > 0 && !(d[t - 1] <= d[t])))
                return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, kBadCandidatesRule);
    }
    return GRANNE_B200_OK;
}

// Enqueues select_neighbors(list_q, k) for nq lists of up to `stride` candidates (device memory) over h's own container
// into `out` (ids | dists | counts in search_batch's layout) on `stream`.  `check`: the lists come from a caller, and
// the kernel checks them (kStatusBadCandidates).  Uses work counter word 7, which the call zeroed.
int enqueue_select(Handle* h, Workspace* w, const uint32_t* ids, const float* dists, const uint32_t* counts,
                   size_t nq, uint32_t stride, uint32_t k, bool check, const QueryOut& out, cudaStream_t stream) {
    const gb::DeviceIndex& d = h->dev;
    const EngineTiles eng = engine_tiles(d);
    gb::DiverseArgs a{};
    a.cand_ids = ids;
    a.cand_dists = dists;
    a.cand_counts = counts;
    a.cand_stride = stride;
    a.nq = nq;
    a.num_neighbors = k;
    a.check = check;
    a.len = h->index_len;
    a.out_ids = out.ids;
    a.out_dists = out.dists;
    a.out_counts = out.counts;
    a.work_counter = w->d_counters.get() + 7;
    a.error_flag = w->d_error;
    a.tiles = eng.tiles;
    const size_t smem = gb::diverse_list_offset(eng.base_smem) + gb::diverse_list_bytes(stride);
    return DistDispatch::call(d, [&](auto e) {
        constexpr auto kern = gb::diverse_kernel<typename decltype(e)::type>;
        int occ = 0;
        const int err = resident_ctas<kern>(h, smem, &occ);
        if (err) return err;
        if (occ < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "diverse selection exceeds shared memory");
        const unsigned grid = (unsigned)std::min<unsigned long long>(nq, (unsigned long long)occ * h->num_sms);
        return launch_warps<kern>(h, grid, smem, stream, d, a);
    });
}

// Enqueues one diverse search on `stream`: stage 1 is the query call's search with k = max_search (any query format;
// QUERY_ID_EXCLUDING drops the element itself from its candidates) into the workspace's candidate block, stage 2 is
// enqueue_select over those lists into the caller's outputs.  Stage 1 writes out.stats as search does.
int enqueue_diverse(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, uint32_t max_search,
                    uint32_t k, const QueryOut& out, bool host_checked, cudaStream_t stream) {
    int rc = w->d_rerank.grow(2 * nq * max_search + nq, stream);
    if (rc) return rc;
    uint32_t* cand_ids = w->d_rerank.get();
    float* cand_dists = reinterpret_cast<float*>(cand_ids + nq * max_search);
    uint32_t* cand_counts = cand_ids + 2 * nq * max_search;
    if ((rc = enqueue_query(h, w, d_queries, nq, fmt, max_search, {cand_ids, cand_dists, cand_counts, out.stats},
                            host_checked, stream, [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                return enqueue_search(h, w, q, nq, f, max_search, kk, o, stream);
                            })))
        return rc;
    return enqueue_select(h, w, cand_ids, cand_dists, cand_counts, nq, max_search, k, false, out, stream);
}

// ---- exact search within candidate lists (within_kernels.cuh) -----------------------------------------------------
// validate_exact's rules, then the lists' pointers: offsets when nq > 0 and, when the lists are in host memory, ids
// when offsets[nq] > 0 (a device call's kernels check a null ids pointer against the lists they are given).
int validate_within(const Handle* h, const void* q, size_t nq, int fmt, uint32_t k, const void* out_ids,
                    const void* out_dists, const uint64_t* offsets, const void* ids, bool host_lists) {
    const int rc = validate_exact(h, q, nq, fmt, k, out_ids, out_dists);
    if (rc) return rc;
    if (nq > 0 && !offsets) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "offsets is null");
    if (nq > 0 && host_lists && offsets[nq] > 0 && !ids) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "ids is null");
    return check_exclude_k(fmt, k, GRANNE_B200_EXACT_MAX_K);
}

// The host checks of nq lists in host memory: the shape of the offsets (which reads no handle), then every id
// against n.
int check_within_offsets(const uint64_t* offsets, size_t nq) {
    if (offsets[0] != 0) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "offsets must start at 0 and not decrease");
    for (size_t q = 0; q < nq; ++q)
        if (offsets[q + 1] < offsets[q])
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "offsets must start at 0 and not decrease");
    return GRANNE_B200_OK;
}
template <class Id>
int check_within_ids(const uint64_t* offsets, size_t nq, const Id* ids, uint64_t n) {
    for (uint64_t i = 0; i < offsets[nq]; ++i)
        if ((uint64_t)ids[i] >= n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "candidate id >= Index::len");
    return GRANNE_B200_OK;
}

// The argument rules of the range calls, in the order they are reported: validate_batch's (a NaN radius as the call's
// own rule), then, when nq > 0, counts NULL (count) or offsets NULL (fill).  None reads the handle.
int validate_range(const Handle* h, const void* q, size_t nq, int fmt, float radius, const void* counts,
                   const uint64_t* offsets, bool fill) {
    const int rc = validate_batch(h, q, nq, fmt, 0, nullptr, nullptr, radius != radius ? "radius is NaN" : nullptr);
    if (rc) return rc;
    if (nq > 0 && !fill && !counts) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "counts is null");
    if (nq > 0 && fill && !offsets) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "offsets is null");
    return GRANNE_B200_OK;
}

// The host checks of a host fill's offsets and outputs: their shape, then ids / dists NULL with offsets[nq] > 0.
int check_range_outputs(const uint64_t* offsets, size_t nq, const void* ids, const void* dists) {
    const int rc = check_within_offsets(offsets, nq);
    if (rc) return rc;
    if (offsets[nq] > 0 && (!ids || !dists)) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null buffer");
    return GRANNE_B200_OK;
}

// Enqueues one exact search within lists on `stream`: nq queries (device memory, the caller's format), their lists
// d_offsets / d_ids (device memory), results in search_batch's layout.  Query chunks of at most kExactMaxChunk: the
// segments kernel, then within_kernel over the chunk's segments, then the rows of the lists of other than one segment.
// A NaN distance sets kStatusNotFinite in w->d_error, a bad list kStatusBadList.
int enqueue_within(Handle* h, Workspace* w, const void* d_queries, size_t nq, int fmt, const uint64_t* d_offsets,
                   const uint32_t* d_ids, uint32_t k, const QueryOut& out, cudaStream_t stream) {
    const gb::DeviceIndex& d = h->dev;
    const size_t in_row = query_row_bytes(d.kind, d.dim, fmt);
    const size_t qc_max = std::min<size_t>(nq, gb::kExactMaxChunk);
    int rc;
    if ((rc = w->d_within.grow(qc_max * k + qc_max + 2, stream)) || (rc = w->d_within_flags.grow(2 * qc_max, stream)))
        return rc;
    unsigned long long* lists = w->d_within.get();
    unsigned long long* prefix = lists + qc_max * k;
    unsigned long long* counter = prefix + qc_max + 1;
    int* locks = w->d_within_flags.get();
    int* qflags = locks + qc_max;
    const EngineTiles eng = engine_tiles(d);
    const size_t smem = gb::rerank_keys_offset(eng.base_smem) + (size_t)gb::within_key_slots(k) * 8;
    return DistDispatch::call(d, [&](auto e) {
        using Dist = typename decltype(e)::type;
        constexpr auto kern = gb::within_kernel<Dist>;
        int occ = 0;
        int err = resident_ctas<kern>(h, smem, &occ);
        if (err) return err;
        if (occ < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "exact search within lists exceeds shared memory");
        for (size_t c0 = 0; c0 < nq; c0 += gb::kExactMaxChunk) {
            const uint32_t qc = (uint32_t)std::min<size_t>(gb::kExactMaxChunk, nq - c0);
            const unsigned long long* offs = reinterpret_cast<const unsigned long long*>(d_offsets) + c0;
            if ((err = launch<gb::within_segments_kernel>(1, gb::kExactMaxChunk, 0, stream, &h->launches, offs, qc,
                                                          c0 == 0, d_ids, prefix, locks, qflags, counter, w->d_error)))
                return err;
            if (k) GB_CUDA(cudaMemsetAsync(lists, 0xFF, (size_t)qc * k * 8, stream));
            gb::WithinArgs a{};
            a.queries = static_cast<const uint8_t*>(d_queries) + c0 * in_row;
            a.query_format = fmt;
            a.nq = qc;
            a.offsets = offs;
            a.ids = d_ids;
            a.len = h->index_len;
            a.num_neighbors = k;
            a.seg_prefix = prefix;
            a.lists = lists;
            a.locks = locks;
            a.qflags = qflags;
            a.work_counter = counter;
            a.out_ids = out.ids ? out.ids + c0 * k : nullptr;
            a.out_dists = out.dists ? out.dists + c0 * k : nullptr;
            a.out_counts = out.counts ? out.counts + c0 : nullptr;
            a.error_flag = w->d_error;
            a.tiles = eng.tiles;
            if ((err = launch_warps<kern>(h, (unsigned)occ * h->num_sms, smem, stream, d, a)) ||
                (err = launch<gb::within_write_kernel>(qc, 128, 0, stream, &h->launches, lists, prefix, qflags, k,
                                                       a.out_ids, a.out_dists, a.out_counts)))
                return err;
        }
        return (int)GRANNE_B200_OK;
    });
}

// ---- filtered search (search_kernel<Dist, R, true>) -----------------------------------------------------------------
// The rules of a filtered call that read no handle, in the order they are reported: validate_batch's, with
// max_search >= 1 and k <= GRANNE_B200_EXACT_MAX_K as the call's own (the exact filtered call: k only); then, when
// nq > 0, the filters' pointer and count, and QUERY_ID_EXCLUDING's k (check_filter_args).
int check_filter_args(size_t nq, int fmt, uint32_t k, const void* filters, uint32_t num_filters) {
    if (nq > 0 && (!filters || num_filters == 0))
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "filters is null or num_filters is 0");
    return check_exclude_k(fmt, k, GRANNE_B200_EXACT_MAX_K);
}
int validate_filtered(const Handle* h, const void* q, size_t nq, int fmt, uint32_t max_search, uint32_t k,
                      const void* ids, const void* dists, const void* filters, uint32_t num_filters) {
    const int rc = validate_batch(h, q, nq, fmt, k, ids, dists,
                                  max_search == 0 ? kMaxSearchRule : k > GRANNE_B200_EXACT_MAX_K ? kExactKRule : nullptr);
    return rc ? rc : check_filter_args(nq, fmt, k, filters, num_filters);
}
// The exact filtered call's: exact_search_batch's, then the filters' (there is no max_search).
int validate_exact_filtered(const Handle* h, const void* q, size_t nq, int fmt, uint32_t k, const void* ids,
                            const void* dists, const void* filters, uint32_t num_filters) {
    const int rc = validate_exact(h, q, nq, fmt, k, ids, dists);
    return rc ? rc : check_filter_args(nq, fmt, k, filters, num_filters);
}

// A bitmap of filter_words words must hold a bit for every id in [0, span).
int check_filter_words(uint64_t filter_words, uint64_t span) {
    if (filter_words < (span + 31) / 32)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "filter_words is less than ceil(Index::len / 32)");
    return GRANNE_B200_OK;
}

// The host check of a host call's query_filter (null: every query uses filter 0).
int check_query_filter(const uint32_t* query_filter, size_t nq, uint32_t num_filters) {
    for (size_t q = 0; query_filter && q < nq; ++q)
        if (query_filter[q] >= num_filters)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "a query_filter entry is >= num_filters");
    return GRANNE_B200_OK;
}

// A filtered search from host buffers (arguments checked, nq > 0), the filters and query_filter copied up for the call
// only (with_call_inputs).  bit_base: the bit of element 0 in the bitmaps (a range-partitioned shard reads the global
// bitmap).
int search_filtered_host(Handle* h, const void* queries, size_t nq, int fmt, uint32_t max_search, uint32_t k,
                         const uint32_t* filters, uint32_t num_filters, uint64_t filter_words,
                         const uint32_t* query_filter, uint64_t bit_base, uint32_t* out_ids, float* out_dists,
                         uint32_t* out_counts, uint64_t* out_stats) {
    return host_batch(h, queries, nq, fmt, k, out_ids, out_dists, out_counts, out_stats,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          const HostInput in[] = {{filters, (size_t)num_filters * filter_words * 4},
                                                  {query_filter, query_filter ? nq * 4 : 0}};
                          return with_call_inputs(stream, in, [&](const void* const* d) {
                              const DeviceFilters f{static_cast<const uint32_t*>(d[0]),
                                                    query_filter ? static_cast<const uint32_t*>(d[1]) : nullptr,
                                                    filter_words, num_filters, bit_base};
                              return enqueue_query(h, w, w->d_queries.get(), nq, fmt, k, out, true, stream,
                                                   [&](const void* q, int f2, uint32_t kk, const QueryOut& o) {
                                                       return enqueue_search(h, w, q, nq, f2, max_search, kk, o,
                                                                             stream, nullptr, nullptr, &f);
                                                   });
                          });
                      });
}

// An exact filtered search from host buffers (arguments checked, nq > 0), its inputs copied up like
// search_filtered_host's.
int exact_filtered_host(Handle* h, const void* queries, size_t nq, int fmt, uint32_t k, const uint32_t* filters,
                        uint32_t num_filters, uint64_t filter_words, const uint32_t* query_filter, uint64_t bit_base,
                        uint32_t* out_ids, float* out_dists, uint32_t* out_counts) {
    return host_batch(h, queries, nq, fmt, k, out_ids, out_dists, out_counts, nullptr,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          const HostInput in[] = {{filters, (size_t)num_filters * filter_words * 4},
                                                  {query_filter, query_filter ? nq * 4 : 0}};
                          return with_call_inputs(stream, in, [&](const void* const* d) {
                              const DeviceFilters f{static_cast<const uint32_t*>(d[0]),
                                                    query_filter ? static_cast<const uint32_t*>(d[1]) : nullptr,
                                                    filter_words, num_filters, bit_base};
                              return enqueue_query(h, w, w->d_queries.get(), nq, fmt, k, out, true, stream,
                                                   [&](const void* q, int f2, uint32_t kk, const QueryOut& o) {
                                                       return enqueue_exact(h, w, q, nq, f2, kk, o, stream, &f);
                                                   });
                          });
                      });
}

}  // namespace

// ---- GranneBuilder (src/index/mod.rs:295-531, 645-960) on the device ---------------------------------------------
struct granne_b200_builder {
    std::unique_ptr<Handle> h;  // search view over the layers built so far (+ the one under construction)
    granne_b200_build_config cfg{};
    uint32_t stride = 0;  // physical row stride (node_width rounded up to 8)
    std::unique_ptr<Workspace> ws;
    // batch scratch
    Buffer<uint32_t> d_ids;
    Buffer<uint32_t> d_cand_ids;
    Buffer<float> d_cand_d;
    Buffer<uint32_t> d_cand_cnt;
    Buffer<int> d_locks;
    Buffer<unsigned int> d_counter;
};

namespace {

using Builder = granne_b200_builder;

// index_elements (:716-802) for the layer at dev.layer_rows[num_layers-1]
int builder_index_elements(Builder* b, uint32_t layer_m, uint32_t ef, uint64_t already, uint64_t num, bool reinsert) {
    Handle* h = b->h.get();
    gb::DeviceIndex& d = h->dev;
    const int cur = d.num_layers - 1;
    uint32_t* rows = const_cast<uint32_t*>(d.layer_rows[cur]);
    cudaStream_t stream = b->ws->stream.get();
    if (make_plan(h, ef).smem == 0) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search too large");
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
    int rc;
    if ((rc = b->d_ids.grow(max_batch, stream)) || (rc = b->d_cand_ids.grow(max_batch * ef, stream)) ||
        (rc = b->d_cand_d.grow(max_batch * ef, stream)) || (rc = b->d_cand_cnt.grow(max_batch, stream)) ||
        (rc = b->d_locks.grow(num, stream)) || (rc = b->d_counter.grow(4, stream)))
        return rc;
    GB_CUDA(cudaMemsetAsync(b->d_locks.get(), 0, num * sizeof(int), stream));
    // shared memory: the engine's SmemLayout, then the link scratch for ef candidates (link) or a node's row (prune)
    const uint32_t nn = b->cfg.num_neighbors;
    const EngineTiles eng = engine_tiles(d);
    const size_t link_smem = gb::LinkLayout<size_t>(eng.base_smem, gb::link_cand_cap(ef, nn), nn).end;
    const size_t prune_smem = gb::LinkLayout<size_t>(eng.base_smem, gb::link_cand_cap(0, nn), nn).end;
    gb::BuildArgs prune{};
    prune.rows = rows;
    prune.stride = b->stride;
    prune.node_width = nn;
    prune.max_neighbors = layer_m;
    prune.tiles = eng.tiles;
    prune.work_counter = b->d_counter.get();
    prune.num_nodes = (uint32_t)num;
    gb::BuildArgs link = prune;  // the prune pass's arguments and a batch's candidates
    link.ids = b->d_ids.get();
    link.cand_ids = b->d_cand_ids.get();
    link.cand_dists = b->d_cand_d.get();
    link.cand_counts = b->d_cand_cnt.get();
    link.cand_stride = ef;
    link.locks = b->d_locks.get();
    uint64_t pos = 0;
    while (pos < total) {
        // nodes already linked into this layer: a batch never exceeds 1/16 of them (its members do not see each other)
        const uint64_t present = reinsert ? num : first + pos;
        const uint64_t bsz = std::min<uint64_t>(std::min<uint64_t>(max_batch, std::max<uint64_t>(1, present / 16)), total - pos);
        const uint32_t start = reinsert ? (uint32_t)(num - 1 - pos) : (uint32_t)(first + pos);
        if ((rc = launch<gb::iota_kernel>((unsigned)((bsz + 255) / 256), 256, 0, stream, &h->launches, b->d_ids.get(),
                                          (uint32_t)bsz, start, reinsert ? -1 : 1)))
            return rc;
        // candidates = search_for_neighbors(layer, prev_layers.search(e,1,1), e, max_search) (:819-820)
        GB_CUDA(cudaMemsetAsync(b->ws->d_counters.get(), 0, kSearchCounterBytes, stream));
        rc = enqueue_search(h, b->ws.get(), b->d_ids.get(), bsz, gb::kQueryById, ef, ef,
                            {b->d_cand_ids.get(), b->d_cand_d.get(), b->d_cand_cnt.get(), nullptr}, stream);
        if (rc) return rc;
        GB_CUDA(cudaMemsetAsync(b->d_counter.get(), 0, 16, stream));
        link.n_batch = (uint32_t)bsz;
        const unsigned grid = (unsigned)std::min<uint64_t>(bsz, link_warps);
        rc = DistDispatch::call(d, [&](auto e) {
            return launch_warps<gb::build_link_kernel<typename decltype(e)::type>>(h, grid, link_smem, stream, d, link);
        });
        if (rc) return rc;
        pos += bsz;
    }
    // limit number of neighbors (:794-797)
    GB_CUDA(cudaMemsetAsync(b->d_counter.get(), 0, 16, stream));
    const unsigned grid = (unsigned)std::min<uint64_t>(num, (uint64_t)h->num_sms * 8);
    rc = DistDispatch::call(d, [&](auto e) {
        return launch_warps<gb::build_prune_kernel<typename decltype(e)::type>>(h, grid, prune_smem, stream, d, prune);
    });
    if (rc) return rc;
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
    Buffer<uint32_t> mem;
    int rc = dev_alloc(&mem, (size_t)num * b->stride);
    if (rc) return rc;
    uint32_t* grown = mem.get();
    cudaStream_t stream = b->ws->stream.get();
    if ((rc = launch<gb::fill_u32_kernel>(h->num_sms * 4, 256, 0, stream, &h->launches, grown,
                                          (unsigned long long)num * b->stride, gb::kUnusedId)))
        return rc;
    if (have) GB_CUDA(cudaMemcpyAsync(grown, d.layer_rows[cur], (size_t)have * b->stride * 4, cudaMemcpyDeviceToDevice, stream));
    // the replaced rows stay alive until the copy out of them has completed: the first pass below synchronises the
    // stream before it returns OK, and a failed pass is synchronised here
    Staged::Slot old = std::move(h->dev_mem.layer_rows[cur]);
    d.layer_rows[cur] = stage(&h->dev_mem.layer_rows[cur], std::move(mem));
    d.layer_len[cur] = num;
    h->layer_max_degree[cur] = b->cfg.num_neighbors;
    finish_handle(h);
    if ((rc = builder_index_elements(b, layer_m, b->cfg.max_search, have, num, false))) {
        cudaStreamSynchronize(stream);
        return rc;
    }
    old = {};  // the copy is done
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
        h->dev_mem.layer_rows[l] = l ? h->dev_mem.layer_rows[l - 1] : Staged::Slot{};
        d.layer_len[l] = l ? d.layer_len[l - 1] : 0;
        d.layer_width[l] = b->stride;
        d.num_layers = l + 1;
        h->layer_max_degree.push_back(b->cfg.num_neighbors);
        finish_handle(h);
        if ((rc = builder_index_last_layer(b, num_elements))) return rc;
    }
    return GRANNE_B200_OK;
}

// GranneBuilder::from_bytes (:440-451): every layer of `graph` becomes a layer of the builder, in its own allocation
// at the builder's row stride.  Row i keeps node i's ids in stored (ascending) order, truncated to the first
// num_neighbors (the lowest ids, not the nearest) or padded with UNUSED, like `neighbors.resize(num_neighbors,
// UNUSED)`.  The link and prune kernels compute the distances of whatever a row holds, so they need no other order.
int builder_load_layers(Builder* b, const gb::HostGraph& graph) {
    Handle* h = b->h.get();
    gb::DeviceIndex& d = h->dev;
    const uint32_t m = b->cfg.num_neighbors;
    std::vector<uint32_t> rows;
    for (size_t l = 0; l < graph.layers.size(); ++l) {
        const gb::HostLayer& L = graph.layers[l];
        if (L.num_nodes > d.num_elements)
            return fail(GRANNE_B200_ERR_FORMAT, "index refers to more elements than the container holds");
        const uint32_t keep = std::min(m, L.width);  // decoded rows are padded with UNUSED up to L.width
        rows.assign((size_t)L.num_nodes * b->stride, gb::kUnusedId);
        for (uint64_t i = 0; i < L.num_nodes; ++i)
            std::copy_n(L.rows.data() + i * L.width, keep, rows.data() + i * b->stride);
        const int rc = stage_layer(h, (int)l, rows.data(), L.num_nodes, b->stride);
        if (rc) return rc;
        h->layer_max_degree.push_back(m);
    }
    d.num_layers = (int)graph.layers.size();
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
    return guarded([&] {
        return open_impl(static_cast<const uint8_t*>(index_bytes), index_len, element_kind,
                         static_cast<const uint8_t*>(elements_bytes), elements_len,
                         static_cast<const uint8_t*>(embeddings_bytes), embeddings_len, device, out);
    });
}

int granne_b200_open_device_elements(const void* index_bytes, size_t index_len, int element_kind,
                                     const void* d_element_rows, uint64_t num_elements, uint32_t dim, int device,
                                     granne_b200_index** out) {
    return guarded([&] {
        if (!d_element_rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
        return open_impl(static_cast<const uint8_t*>(index_bytes), index_len, element_kind, nullptr, 0, nullptr, 0,
                         device, out, d_element_rows, num_elements, dim);
    });
}

int granne_b200_open_files(const char* index_path, int element_kind, const char* elements_path,
                           const char* embeddings_path, int device, granne_b200_index** out) {
    return guarded([&] {
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
    });
}

void granne_b200_close(granne_b200_index* h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    cudaDeviceSynchronize();
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
// Counts each allocation once: a builder's new layer shares its rows with the layer above until it grows.
uint64_t granne_b200_device_bytes(const granne_b200_index* h) {
    if (!h) return 0;
    std::lock_guard<std::mutex> g(h->rerank_mu);
    const void* counted[2 * (3 + gb::kMaxLayers)];
    size_t n = 0;
    uint64_t bytes = 0;
    auto count = [&](const Staged::Slot& s) {
        if (!s.mem || std::find(counted, counted + n, s.mem.get()) != counted + n) return;
        counted[n++] = s.mem.get();
        bytes += s.bytes;
    };
    for (const Staged* m : {&h->dev_mem, &h->rerank_mem}) {
        for (const Staged::Slot* s : {&m->vectors, &m->sum_offsets, &m->sum_terms}) count(*s);
        for (const Staged::Slot& s : m->layer_rows) count(s);
    }
    return bytes;
}

int granne_b200_get_neighbors(const granne_b200_index* h, uint64_t idx, uint64_t layer, uint32_t* out, size_t cap,
                              size_t* out_n) {
    if (!h || !out_n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (layer >= (uint64_t)h->dev.num_layers || idx >= h->dev.layer_len[layer])
        return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "node or layer out of range");
    return guarded([&] {
        GB_DEVICE(h->device);
        const uint32_t w = h->dev.layer_width[layer];
        std::vector<uint32_t> row(w);
        GB_CUDA(cudaMemcpy(row.data(), h->dev.layer_rows[layer] + idx * w, w * 4, cudaMemcpyDeviceToHost));
        size_t n = 0;
        while (n < w && row[n] != gb::kUnusedId) ++n;
        *out_n = n;
        for (size_t i = 0; i < n && i < cap && out; ++i) out[i] = row[i];
        return GRANNE_B200_OK;
    });
}

int granne_b200_get_element(const granne_b200_index* hc, uint64_t idx, void* out) {
    granne_b200_index* h = const_cast<granne_b200_index*>(hc);
    if (!h || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (idx >= h->dev.num_elements) return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "element index out of range");
    return guarded([&] {
        GB_DEVICE(h->device);
        const size_t bytes = h->dev.kind == gb::kAngularI8 ? h->dev.dim : (size_t)h->dev.dim * 4;
        Buffer<uint8_t> d;
        int rc = d.grow(bytes, nullptr);
        if (rc) return rc;
        if ((rc = launch<gb::get_element_kernel>(1, 32, 0, nullptr, &h->launches, h->dev, idx, d.get()))) return rc;
        GB_CUDA(cudaMemcpy(out, d.get(), bytes, cudaMemcpyDeviceToHost));
        return GRANNE_B200_OK;
    });
}

int granne_b200_get_elements(granne_b200_index* h, const uint32_t* ids, size_t n, void* out) {
    if (!h || (n && (!ids || !out))) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    int rc = check_element_ids(h, ids, n);
    if (rc || n == 0) return rc;
    return guarded([&] {
        GB_DEVICE(h->device);
        std::unique_ptr<Workspace> ws;
        int rc = ws_acquire(h, &ws);
        if (rc) return rc;
        Workspace* w = ws.get();
        const int status = [&] {
            cudaStream_t stream = w->stream.get();
            const size_t bytes = n * query_row_bytes(h->dev.kind, h->dev.dim, GRANNE_B200_QUERY_ELEMENT);
            int rc;
            if ((rc = w->d_queries.grow(n * 4, stream)) || (rc = w->d_id_rows.grow(std::max<size_t>(bytes, 16), stream)))
                return rc;
            GB_CUDA(cudaMemcpyAsync(w->d_queries.get(), ids, n * 4, cudaMemcpyHostToDevice, stream));
            const size_t smem = h->dev.kind == gb::kSumEmbeddings ? (size_t)h->dev.dim * 4 : 0;
            if ((rc = launch<gb::get_elements_kernel>((unsigned)std::min<uint64_t>(n, (uint64_t)h->num_sms * 32), 32, smem,
                                                      stream, &h->launches, h->dev,
                                                      reinterpret_cast<const uint32_t*>(w->d_queries.get()), n,
                                                      h->dev.num_elements, w->d_id_rows.get(), nullptr, w->d_error)))
                return rc;
            GB_CUDA(cudaMemcpyAsync(out, w->d_id_rows.get(), bytes, cudaMemcpyDeviceToHost, stream));
            GB_CUDA(cudaStreamSynchronize(stream));
            return (int)GRANNE_B200_OK;
        }();
        ws_release(h, std::move(ws));
        return status;
    });
}

int granne_b200_get_elements_device(granne_b200_index* h, const uint32_t* d_ids, size_t n, void* d_out,
                                    void* cuda_stream) {
    if (!h || (n && (!d_ids || !d_out))) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (n == 0) return GRANNE_B200_OK;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        const size_t smem = h->dev.kind == gb::kSumEmbeddings ? (size_t)h->dev.dim * 4 : 0;
        return launch<gb::get_elements_kernel>((unsigned)std::min<uint64_t>(n, (uint64_t)h->num_sms * 32), 32, smem,
                                               stream, &h->launches, h->dev, d_ids, n, h->dev.num_elements, d_out,
                                               nullptr, w->d_error);
    });
}

static int search_device_impl(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                              uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                              uint32_t* d_out_counts, uint64_t* d_out_stats, void* cuda_stream,
                              const granne_b200_peer_gather* pg) {
    int rc = validate_search(h, d_queries, nq, query_format, max_search, num_neighbors, pg ? (void*)pg : d_out_ids,
                             pg ? (void*)pg : d_out_dists, !pg);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, UINT32_MAX))) return rc;
    if (pg) {
        if (pg->n_peers < 1 || pg->n_peers > GRANNE_B200_MAX_PEERS || pg->my_rank >= pg->n_peers)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "peer gather: n_peers must be 1..8 and my_rank < n_peers");
        for (uint32_t p = 0; p < pg->n_peers; ++p)
            if (!pg->ids[p] || !pg->dists[p] || !pg->flags[p])
                return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "peer gather: null peer pointer");
    }
    if (nq == 0 && !pg) return GRANNE_B200_OK;
    if (nq == 0)  // nothing to store, but the peers wait for this call's sequence number all the same
        return guarded([&] {
            GB_DEVICE(h->device);
            return launch<gb::publish_seq_kernel>(1, 1, 0, static_cast<cudaStream_t>(cuda_stream), &h->launches,
                                                  device_gather(*pg, nullptr));
        });
    return device_batch(h, cuda_stream, true, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_query(h, w, d_queries, nq, query_format, num_neighbors,
                             {d_out_ids, d_out_dists, d_out_counts, d_out_stats}, false, stream,
                             [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                 return enqueue_search(h, w, q, nq, f, max_search, kk, o, stream, pg);
                             });
    });
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
    return guarded([&] {
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
        return GRANNE_B200_OK;
    });
}

int granne_b200_stream_status_of(granne_b200_index* h, void* cuda_stream) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    return guarded([&] {
        GB_DEVICE(h->device);
        cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
        GB_CUDA(cudaStreamSynchronize(stream));
        std::lock_guard<std::mutex> g(h->pool_mu);
        auto it = h->stream_ws.find(stream);
        if (it == h->stream_ws.end()) return (int)GRANNE_B200_OK;
        int e[4] = {0, 0, 0, 0};
        GB_CUDA(cudaMemcpy(e, it->second->d_error, sizeof(e), cudaMemcpyDeviceToHost));
        GB_CUDA(cudaMemset(it->second->d_error, 0, sizeof(e)));
        return error_from_bits(e[0]);
    });
}

int granne_b200_stream_status(granne_b200_index* h) {
    if (!h) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index handle is null");
    return guarded([&] {
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
    });
}

int granne_b200_search_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                             uint32_t max_search, uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                             uint32_t* out_counts, uint64_t* out_stats) {
    int rc = validate_search(h, queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, UINT32_MAX))) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    if ((rc = check_host_query_ids(h, queries, nq, query_format))) return rc;
    return host_batch(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts, out_stats,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          return enqueue_query(h, w, w->d_queries.get(), nq, query_format, num_neighbors, out, true,
                                               stream, [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                                   return enqueue_search(h, w, q, nq, f, max_search, kk, o, stream);
                                               });
                      });
}

int granne_b200_exact_search_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                   uint32_t num_neighbors, uint32_t* out_ids, float* out_dists, uint32_t* out_counts) {
    int rc = validate_exact(h, queries, nq, query_format, num_neighbors, out_ids, out_dists);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, GRANNE_B200_EXACT_MAX_K))) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    if ((rc = check_host_query_ids(h, queries, nq, query_format))) return rc;
    return host_batch(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts, nullptr,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          return enqueue_query(h, w, w->d_queries.get(), nq, query_format, num_neighbors, out, true,
                                               stream, [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                                   return enqueue_exact(h, w, q, nq, f, kk, o, stream);
                                               });
                      });
}

int granne_b200_exact_search_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                          uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                          uint32_t* d_out_counts, void* cuda_stream) {
    int rc = validate_exact(h, d_queries, nq, query_format, num_neighbors, d_out_ids, d_out_dists);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, GRANNE_B200_EXACT_MAX_K))) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_query(h, w, d_queries, nq, query_format, num_neighbors,
                             {d_out_ids, d_out_dists, d_out_counts, nullptr}, false, stream,
                             [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                 return enqueue_exact(h, w, q, nq, f, kk, o, stream);
                             });
    });
}

int granne_b200_exact_search_within_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                          const uint64_t* offsets, const uint32_t* ids, uint32_t num_neighbors,
                                          uint32_t* out_ids, float* out_dists, uint32_t* out_counts) {
    int rc = validate_within(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, offsets, ids, true);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    if ((rc = check_within_offsets(offsets, nq)) || (rc = check_within_ids(offsets, nq, ids, h->index_len)) ||
        (rc = check_host_query_ids(h, queries, nq, query_format)))
        return rc;
    return host_batch(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts, nullptr,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          const HostInput in[] = {{offsets, (nq + 1) * 8}, {ids, offsets[nq] * 4}};
                          return with_call_inputs(stream, in, [&](const void* const* d) {
                              return enqueue_query(
                                  h, w, w->d_queries.get(), nq, query_format, num_neighbors, out, true, stream,
                                  [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                      return enqueue_within(h, w, q, nq, f, static_cast<const uint64_t*>(d[0]),
                                                            static_cast<const uint32_t*>(d[1]), kk, o, stream);
                                  });
                          });
                      });
}

int granne_b200_exact_search_within_batch_device(granne_b200_index* h, const void* d_queries, size_t nq,
                                                 int query_format, const uint64_t* d_offsets, const uint32_t* d_ids,
                                                 uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                                 uint32_t* d_out_counts, void* cuda_stream) {
    int rc = validate_within(h, d_queries, nq, query_format, num_neighbors, d_out_ids, d_out_dists, d_offsets, d_ids,
                             false);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_query(h, w, d_queries, nq, query_format, num_neighbors,
                             {d_out_ids, d_out_dists, d_out_counts, nullptr}, false, stream,
                             [&](const void* q, int f, uint32_t kk, const QueryOut& o) {
                                 return enqueue_within(h, w, q, nq, f, d_offsets, d_ids, kk, o, stream);
                             });
    });
}

int granne_b200_exact_range_count(granne_b200_index* h, const void* queries, size_t nq, int query_format, float radius,
                                  uint64_t* counts) {
    int rc = validate_range(h, queries, nq, query_format, radius, counts, nullptr, false);
    if (rc || nq == 0) return rc;
    if ((rc = check_host_query_ids(h, queries, nq, query_format))) return rc;
    // the nq u64 counts fill the ids and dists columns of a result block of nq entries (2 nq words)
    uint32_t* words = reinterpret_cast<uint32_t*>(counts);
    return host_batch_entries(h, queries, nq, query_format, nq, words, reinterpret_cast<float*>(words + nq), nullptr,
                              nullptr, [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                                  return enqueue_range_query(
                                      h, w, w->d_queries.get(), nq, query_format, true, stream,
                                      [&](const void* q, int f, const RangeIds& ri) {
                                          return enqueue_range_count(h, w, q, nq, f, radius, ri,
                                                                     reinterpret_cast<uint64_t*>(out.ids), stream);
                                      });
                              });
}

int granne_b200_exact_range_count_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                         float radius, uint64_t* d_counts, void* cuda_stream) {
    int rc = validate_range(h, d_queries, nq, query_format, radius, d_counts, nullptr, false);
    if (rc || nq == 0) return rc;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_range_query(h, w, d_queries, nq, query_format, false, stream,
                                   [&](const void* q, int f, const RangeIds& ri) {
                                       return enqueue_range_count(h, w, q, nq, f, radius, ri, d_counts, stream);
                                   });
    });
}

int granne_b200_exact_range_search(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                   float radius, const uint64_t* offsets, uint32_t* ids, float* dists) {
    int rc = validate_range(h, queries, nq, query_format, radius, nullptr, offsets, true);
    if (rc || nq == 0) return rc;
    if ((rc = check_range_outputs(offsets, nq, ids, dists)) ||
        (rc = check_host_query_ids(h, queries, nq, query_format)))
        return rc;
    return host_batch_entries(h, queries, nq, query_format, offsets[nq], ids, dists, nullptr, nullptr,
                              [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                                  const HostInput in[] = {{offsets, (nq + 1) * 8}};
                                  return with_call_inputs(stream, in, [&](const void* const* d) {
                                      return enqueue_range_query(
                                          h, w, w->d_queries.get(), nq, query_format, true, stream,
                                          [&](const void* q, int f, const RangeIds& ri) {
                                              return enqueue_range_fill(h, w, q, nq, f, radius, ri,
                                                                        static_cast<const uint64_t*>(d[0]), out.ids,
                                                                        out.dists, stream);
                                          });
                                  });
                              });
}

int granne_b200_exact_range_search_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                          float radius, const uint64_t* d_offsets, uint32_t* d_ids, float* d_dists,
                                          void* cuda_stream) {
    int rc = validate_range(h, d_queries, nq, query_format, radius, nullptr, d_offsets, true);
    if (rc || nq == 0) return rc;
    // without both outputs every segment must be empty (the kernels flag any other)
    uint32_t* ids = d_ids && d_dists ? d_ids : nullptr;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_range_query(h, w, d_queries, nq, query_format, false, stream,
                                   [&](const void* q, int f, const RangeIds& ri) {
                                       return enqueue_range_fill(h, w, q, nq, f, radius, ri, d_offsets, ids,
                                                                 ids ? d_dists : nullptr, stream);
                                   });
    });
}

int granne_b200_search_filtered_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                      uint32_t max_search, uint32_t num_neighbors, const uint32_t* filters,
                                      uint32_t num_filters, uint64_t filter_words, const uint32_t* query_filter,
                                      uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint64_t* out_stats) {
    int rc = validate_filtered(h, queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists, filters,
                               num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, h->index_len)) ||
        (rc = check_query_filter(query_filter, nq, num_filters)) ||
        (rc = check_host_query_ids(h, queries, nq, query_format)))
        return rc;
    return search_filtered_host(h, queries, nq, query_format, max_search, num_neighbors, filters, num_filters,
                                filter_words, query_filter, 0, out_ids, out_dists, out_counts, out_stats);
}

int granne_b200_search_filtered_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                             uint32_t max_search, uint32_t num_neighbors, const uint32_t* d_filters,
                                             uint32_t num_filters, uint64_t filter_words,
                                             const uint32_t* d_query_filter, uint32_t* d_out_ids, float* d_out_dists,
                                             uint32_t* d_out_counts, uint64_t* d_out_stats, void* cuda_stream) {
    int rc = validate_filtered(h, d_queries, nq, query_format, max_search, num_neighbors, d_out_ids, d_out_dists,
                               d_filters, num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, h->index_len))) return rc;
    return device_batch(h, cuda_stream, true, [&](Workspace* w, cudaStream_t stream) {
        const DeviceFilters f{d_filters, d_query_filter, filter_words, num_filters, 0};
        return enqueue_query(h, w, d_queries, nq, query_format, num_neighbors,
                             {d_out_ids, d_out_dists, d_out_counts, d_out_stats}, false, stream,
                             [&](const void* q, int f2, uint32_t kk, const QueryOut& o) {
                                 return enqueue_search(h, w, q, nq, f2, max_search, kk, o, stream, nullptr, nullptr,
                                                       &f);
                             });
    });
}

int granne_b200_exact_search_filtered_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                            const uint32_t* filters, uint32_t num_filters, uint64_t filter_words,
                                            const uint32_t* query_filter, uint32_t num_neighbors, uint32_t* out_ids,
                                            float* out_dists, uint32_t* out_counts) {
    int rc = validate_exact_filtered(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, filters,
                                     num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, h->index_len)) ||
        (rc = check_query_filter(query_filter, nq, num_filters)) ||
        (rc = check_host_query_ids(h, queries, nq, query_format)))
        return rc;
    return exact_filtered_host(h, queries, nq, query_format, num_neighbors, filters, num_filters, filter_words,
                               query_filter, 0, out_ids, out_dists, out_counts);
}

int granne_b200_exact_search_filtered_batch_device(granne_b200_index* h, const void* d_queries, size_t nq,
                                                   int query_format, const uint32_t* d_filters, uint32_t num_filters,
                                                   uint64_t filter_words, const uint32_t* d_query_filter,
                                                   uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                                   uint32_t* d_out_counts, void* cuda_stream) {
    int rc = validate_exact_filtered(h, d_queries, nq, query_format, num_neighbors, d_out_ids, d_out_dists, d_filters,
                                     num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, h->index_len))) return rc;
    return device_batch(h, cuda_stream, false, [&](Workspace* w, cudaStream_t stream) {
        const DeviceFilters f{d_filters, d_query_filter, filter_words, num_filters, 0};
        return enqueue_query(h, w, d_queries, nq, query_format, num_neighbors,
                             {d_out_ids, d_out_dists, d_out_counts, nullptr}, false, stream,
                             [&](const void* q, int f2, uint32_t kk, const QueryOut& o) {
                                 return enqueue_exact(h, w, q, nq, f2, kk, o, stream, &f);
                             });
    });
}

int granne_b200_set_rerank_elements(granne_b200_index* h, const void* elements_bytes, size_t elements_len) {
    int rc = check_rerank_target(h);
    if (rc) return rc;
    if (!elements_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements buffer is null");
    return guarded([&] {
        gb::DenseView dv;
        std::string err;
        if (!gb::parse_dense(static_cast<const uint8_t*>(elements_bytes), elements_len, 4, &dv, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        if ((rc = check_rerank_shape(h, dv.num, dv.dim))) return rc;
        GB_DEVICE(h->device);
        return stage_rerank_rows(h, dv.data, dv.num, (uint32_t)dv.dim, false);
    });
}

int granne_b200_set_rerank_elements_device(granne_b200_index* h, const float* d_rows, uint64_t n, uint32_t dim) {
    int rc = check_rerank_target(h);
    if (rc) return rc;
    if (!d_rows && n) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
    if ((rc = check_rerank_shape(h, n, dim))) return rc;
    return guarded([&] {
        GB_DEVICE(h->device);
        if (n && (rc = check_device_pointer(d_rows, h->device, "elements pointer"))) return rc;
        return stage_rerank_rows(h, reinterpret_cast<const uint8_t*>(d_rows), n, dim, true);
    });
}

int granne_b200_set_rerank_embeddings(granne_b200_index* h, const void* elements_bytes, size_t elements_len,
                                      const void* embeddings_bytes, size_t embeddings_len) {
    int rc = check_rerank_target(h);
    if (rc) return rc;
    return guarded([&] {
        gb::DenseView ev;
        gb::SumElements se;
        if ((rc = check_rerank_sum(h, elements_bytes, elements_len, embeddings_bytes, embeddings_len, &ev, &se)))
            return rc;
        GB_DEVICE(h->device);
        return stage_rerank(h, [&](gb::DeviceIndex& r, Staged& mem) { return stage_sum(h, r, mem, ev, se); });
    });
}

int granne_b200_search_rerank_batch(granne_b200_index* h, const float* queries, size_t nq, int query_format,
                                    uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                    uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint64_t* out_stats) {
    int rc = validate_rerank(h, queries, nq, query_format, max_search, num_candidates, num_neighbors, out_ids,
                             out_dists);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    return host_batch(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts, out_stats,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          return enqueue_rerank(h, w, w->d_queries.get(), nq, max_search, num_candidates,
                                                num_neighbors, out, stream);
                      });
}

int granne_b200_search_rerank_batch_device(granne_b200_index* h, const float* d_queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                           uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                           uint64_t* d_out_stats, void* cuda_stream) {
    int rc = validate_rerank(h, d_queries, nq, query_format, max_search, num_candidates, num_neighbors, d_out_ids,
                             d_out_dists);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    return device_batch(h, cuda_stream, true, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_rerank(h, w, d_queries, nq, max_search, num_candidates, num_neighbors,
                              {d_out_ids, d_out_dists, d_out_counts, d_out_stats}, stream);
    });
}

int granne_b200_search_diverse_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                     uint32_t max_search, uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                                     uint32_t* out_counts, uint64_t* out_stats) {
    int rc = validate_diverse(h, queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists);
    if (rc || nq == 0) return rc;
    if ((rc = check_host_query_ids(h, queries, nq, query_format))) return rc;
    return host_batch(h, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts, out_stats,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          return enqueue_diverse(h, w, w->d_queries.get(), nq, query_format, max_search,
                                                 num_neighbors, out, true, stream);
                      });
}

int granne_b200_search_diverse_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                            uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids,
                                            float* d_out_dists, uint32_t* d_out_counts, uint64_t* d_out_stats,
                                            void* cuda_stream) {
    int rc = validate_diverse(h, d_queries, nq, query_format, max_search, num_neighbors, d_out_ids, d_out_dists);
    if (rc || nq == 0) return rc;
    return device_batch(h, cuda_stream, true, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_diverse(h, w, d_queries, nq, query_format, max_search, num_neighbors,
                               {d_out_ids, d_out_dists, d_out_counts, d_out_stats}, false, stream);
    });
}

int granne_b200_select_neighbors_batch(granne_b200_index* h, const uint32_t* cand_ids, const float* cand_dists,
                                       const uint32_t* cand_counts, size_t nq, uint32_t stride,
                                       uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                                       uint32_t* out_counts) {
    int rc = validate_select(h, cand_ids, cand_dists, cand_counts, nq, stride, num_neighbors, out_ids, out_dists);
    if (rc || nq == 0) return rc;
    if ((rc = check_candidate_lists(h, cand_ids, cand_dists, cand_counts, nq, stride))) return rc;
    // the counts go up as the call's 4-byte query rows, the lists as its inputs
    return host_batch(h, cand_counts, nq, GRANNE_B200_QUERY_ID, num_neighbors, out_ids, out_dists, out_counts, nullptr,
                      [&](Workspace* w, cudaStream_t stream, const QueryOut& out) {
                          const HostInput in[] = {{cand_ids, nq * stride * 4}, {cand_dists, nq * stride * 4}};
                          return with_call_inputs(stream, in, [&](const void* const* d) {
                              return enqueue_select(h, w, static_cast<const uint32_t*>(d[0]),
                                                    static_cast<const float*>(d[1]),
                                                    reinterpret_cast<const uint32_t*>(w->d_queries.get()), nq, stride,
                                                    num_neighbors, false, out, stream);
                          });
                      });
}

int granne_b200_select_neighbors_batch_device(granne_b200_index* h, const uint32_t* d_cand_ids,
                                              const float* d_cand_dists, const uint32_t* d_cand_counts, size_t nq,
                                              uint32_t stride, uint32_t num_neighbors, uint32_t* d_out_ids,
                                              float* d_out_dists, uint32_t* d_out_counts, void* cuda_stream) {
    int rc = validate_select(h, d_cand_ids, d_cand_dists, d_cand_counts, nq, stride, num_neighbors, d_out_ids,
                             d_out_dists);
    if (rc || nq == 0) return rc;
    return device_batch(h, cuda_stream, true, [&](Workspace* w, cudaStream_t stream) {
        return enqueue_select(h, w, d_cand_ids, d_cand_dists, d_cand_counts, nq, stride, num_neighbors, true,
                              {d_out_ids, d_out_dists, d_out_counts, nullptr}, stream);
    });
}

int granne_b200_inspect_index(const void* index_bytes, size_t index_len, uint64_t* out_num_layers,
                              uint64_t* out_layer_len, uint32_t* out_max_degree, uint32_t* out_row_width, size_t cap) {
    if (!index_bytes || !out_num_layers) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
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
    });
}

int granne_b200_decode_layer(const void* index_bytes, size_t index_len, uint64_t layer, uint32_t* rows,
                             size_t rows_cap_u32) {
    if (!index_bytes || !rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        if (layer >= graph.layers.size()) return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "layer out of range");
        const gb::HostLayer& L = graph.layers[layer];
        if (L.rows.size() > rows_cap_u32) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "rows buffer too small");
        std::memcpy(rows, L.rows.data(), L.rows.size() * 4);
        return GRANNE_B200_OK;
    });
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

// `index_bytes` != nullptr: GranneBuilder::from_bytes, the builder continues from that index image
static int builder_new_impl(const granne_b200_build_config* cfg, int element_kind, const void* elements_bytes,
                            size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                            granne_b200_builder** out, const void* dev_rows, uint64_t n_dev, uint32_t dim_dev,
                            const void* index_bytes = nullptr, size_t index_len = 0) {
    if (!out || !cfg) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    // the on-disk format counts a list's entries in one byte (set_vector.rs:91-99): 255 is the format's limit
    if (cfg->num_neighbors < 1 || cfg->num_neighbors > 255)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "num_neighbors must be in 1..255");
    if (cfg->max_search < 1) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "max_search must be >= 1");
    if (!(cfg->layer_multiplier > 1.0f)) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "layer_multiplier must be > 1");
    return guarded([&] {
        // the image is decoded and checked on the host first, so that a malformed one is reported without a device
        gb::HostGraph graph;
        if (index_bytes) {
            std::string err;
            if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
                return fail(GRANNE_B200_ERR_FORMAT, err);
            if (graph.layers.size() > (size_t)gb::kMaxLayers) return fail(GRANNE_B200_ERR_FORMAT, "too many layers");
        }
        DeviceGuard guard;
        std::unique_ptr<granne_b200_builder> b(new granne_b200_builder());
        b->cfg = *cfg;
        b->stride = (cfg->num_neighbors + 7u) & ~7u;
        int rc = new_handle(&guard, device, element_kind, static_cast<const uint8_t*>(elements_bytes), elements_len,
                            static_cast<const uint8_t*>(embeddings_bytes), embeddings_len, dev_rows, n_dev, dim_dev,
                            &b->h);
        if (rc) return rc;
        Handle* h = b->h.get();
        if (h->dev.num_elements >= 0xFFFFFFFFull)  // assert!(elements.len() < UNUSED) (:420)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many elements");
        h->dev.num_layers = 0;
        if ((rc = builder_load_layers(b.get(), graph))) return rc;
        finish_handle(h);
        if ((rc = ws_acquire(h, &b->ws))) return rc;
        GB_CUDA(cudaMemset(b->ws->d_error, 0, 4 * sizeof(int)));
        *out = b.release();
        return GRANNE_B200_OK;
    });
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

int granne_b200_builder_from_index(const granne_b200_build_config* cfg, const void* index_bytes, size_t index_len,
                                   int element_kind, const void* elements_bytes, size_t elements_len,
                                   const void* embeddings_bytes, size_t embeddings_len, int device,
                                   granne_b200_builder** out) {
    if (!index_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index buffer is null");
    return builder_new_impl(cfg, element_kind, elements_bytes, elements_len, embeddings_bytes, embeddings_len, device,
                            out, nullptr, 0, 0, index_bytes, index_len);
}

int granne_b200_builder_from_index_device_elements(const granne_b200_build_config* cfg, const void* index_bytes,
                                                   size_t index_len, int element_kind, const void* d_element_rows,
                                                   uint64_t num_elements, uint32_t dim, int device,
                                                   granne_b200_builder** out) {
    if (!index_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "index buffer is null");
    if (!d_element_rows) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements pointer is null");
    return builder_new_impl(cfg, element_kind, nullptr, 0, nullptr, 0, device, out, d_element_rows, num_elements, dim,
                            index_bytes, index_len);
}

// GranneBuilder::push for the dense containers (ExtendableElementContainer::push, src/index/mod.rs:512-531;
// src/elements/dense_vector.rs:120-136): `elements_bytes` is an elements file image of the same width whose rows are
// appended to the staged container.  The appended elements are indexed by the next build() / build_partial().
int granne_b200_builder_append(granne_b200_builder* b, const void* elements_bytes, size_t elements_len) {
    if (!b || !elements_bytes) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
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
            GB_CUDA(cudaStreamSynchronize(b->ws->stream.get()));
            unsigned long long old_terms = 0;
            if (old_n)
                GB_CUDA(cudaMemcpy(&old_terms, d.sum_offsets + old_n, 8, cudaMemcpyDeviceToHost));
            std::vector<unsigned long long> off(add + 1);
            for (uint64_t i = 0; i <= add; ++i) off[i] = old_terms + se.offsets[i];
            Buffer<unsigned long long> doff;
            Buffer<uint32_t> dterms;
            int rc;
            if ((rc = dev_alloc(&doff, new_n + 1)) || (rc = dev_alloc(&dterms, (size_t)old_terms + se.terms.size())))
                return rc;
            if (old_n) {
                GB_CUDA(cudaMemcpy(doff.get(), d.sum_offsets, (size_t)old_n * 8, cudaMemcpyDeviceToDevice));
                if (old_terms)
                    GB_CUDA(cudaMemcpy(dterms.get(), d.sum_terms, (size_t)old_terms * 4, cudaMemcpyDeviceToDevice));
            }
            GB_CUDA(cudaMemcpy(doff.get() + old_n, off.data(), (add + 1) * 8, cudaMemcpyHostToDevice));
            if (!se.terms.empty())
                GB_CUDA(cudaMemcpy(dterms.get() + old_terms, se.terms.data(), se.terms.size() * 4,
                                   cudaMemcpyHostToDevice));
            d.sum_offsets = stage(&h->dev_mem.sum_offsets, std::move(doff));
            d.sum_terms = stage(&h->dev_mem.sum_terms, std::move(dterms));
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
        GB_CUDA(cudaStreamSynchronize(b->ws->stream.get()));
        const size_t row_bytes = (size_t)d.row_stride * esz;
        Buffer<uint8_t> rows;
        int rc;
        if ((rc = dev_alloc(&rows, (size_t)new_n * row_bytes))) return rc;
        if (old_n) GB_CUDA(cudaMemcpy(rows.get(), d.vectors, (size_t)old_n * row_bytes, cudaMemcpyDeviceToDevice));
        if ((rc = upload_rows(h, d, dv.data, dv.num, false, rows.get() + (size_t)old_n * row_bytes))) return rc;
        d.vectors = stage(&h->dev_mem.vectors, std::move(rows));
        d.num_vectors = new_n;
        d.num_elements = new_n;
        return GRANNE_B200_OK;
    });
}

int granne_b200_builder_build(granne_b200_builder* b, uint64_t num_elements) {
    if (!b) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "builder is null");
    return guarded([&] { return builder_build_partial(b, num_elements ? num_elements : b->h->dev.num_elements); });
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
    return guarded([&] {
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
        return copy_image_out(image, out, cap, out_len);
    });
}

int granne_b200_builder_write_index(granne_b200_builder* b, void* out, size_t cap, size_t* out_len) {
    if (!b) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return granne_b200_write_index(b->h.get(), out, cap, out_len);
}

int granne_b200_builder_get_index(granne_b200_builder* b, granne_b200_index** out) {
    if (!b || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        const Handle* src = b->h.get();
        std::unique_ptr<Handle> h(new Handle());
        h->device = src->device;
        h->num_sms = src->num_sms;
        h->smem_optin = src->smem_optin;
        h->dev = src->dev;
        h->dev_mem = src->dev_mem;  // shared ownership of the staged elements and layers
        h->layer_max_degree = src->layer_max_degree;
        finish_handle(h.get());
        *out = h.release();
        return GRANNE_B200_OK;
    });
}

void granne_b200_builder_free(granne_b200_builder* b) {
    if (!b) return;
    DeviceGuard guard(b->h->device);
    cudaDeviceSynchronize();
    delete b;
}

int granne_b200_elements_from_raw(int element_kind, const float* raw, uint64_t n, uint32_t dim, int device, void* out,
                                  size_t cap, size_t* out_len) {
    if (!out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (element_kind != GRANNE_B200_ANGULAR && element_kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements_from_raw builds angular or angular_int vectors");
    if (dim == 0 || dim > 12000) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "dim must be in 1..12000");
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
    write_width_header(o, dim);
    const uint64_t slab = std::max<uint64_t>(1, (256ull << 20) / ((size_t)dim * 4));
    const uint64_t rows_alloc = std::min<uint64_t>(slab, std::max<uint64_t>(n, 1));
    Buffer<float> d_raw;
    Buffer<uint8_t> d_out;
    if ((rc = d_raw.grow(rows_alloc * dim, nullptr)) || (rc = d_out.grow(rows_alloc * dim * esz, nullptr))) return rc;
    for (uint64_t r0 = 0; r0 < n; r0 += slab) {
        const uint64_t nr = std::min(slab, n - r0);
        GB_CUDA(cudaMemcpy(d_raw.get(), raw + r0 * dim, (size_t)nr * dim * 4, cudaMemcpyHostToDevice));
        if ((rc = launch<gb::make_elements_kernel>((unsigned)std::min<uint64_t>(nr, (uint64_t)sms * 32), 32,
                                                   (size_t)dim * 4, nullptr, nullptr, d_raw.get(), nr, dim,
                                                   element_kind, d_out.get())))
            return rc;
        GB_CUDA(cudaMemcpy(o + 8 + (size_t)r0 * dim * esz, d_out.get(), (size_t)nr * dim * esz,
                           cudaMemcpyDeviceToHost));
    }
    return GRANNE_B200_OK;
}

// Vector::from per row (angular.rs:55-61 / angular_int.rs:28-45), device to device: d_raw = n x dim f32 rows in HBM,
// d_out = n x dim elements (f32 or i8), both on `device`; runs on `cuda_stream` (asynchronous).
int granne_b200_elements_from_raw_device(int element_kind, const float* d_raw, uint64_t n, uint32_t dim, int device,
                                         void* d_out, void* cuda_stream) {
    if (element_kind != GRANNE_B200_ANGULAR && element_kind != GRANNE_B200_ANGULAR_INT)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements_from_raw supports angular and angular_int");
    if (dim == 0 || dim > 12000) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "dim must be in 1..12000");
    if (n == 0) return GRANNE_B200_OK;
    if (!d_raw || !d_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    int sms = 0;
    size_t optin = 0;
    int rc = check_device(device, &sms, &optin);
    if (rc) return rc;
    GB_DEVICE(device);
    return launch<gb::make_elements_kernel>((unsigned)std::min<uint64_t>(n, (uint64_t)sms * 32), 32, (size_t)dim * 4,
                                            static_cast<cudaStream_t>(cuda_stream), nullptr, d_raw, n, dim,
                                            element_kind, d_out);
}

// compute_embeddings_and_save_to_disk (embeddings/parsing.rs:102-152) into a caller buffer.  Two windows are in
// flight on two streams: while one window's kernels run, the other's rows come back through pinned memory and the
// next window's term lists go out.
int granne_b200_compute_embeddings(int element_kind, const void* elements_bytes, size_t elements_len,
                                   const void* embeddings_bytes, size_t embeddings_len, int device, void* out,
                                   size_t cap, size_t* out_len) {
    if (!out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        EmbeddingsInput in;
        int rc = check_embeddings_input(element_kind, elements_bytes, elements_len, embeddings_bytes, embeddings_len,
                                        &in);
        if (rc) return rc;
        const size_t row_bytes = (size_t)in.dim * (element_kind == GRANNE_B200_ANGULAR ? 4 : 1);
        const size_t need = 8 + (size_t)in.n * row_bytes;
        *out_len = need;
        if (!out) return GRANNE_B200_OK;
        if (cap < need) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "output buffer too small");
        int sms = 0;
        size_t optin = 0;
        if ((rc = check_device(device, &sms, &optin))) return rc;
        GB_DEVICE(device);
        uint8_t* o = static_cast<uint8_t*>(out);
        write_width_header(o, in.dim);
        if (in.dim == 0) return GRANNE_B200_OK;

        const uint64_t* off = in.el.offsets.data();
        const uint64_t rows = std::min(in.n, emb_window_rows(in.dim));
        Buffer<float> d_table;
        Buffer<int> d_status;
        if ((rc = dev_alloc(&d_table, in.table.num * in.dim)) || (rc = dev_alloc(&d_status, 1))) return rc;
        GB_CUDA(cudaMemcpy(d_table.get(), in.table.data, in.table.num * in.dim * 4, cudaMemcpyHostToDevice));
        GB_CUDA(cudaMemset(d_status.get(), 0, 4));
        GB_CUDA(cudaStreamSynchronize(nullptr));  // the windows' streams do not wait for the legacy stream
        struct Window {
            Stream stream;  // declared first: destroyed after the buffers
            Buffer<unsigned long long> d_off;
            Buffer<uint32_t> d_terms;
            Buffer<float> d_raw;
            Buffer<int8_t> d_i8;
            Pinned<unsigned long long> h_off;
            Pinned<uint32_t> h_terms;
            Pinned<uint8_t> h_out;
            uint64_t r0 = 0, nr = 0;  // the elements in flight
        } win[2];
        for (Window& w : win) {
            cudaStream_t s = nullptr;
            GB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
            w.stream.reset(s);
            if ((rc = w.d_off.grow(rows + 1, s)) || (rc = w.d_raw.grow(rows * in.dim, s)) ||
                (rc = w.h_off.grow(rows + 1, s)) || (rc = w.h_out.grow(rows * row_bytes, s)) ||
                (element_kind == GRANNE_B200_ANGULAR_INT && (rc = w.d_i8.grow(rows * in.dim, s))))
                return rc;
        }
        // waits for a window's rows and moves them into the image
        auto land = [&](Window& w) {
            if (!w.nr) return GRANNE_B200_OK;
            GB_CUDA(cudaStreamSynchronize(w.stream.get()));
            std::memcpy(o + 8 + w.r0 * row_bytes, w.h_out.get(), w.nr * row_bytes);
            w.nr = 0;
            return GRANNE_B200_OK;
        };
        uint64_t k = 0;
        for (uint64_t r0 = 0; r0 < in.n; ++k) {
            Window& w = win[k & 1];
            cudaStream_t s = w.stream.get();
            if ((rc = land(w))) return rc;
            const uint64_t r1 = emb_window_end(in, r0), nr = r1 - r0, t0 = off[r0], nt = off[r1] - t0;
            if ((rc = w.d_terms.grow(std::max<uint64_t>(nt, 1), s)) || (rc = w.h_terms.grow(std::max<uint64_t>(nt, 1), s)))
                return rc;
            std::memcpy(w.h_off.get(), off + r0, (nr + 1) * 8);
            if (nt) std::memcpy(w.h_terms.get(), in.el.terms.data() + t0, nt * 4);
            GB_CUDA(cudaMemcpyAsync(w.d_off.get(), w.h_off.get(), (nr + 1) * 8, cudaMemcpyHostToDevice, s));
            if (nt) GB_CUDA(cudaMemcpyAsync(w.d_terms.get(), w.h_terms.get(), nt * 4, cudaMemcpyHostToDevice, s));
            void* rows_out = element_kind == GRANNE_B200_ANGULAR ? static_cast<void*>(w.d_raw.get()) : w.d_i8.get();
            if ((rc = launch_embeddings(in, element_kind, sms, d_table.get(), w.d_off.get(), t0, w.d_terms.get(), nr,
                                        w.d_raw.get(), rows_out, d_status.get(), s, nullptr)))
                return rc;
            GB_CUDA(cudaMemcpyAsync(w.h_out.get(), rows_out, nr * row_bytes, cudaMemcpyDeviceToHost, s));
            w.r0 = r0;
            w.nr = nr;
            r0 = r1;
        }
        if ((rc = land(win[k & 1])) || (rc = land(win[(k + 1) & 1]))) return rc;
        return embeddings_status(d_status.get());
    });
}

// The rows of granne_b200_compute_embeddings, written to device memory on the caller's stream.
int granne_b200_compute_embeddings_device(int element_kind, const void* elements_bytes, size_t elements_len,
                                          const void* embeddings_bytes, size_t embeddings_len, int device,
                                          void* d_out, uint64_t* out_n, uint32_t* out_dim, void* cuda_stream) {
    if (!out_n || !out_dim) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        EmbeddingsInput in;
        int rc = check_embeddings_input(element_kind, elements_bytes, elements_len, embeddings_bytes, embeddings_len,
                                        &in);
        if (rc) return rc;
        *out_n = in.n;
        *out_dim = in.dim;
        if (!d_out) return GRANNE_B200_OK;
        int sms = 0;
        size_t optin = 0;
        if ((rc = check_device(device, &sms, &optin))) return rc;
        GB_DEVICE(device);
        if (in.dim == 0) return GRANNE_B200_OK;
        if ((rc = check_device_pointer(d_out, device, "d_out"))) return rc;
        const cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
        const uint64_t rows = std::min(in.n, emb_window_rows(in.dim));
        Buffer<float> d_table, d_raw;
        Buffer<unsigned long long> d_off;
        Buffer<uint32_t> d_terms;
        Buffer<int> d_status;
        if ((rc = dev_alloc(&d_table, in.table.num * in.dim)) || (rc = dev_alloc(&d_off, in.n + 1)) ||
            (rc = dev_alloc(&d_terms, in.el.terms.size())) || (rc = dev_alloc(&d_status, 1)) ||
            (element_kind == GRANNE_B200_ANGULAR_INT && (rc = d_raw.grow(rows * in.dim, nullptr))))
            return rc;
        GB_CUDA(cudaMemcpy(d_table.get(), in.table.data, in.table.num * in.dim * 4, cudaMemcpyHostToDevice));
        GB_CUDA(cudaMemcpy(d_off.get(), in.el.offsets.data(), (in.n + 1) * 8, cudaMemcpyHostToDevice));
        if (!in.el.terms.empty())
            GB_CUDA(cudaMemcpy(d_terms.get(), in.el.terms.data(), in.el.terms.size() * 4, cudaMemcpyHostToDevice));
        GB_CUDA(cudaMemset(d_status.get(), 0, 4));
        GB_CUDA(cudaStreamSynchronize(nullptr));  // the caller's stream may not wait for the legacy stream
        for (uint64_t r0 = 0; r0 < in.n;) {
            const uint64_t r1 = emb_window_end(in, r0), nr = r1 - r0;
            float* raw = element_kind == GRANNE_B200_ANGULAR ? static_cast<float*>(d_out) + r0 * in.dim : d_raw.get();
            void* rows_out = element_kind == GRANNE_B200_ANGULAR ? static_cast<void*>(raw)
                                                                  : static_cast<int8_t*>(d_out) + r0 * in.dim;
            if ((rc = launch_embeddings(in, element_kind, sms, d_table.get(), d_off.get() + r0, 0, d_terms.get(), nr,
                                        raw, rows_out, d_status.get(), s, nullptr)))
                return rc;
            r0 = r1;
        }
        GB_CUDA(cudaStreamSynchronize(s));
        return embeddings_status(d_status.get());
    });
}

// ---- compute_distance (py/src/lib.rs:71-89) -----------------------------------------------------------------------
int granne_b200_compute_distances(int element_kind, const float* a, const float* b, uint64_t n, uint32_t dim, int device,
                                  float* out) {
    if (n == 0) return GRANNE_B200_OK;
    if (!a || !b || !out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    if (n > 0xFFFFFFFFull) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "too many pairs for one call");
    return guarded([&] {
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
        GB_DEVICE(device);
        Buffer<float> d_a, d_out;
        Buffer<int> d_err;
        if ((rc = d_a.grow((size_t)n * dim, nullptr)) || (rc = d_out.grow(n, nullptr)) || (rc = d_err.grow(1, nullptr)))
            return rc;
        GB_CUDA(cudaMemcpy(d_a.get(), a, (size_t)n * dim * 4, cudaMemcpyHostToDevice));
        GB_CUDA(cudaMemset(d_err.get(), 0, 4));
        const EngineTiles eng = engine_tiles(h->dev);
        gb::PairArgs args{};
        args.queries = d_a.get();
        args.n = (uint32_t)n;
        args.out = d_out.get();
        args.error_flag = d_err.get();
        args.tiles = eng.tiles;
        const unsigned grid = (unsigned)std::min<uint64_t>(n, (uint64_t)h->num_sms * 16);
        const size_t smem = gb::LinkLayout<size_t>(eng.base_smem, 8, 32).end;  // pair_distance_kernel's setup_ctx
        rc = DistDispatch::call(h->dev, [&](auto e) {
            return launch_warps<gb::pair_distance_kernel<typename decltype(e)::type>>(h.get(), grid, smem, nullptr,
                                                                                     h->dev, args);
        });
        if (rc) return rc;
        GB_CUDA(cudaDeviceSynchronize());
        int herr = 0;
        GB_CUDA(cudaMemcpy(&herr, d_err.get(), 4, cudaMemcpyDeviceToHost));
        GB_CUDA(cudaMemcpy(out, d_out.get(), (size_t)n * 4, cudaMemcpyDeviceToHost));
        return error_from_bits(herr);
    });
}

int granne_b200_reencode_index(const void* index_bytes, size_t index_len, void* out, size_t cap, size_t* out_len) {
    if (!index_bytes || !out_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        gb::HostGraph graph;
        std::string err;
        if (!gb::parse_index(static_cast<const uint8_t*>(index_bytes), index_len, &graph, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        std::vector<gb::LayerView> views;
        for (const gb::HostLayer& L : graph.layers) views.push_back({L.rows.data(), L.num_nodes, L.width});
        std::vector<uint8_t> image;
        if (!gb::encode_index(views, &image, &err)) return fail(GRANNE_B200_ERR_FORMAT, err);
        return copy_image_out(image, out, cap, out_len);
    });
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
    return guarded([&] {
        GB_DEVICE(h->device);
        std::vector<uint64_t> layer_lens(nl);
        for (int l = 0; l < nl; ++l) layer_lens[l] = h->dev.layer_len[l];
        const size_t trail_layers = std::min<size_t>(gb::kTrailLayers, (size_t)nl - 1);
        std::vector<std::vector<uint32_t>> eps(trail_layers);
        std::unique_ptr<Workspace> ws;
        int rc = ws_acquire(h, &ws);
        if (rc) return rc;
        Workspace* w = ws.get();
        const int status = [&] {
            const size_t batch = (size_t)std::min<uint64_t>(std::max<uint64_t>(n, 1), 1u << 20);
            cudaStream_t stream = w->stream.get();
            Buffer<uint32_t> d_q, d_ids, d_cnt;
            Buffer<float> d_d;
            if ((rc = d_q.grow(batch, stream)) || (rc = d_ids.grow(batch, stream)) || (rc = d_cnt.grow(batch, stream)) ||
                (rc = d_d.grow(batch, stream)))
                return rc;
            // the trail searches run over a PRIVATE single-layer view of the staged index: the shared handle is never
            // modified, so concurrent searches on it stay correct
            gb::DeviceIndex view = h->dev;
            for (size_t j = 0; j < trail_layers; ++j) {
                eps[j].resize(n - layer_lens[j]);
                view.num_layers = 1;
                view.layer_rows[0] = h->dev.layer_rows[j];
                view.layer_width[0] = h->dev.layer_width[j];
                view.layer_len[0] = h->dev.layer_len[j];
                for (uint64_t base = layer_lens[j]; base < n; base += batch) {
                    const uint64_t bsz = std::min<uint64_t>(batch, n - base);
                    if ((rc = launch<gb::iota_kernel>((unsigned)((bsz + 255) / 256), 256, 0, stream, &h->launches,
                                                      d_q.get(), (uint32_t)bsz, (uint32_t)base, 1)))
                        return rc;
                    GB_CUDA(cudaMemsetAsync(w->d_counters.get(), 0, kHostCallBytes, stream));
                    rc = enqueue_search(h, w, d_q.get(), bsz, gb::kQueryById, 1, 1,
                                        {d_ids.get(), d_d.get(), d_cnt.get(), nullptr}, stream, nullptr, &view);
                    if (rc) return rc;
                    GB_CUDA(cudaMemcpyAsync(eps[j].data() + (base - layer_lens[j]), d_ids.get(), bsz * 4,
                                            cudaMemcpyDeviceToHost, stream));
                    int herr[4] = {0, 0, 0, 0};
                    GB_CUDA(cudaMemcpyAsync(herr, w->d_error, sizeof(herr), cudaMemcpyDeviceToHost, stream));
                    GB_CUDA(cudaStreamSynchronize(stream));
                    if ((rc = error_from_bits(herr[0]))) return rc;
                }
            }
            return GRANNE_B200_OK;
        }();
        ws_release(h, std::move(ws));  // back to the pool on every path
        if (status) return status;
        gb::order_from_trails(layer_lens, eps, order_out);
        return GRANNE_B200_OK;
    });
}

int granne_b200_order_from_trails(const uint64_t* layer_lens, uint32_t num_layers, const uint32_t* trails, uint64_t n,
                                  uint64_t* order_out) {
    if (!layer_lens || !trails || !order_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
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
    });
}

int granne_b200_order_by_keys(const void* index_bytes, size_t index_len, const uint64_t* keys, uint64_t num_keys,
                              uint32_t key_width, uint64_t* order_out) {
    if (!index_bytes || !keys || !order_out || key_width == 0)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
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
    });
}

int granne_b200_embedding_reorder_keys(const void* elements_bytes, size_t elements_len, const void* embeddings_bytes,
                                       size_t embeddings_len, uint64_t* keys_out) {
    if (!elements_bytes || !embeddings_bytes || !keys_out) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
        std::string err;
        if (!gb::embedding_reorder_keys(static_cast<const uint8_t*>(elements_bytes), elements_len,
                                        static_cast<const uint8_t*>(embeddings_bytes), embeddings_len, keys_out, &err))
            return fail(GRANNE_B200_ERR_FORMAT, err);
        return GRANNE_B200_OK;
    });
}

int granne_b200_apply_order(const void* index_bytes, size_t index_len, int element_kind, const void* elements_bytes,
                            size_t elements_len, const uint64_t* order, uint64_t n, void* out_index, size_t index_cap,
                            size_t* index_out_len, void* out_elements, size_t elements_cap, size_t* elements_out_len) {
    if (!index_bytes || !elements_bytes || !order || !index_out_len || !elements_out_len)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    return guarded([&] {
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
    });
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
    const int rc = launch<gb::merge_topk_kernel>(grid, block, 0, stream, nullptr, d_part_ids, d_part_dists, d_base,
                                                 (uint32_t)num_parts, nq, k,
                                                 reinterpret_cast<unsigned long long*>(d_out_ids), d_out_dists);
    if (rc) return rc;
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
    return guarded([&] {
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
    });
}

void granne_b200_multi_close(granne_b200_multi* m) {
    if (!m) return;
    for (auto* p : m->parts) granne_b200_close(p);
    delete m;
}

uint64_t granne_b200_multi_len(const granne_b200_multi* m) { return m ? m->total_len : 0; }
size_t granne_b200_multi_num_parts(const granne_b200_multi* m) { return m ? m->parts.size() : 0; }
uint64_t granne_b200_multi_part_len(const granne_b200_multi* m, size_t s) {
    return (m && s < m->parts.size()) ? m->parts[s]->index_len : 0;
}
uint64_t granne_b200_multi_shard_base(const granne_b200_multi* m, size_t s) {
    return (m && s < m->base.size()) ? m->base[s] : 0;
}

}  // extern "C"

namespace {

// A batch on a multi handle: `part(i, b, q, cnt, ids, dists, counts)` runs the single-device call on part i for the
// queries [b, b + cnt), whose rows start at q.  REPLICATED slices the queries over the devices; RANGE_PARTITIONED runs
// every query on every shard (b = 0, cnt = nq) and merges the shard lists.
template <class Part>
int multi_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format, uint32_t num_neighbors,
                uint64_t* out_ids, float* out_dists, uint32_t* out_counts, Part&& part) {
    return guarded([&] {
        const size_t n = m->parts.size(), k = num_neighbors;
        const size_t qrow = query_row_bytes(m->kind, m->dim, query_format);
        const uint8_t* q = static_cast<const uint8_t*>(queries);
        if (m->mode == GRANNE_B200_MODE_REPLICATED) {
            // contiguous, balanced query slices (the first nq % n devices take one more)
            std::vector<uint32_t> ids(nq * k);
            std::vector<uint32_t> cnt(nq);
            const size_t per = nq / n, extra = nq % n;
            int rc = for_each_part(n, [&](size_t i) {
                const size_t b = i * per + std::min(i, extra), cntq = per + (i < extra ? 1 : 0);
                if (cntq == 0) return (int)GRANNE_B200_OK;
                return part(i, b, q + b * qrow, cntq, ids.data() + b * k, out_dists + b * k, cnt.data() + b);
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
            return part(i, 0, q, nq, ids.data() + i * nq * k, ds.data() + i * nq * k, nullptr);
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
    });
}

// A multi-handle call whatever its query format: `call(q, fmt, k, ids, dists, counts)` runs it for host query rows q.
// RAW_F32 and ELEMENT queries go straight to it.  Ids are u64 global ids, each in some part's [shard_base, shard_base +
// Index::len) (checked on the host before any device call); their rows are read from the parts that own them
// (granne_b200_get_elements), and the call runs on those rows as ELEMENT queries: into the caller's outputs for
// QUERY_ID, with k + 1 columns for QUERY_ID_EXCLUDING, whose entry of the query's own global id is then removed.
// nq u64 global ids by the part that owns them: local[s] the local ids of the queries rows_of[s] of part s.  An id in
// no part's [shard_base, shard_base + Index::len) is ERR_OUT_OF_RANGE.
struct MultiIds {
    std::vector<std::vector<uint32_t>> local;
    std::vector<std::vector<size_t>> rows_of;
};
int multi_ids(const granne_b200_multi* m, const uint64_t* gids, size_t nq, MultiIds* out) {
    const size_t n = m->parts.size();
    out->local.assign(n, {});
    out->rows_of.assign(n, {});
    for (size_t q = 0; q < nq; ++q) {
        size_t s = 0;
        if (m->mode == GRANNE_B200_MODE_RANGE_PARTITIONED)
            s = std::upper_bound(m->base.begin(), m->base.end(), gids[q]) - m->base.begin() - 1;
        if (gids[q] - m->base[s] >= m->parts[s]->index_len)
            return fail(GRANNE_B200_ERR_OUT_OF_RANGE, "element id is in no part's Index::len range");
        out->local[s].push_back((uint32_t)(gids[q] - m->base[s]));
        out->rows_of[s].push_back(q);
    }
    return GRANNE_B200_OK;
}

// The ELEMENT rows of nq queries by global id, read from the parts that own them (granne_b200_get_elements).
int multi_id_rows(granne_b200_multi* m, const MultiIds& ids, size_t nq, std::vector<uint8_t>* rows) {
    const size_t row = query_row_bytes(m->kind, m->dim, GRANNE_B200_QUERY_ELEMENT);
    std::vector<uint8_t> part;
    rows->assign(nq * row, 0);
    for (size_t s = 0; s < m->parts.size(); ++s) {
        if (ids.local[s].empty()) continue;
        part.resize(ids.local[s].size() * row);
        const int rc = granne_b200_get_elements(m->parts[s], ids.local[s].data(), ids.local[s].size(), part.data());
        if (rc) return rc;
        for (size_t j = 0; j < ids.rows_of[s].size(); ++j)
            std::memcpy(rows->data() + ids.rows_of[s][j] * row, part.data() + j * row, row);
    }
    return GRANNE_B200_OK;
}

template <class Call>
int multi_query(granne_b200_multi* m, const void* queries, size_t nq, int fmt, uint32_t k, uint64_t* out_ids,
                float* out_dists, uint32_t* out_counts, Call&& call) {
    if (!by_id(fmt)) return call(queries, fmt, k, out_ids, out_dists, out_counts);
    return guarded([&] {
        const uint64_t* gids = static_cast<const uint64_t*>(queries);
        MultiIds mi;
        std::vector<uint8_t> rows;
        int rc0 = multi_ids(m, gids, nq, &mi);
        if (rc0 || (rc0 = multi_id_rows(m, mi, nq, &rows))) return rc0;
        if (fmt == GRANNE_B200_QUERY_ID)
            return call(rows.data(), (int)GRANNE_B200_QUERY_ELEMENT, k, out_ids, out_dists, out_counts);
        const size_t kk = (size_t)k + 1;
        std::vector<uint64_t> ids(nq * kk);
        std::vector<float> ds(nq * kk);
        std::vector<uint32_t> cnt(nq);
        const int rc = call(rows.data(), (int)GRANNE_B200_QUERY_ELEMENT, (uint32_t)kk, ids.data(), ds.data(), cnt.data());
        if (rc) return rc;
        for (size_t q = 0; q < nq; ++q) {
            uint32_t r = 0;
            for (size_t j = 0; j < cnt[q] && r < k; ++j) {
                if (ids[q * kk + j] == gids[q]) continue;
                out_ids[q * k + r] = ids[q * kk + j];
                out_dists[q * k + r] = ds[q * kk + j];
                ++r;
            }
            if (out_counts) out_counts[q] = r;
            for (size_t j = r; j < k; ++j) {
                out_ids[q * k + j] = ~0ull;
                out_dists[q * k + j] = std::numeric_limits<float>::infinity();
            }
        }
        return (int)GRANNE_B200_OK;
    });
}

// The ids a multi handle's bitmaps must cover: [0, span) holds the global id of every part's elements.
uint64_t multi_filter_span(const granne_b200_multi* m) {
    uint64_t span = m->total_len;
    for (size_t s = 0; m->mode == GRANNE_B200_MODE_RANGE_PARTITIONED && s < m->parts.size(); ++s)
        span = std::max(span, m->base[s] + m->parts[s]->index_len);
    return span;
}

// A range call on a multi handle (host buffers; arguments checked, nq > 0): counts when offsets is null, else the fill
// of out_ids / out_dists.  REPLICATED: each device runs its slice of the queries (by id: the global ids are its local
// ids), a fill with its slice's offsets rebased to the slice.  RANGE_PARTITIONED: every shard counts every query (by id:
// on the rows the owning parts read); a fill then fills each shard's runs at offsets from those counts (a second scan)
// and sorts each query's entries from all shards by (distance, global id) into its segment.  For QUERY_ID_EXCLUDING the
// owning shard's distance of the query to itself (granne_b200_exact_search_within_batch on the one id) decides whether
// the query's own global id is in its range, and it is removed from the count and the segment.
int multi_range(granne_b200_multi* m, const void* queries, size_t nq, int fmt, float radius, const uint64_t* offsets,
                uint64_t* out_ids, float* out_dists, uint64_t* counts) {
    return guarded([&] {
        const size_t n = m->parts.size();
        const bool fill = offsets != nullptr;
        const uint64_t* gids = static_cast<const uint64_t*>(queries);
        MultiIds mi;
        int rc;
        if (by_id(fmt) && (rc = multi_ids(m, gids, nq, &mi))) return rc;
        if (m->mode == GRANNE_B200_MODE_REPLICATED) {
            std::vector<uint32_t> lids(by_id(fmt) ? nq : 0);
            for (size_t q = 0; q < lids.size(); ++q) lids[q] = (uint32_t)gids[q];
            const uint8_t* q0 = by_id(fmt) ? reinterpret_cast<const uint8_t*>(lids.data())
                                           : static_cast<const uint8_t*>(queries);
            const size_t qrow = query_row_bytes(m->kind, m->dim, fmt), per = nq / n, extra = nq % n;
            return for_each_part(n, [&](size_t i) {
                const size_t b = i * per + std::min(i, extra), cnt = per + (i < extra ? 1 : 0);
                if (cnt == 0) return (int)GRANNE_B200_OK;
                if (!fill) return granne_b200_exact_range_count(m->parts[i], q0 + b * qrow, cnt, fmt, radius, counts + b);
                return guarded([&] {
                    std::vector<uint64_t> off(cnt + 1);
                    for (size_t j = 0; j <= cnt; ++j) off[j] = offsets[b + j] - offsets[b];
                    std::vector<uint32_t> pids(off[cnt]);
                    const int r = granne_b200_exact_range_search(m->parts[i], q0 + b * qrow, cnt, fmt, radius,
                                                                 off.data(), pids.data(), out_dists + offsets[b]);
                    for (size_t j = 0; j < pids.size(); ++j)
                        out_ids[offsets[b] + j] = pids[j] == gb::kUnusedId ? ~0ull : (uint64_t)pids[j];
                    return r;
                });
            });
        }
        // range-partitioned: by id, the rows the owners read, as ELEMENT queries on every shard
        std::vector<uint8_t> rows;
        const void* q = queries;
        int f = fmt;
        if (by_id(fmt)) {
            if ((rc = multi_id_rows(m, mi, nq, &rows))) return rc;
            q = rows.data();
            f = GRANNE_B200_QUERY_ELEMENT;
        }
        std::vector<char> self_in(nq, 0);
        if (fmt == GRANNE_B200_QUERY_ID_EXCLUDING) {
            rc = for_each_part(n, [&](size_t s) {
                const size_t c = mi.local[s].size();
                if (c == 0) return (int)GRANNE_B200_OK;
                return guarded([&] {
                    std::vector<uint64_t> off(c + 1);
                    for (size_t j = 0; j <= c; ++j) off[j] = j;
                    std::vector<uint32_t> sid(c), scnt(c);
                    std::vector<float> sd(c);
                    const int r = granne_b200_exact_search_within_batch(m->parts[s], mi.local[s].data(), c,
                                                                        GRANNE_B200_QUERY_ID, off.data(),
                                                                        mi.local[s].data(), 1, sid.data(), sd.data(),
                                                                        scnt.data());
                    for (size_t j = 0; j < c && r == GRANNE_B200_OK; ++j)
                        self_in[mi.rows_of[s][j]] = scnt[j] == 1 && sd[j] <= radius;
                    return r;
                });
            });
            if (rc) return rc;
        }
        std::vector<uint64_t> pc(n * nq);
        if ((rc = for_each_part(n, [&](size_t i) {
                 return granne_b200_exact_range_count(m->parts[i], q, nq, f, radius, pc.data() + i * nq);
             })))
            return rc;
        if (!fill) {
            for (size_t qi = 0; qi < nq; ++qi) {
                uint64_t c = 0;
                for (size_t i = 0; i < n; ++i) c += pc[i * nq + qi];
                counts[qi] = c - (uint64_t)self_in[qi];
            }
            return (int)GRANNE_B200_OK;
        }
        std::vector<std::vector<uint64_t>> poff(n, std::vector<uint64_t>(nq + 1, 0));
        std::vector<std::vector<uint32_t>> pid(n);
        std::vector<std::vector<float>> pd(n);
        for (size_t i = 0; i < n; ++i) {
            for (size_t qi = 0; qi < nq; ++qi) poff[i][qi + 1] = poff[i][qi] + pc[i * nq + qi];
            pid[i].resize(poff[i][nq]);
            pd[i].resize(poff[i][nq]);
        }
        if ((rc = for_each_part(n, [&](size_t i) {
                 return granne_b200_exact_range_search(m->parts[i], q, nq, f, radius, poff[i].data(), pid[i].data(),
                                                       pd[i].data());
             })))
            return rc;
        bool mismatch = false;
        std::vector<std::pair<float, uint64_t>> all;
        for (size_t qi = 0; qi < nq; ++qi) {
            all.clear();
            for (size_t i = 0; i < n; ++i)
                for (uint64_t j = poff[i][qi]; j < poff[i][qi + 1]; ++j) {
                    const uint64_t g = m->base[i] + pid[i][j];
                    if (fmt == GRANNE_B200_QUERY_ID_EXCLUDING && g == gids[qi]) continue;
                    all.emplace_back(pd[i][j], g);
                }
            std::sort(all.begin(), all.end());  // distances are never NaN here (a NaN fails the shard call)
            const uint64_t b = offsets[qi], len = offsets[qi + 1] - b;
            const bool ok = all.size() == len;
            mismatch |= !ok;
            for (uint64_t j = 0; j < len; ++j) {
                out_ids[b + j] = ok ? all[j].second : ~0ull;
                out_dists[b + j] = ok ? all[j].first : std::numeric_limits<float>::infinity();
            }
        }
        if (mismatch)
            return fail(GRANNE_B200_ERR_INVALID_ARGUMENT,
                        "a range search segment's length differs from its query's count (it is padded)");
        return (int)GRANNE_B200_OK;
    });
}

// Attaches a re-rank container to every part: check(i) runs every host check of part i's images (i: the part, whose
// image is 0 for a replicated handle), for every part, before attach(i) stages any.  If a part then fails to stage (a
// device error), the parts this call attached drop their containers again, so that the call can be repeated.
template <class Check, class Attach>
int multi_attach_rerank(granne_b200_multi* m, Check&& check, Attach&& attach) {
    return guarded([&] {
        const size_t n = m->parts.size();
        for (size_t i = 0; i < n; ++i) {
            int rc = check_rerank_target(m->parts[i]);
            if (rc) return rc;
            if ((rc = check(i))) return rc;
        }
        std::vector<char> attached(n, 0);
        const int rc = for_each_part(n, [&](size_t i) {
            const int r = attach(i);
            attached[i] = r == GRANNE_B200_OK;
            return r;
        });
        if (rc) {
            for (size_t i = 0; i < n; ++i) {
                if (!attached[i]) continue;
                DeviceGuard guard(m->parts[i]->device);
                release_rerank(m->parts[i]);
            }
        }
        return rc;
    });
}

}  // namespace

extern "C" {

int granne_b200_multi_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                   uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                   uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_search(m->parts[0], queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, UINT32_MAX)) || nq == 0) return rc;
    return multi_query(m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                       [&](const void* rows, int fmt, uint32_t k, uint64_t* oi, float* od, uint32_t* oc) {
                           return multi_batch(
                               m, rows, nq, fmt, k, oi, od, oc,
                               [&](size_t i, size_t, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                                   return granne_b200_search_batch(m->parts[i], q, cnt, fmt, max_search, k, ids, ds,
                                                                   c, nullptr);
                               });
                       });
}

// Each shard's exact answer is exact, and a shard's ids are monotone in the global ids, so merging the shard lists by
// (distance, global id) gives the exact answer over the union of the shards.
int granne_b200_multi_exact_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                         uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                         uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_exact(m->parts[0], queries, nq, query_format, num_neighbors, out_ids, out_dists);
    if (rc || (rc = check_exclude_k(query_format, num_neighbors, GRANNE_B200_EXACT_MAX_K)) || nq == 0) return rc;
    return multi_query(m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                       [&](const void* rows, int fmt, uint32_t k, uint64_t* oi, float* od, uint32_t* oc) {
                           return multi_batch(
                               m, rows, nq, fmt, k, oi, od, oc,
                               [&](size_t i, size_t, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                                   return granne_b200_exact_search_batch(m->parts[i], q, cnt, fmt, k, ids, ds, c);
                               });
                       });
}

// REPLICATED: each device runs its slice of the queries on their lists, offsets rebased to the slice.
// RANGE_PARTITIONED: each global id goes to the shard that owns it as a local id, every shard runs every query on its
// local lists, and multi_batch merges the shard lists by (distance, global id) as for the exact search.
int granne_b200_multi_exact_search_within_batch(granne_b200_multi* m, const void* queries, size_t nq,
                                                int query_format, const uint64_t* offsets, const uint64_t* ids,
                                                uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                                uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_within(m->parts[0], queries, nq, query_format, num_neighbors, out_ids, out_dists, offsets, ids,
                             true);
    if (rc) return rc;
    if (nq == 0) return GRANNE_B200_OK;
    if ((rc = check_within_offsets(offsets, nq)) || (rc = check_within_ids(offsets, nq, ids, m->total_len))) return rc;
    return guarded([&] {
        const size_t n = m->parts.size();
        const bool range = m->mode == GRANNE_B200_MODE_RANGE_PARTITIONED;
        std::vector<std::vector<uint64_t>> loff(range ? n : 0, std::vector<uint64_t>(1, 0));
        std::vector<std::vector<uint32_t>> lids(range ? n : 0);
        for (size_t q = 0; range && q < nq; ++q) {
            for (uint64_t i = offsets[q]; i < offsets[q + 1]; ++i) {
                const size_t s = std::upper_bound(m->base.begin(), m->base.end(), ids[i]) - m->base.begin() - 1;
                const uint64_t local = ids[i] - m->base[s];
                if (local >= m->parts[s]->index_len)
                    return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "candidate id is in no shard's Index::len range");
                lids[s].push_back((uint32_t)local);
            }
            for (size_t s = 0; s < n; ++s) loff[s].push_back(lids[s].size());
        }
        return multi_query(
            m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
            [&](const void* rows, int fmt, uint32_t k, uint64_t* oi, float* od, uint32_t* oc) {
                return multi_batch(
                    m, rows, nq, fmt, k, oi, od, oc,
                    [&](size_t i, size_t b, const void* q, size_t cnt, uint32_t* pids, float* ds, uint32_t* c) {
                        if (range)
                            return granne_b200_exact_search_within_batch(m->parts[i], q, cnt, fmt, loff[i].data(),
                                                                         lids[i].data(), k, pids, ds, c);
                        // the slice of queries [b, b + cnt) and their lists
                        return guarded([&] {
                            std::vector<uint64_t> off(cnt + 1);
                            for (size_t j = 0; j <= cnt; ++j) off[j] = offsets[b + j] - offsets[b];
                            const std::vector<uint32_t> sl(ids + offsets[b], ids + offsets[b + cnt]);
                            return granne_b200_exact_search_within_batch(m->parts[i], q, cnt, fmt, off.data(),
                                                                         sl.data(), k, pids, ds, c);
                        });
                    });
            });
    });
}

// REPLICATED: each device runs its slice of the queries with their query_filter entries.  RANGE_PARTITIONED: every
// shard runs every query on the global bitmaps, reading bit shard_base[s] + local id, and multi_batch merges the shard
// lists by (distance, global id): shard s scores S_s(q), so the result is the first k of the union of the shards'
// admitted lists.
int granne_b200_multi_search_filtered_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                            uint32_t max_search, uint32_t num_neighbors, const uint32_t* filters,
                                            uint32_t num_filters, uint64_t filter_words, const uint32_t* query_filter,
                                            uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_filtered(m->parts[0], queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists,
                               filters, num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, multi_filter_span(m))) ||
        (rc = check_query_filter(query_filter, nq, num_filters)))
        return rc;
    return multi_query(m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                       [&](const void* rows, int fmt, uint32_t k, uint64_t* oi, float* od, uint32_t* oc) {
                           return multi_batch(
                               m, rows, nq, fmt, k, oi, od, oc,
                               [&](size_t i, size_t b, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                                   return search_filtered_host(m->parts[i], q, cnt, fmt, max_search, k, filters,
                                                               num_filters, filter_words,
                                                               query_filter ? query_filter + b : nullptr, m->base[i],
                                                               ids, ds, c, nullptr);
                               });
                       });
}

// As granne_b200_multi_search_filtered_batch: REPLICATED slices the queries with their query_filter entries;
// RANGE_PARTITIONED runs every query on every shard over the global bitmaps (bit shard_base[s] + local id), and
// multi_batch merges the shards' exact filtered lists by (distance, global id), which is the exact filtered answer over
// the union of the shards.
int granne_b200_multi_exact_search_filtered_batch(granne_b200_multi* m, const void* queries, size_t nq,
                                                  int query_format, const uint32_t* filters, uint32_t num_filters,
                                                  uint64_t filter_words, const uint32_t* query_filter,
                                                  uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                                  uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_exact_filtered(m->parts[0], queries, nq, query_format, num_neighbors, out_ids, out_dists,
                                     filters, num_filters);
    if (rc || nq == 0) return rc;
    if ((rc = check_filter_words(filter_words, multi_filter_span(m))) ||
        (rc = check_query_filter(query_filter, nq, num_filters)))
        return rc;
    return multi_query(m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                       [&](const void* rows, int fmt, uint32_t k, uint64_t* oi, float* od, uint32_t* oc) {
                           return multi_batch(
                               m, rows, nq, fmt, k, oi, od, oc,
                               [&](size_t i, size_t b, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                                   return exact_filtered_host(m->parts[i], q, cnt, fmt, k, filters, num_filters,
                                                              filter_words, query_filter ? query_filter + b : nullptr,
                                                              m->base[i], ids, ds, c);
                               });
                       });
}

int granne_b200_multi_exact_range_count(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                        float radius, uint64_t* counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    const int rc = validate_range(m->parts[0], queries, nq, query_format, radius, counts, nullptr, false);
    if (rc || nq == 0) return rc;
    return multi_range(m, queries, nq, query_format, radius, nullptr, nullptr, nullptr, counts);
}

int granne_b200_multi_exact_range_search(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                         float radius, const uint64_t* offsets, uint64_t* ids, float* dists) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_range(m->parts[0], queries, nq, query_format, radius, nullptr, offsets, true);
    if (rc || nq == 0 || (rc = check_range_outputs(offsets, nq, ids, dists))) return rc;
    return multi_range(m, queries, nq, query_format, radius, offsets, ids, dists, nullptr);
}

// Every image is checked on the host against its part before any part stages rows (multi_attach_rerank).
int granne_b200_multi_set_rerank_elements(granne_b200_multi* m, const void* const* elements_bytes,
                                          const size_t* elements_len) {
    if (!m || !elements_bytes || !elements_len) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    auto image = [&](size_t i) { return m->mode == GRANNE_B200_MODE_REPLICATED ? 0 : i; };
    return multi_attach_rerank(
        m,
        [&](size_t i) {
            if (!elements_bytes[image(i)]) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "elements buffer is null");
            gb::DenseView dv;
            std::string err;
            if (!gb::parse_dense(static_cast<const uint8_t*>(elements_bytes[image(i)]), elements_len[image(i)], 4, &dv,
                                 &err))
                return fail(GRANNE_B200_ERR_FORMAT, err);
            return check_rerank_shape(m->parts[i], dv.num, dv.dim);
        },
        [&](size_t i) {
            return granne_b200_set_rerank_elements(m->parts[i], elements_bytes[image(i)], elements_len[image(i)]);
        });
}

// One term-list image per part's shard (one for a replicated handle), one embedding table for all parts, as
// granne_b200_multi_open takes them; every image is checked on the host before any part stages (multi_attach_rerank).
int granne_b200_multi_set_rerank_embeddings(granne_b200_multi* m, const void* const* elements_bytes,
                                            const size_t* elements_len, const void* embeddings_bytes,
                                            size_t embeddings_len) {
    if (!m || !elements_bytes || !elements_len || !embeddings_bytes)
        return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "null argument");
    auto image = [&](size_t i) { return m->mode == GRANNE_B200_MODE_REPLICATED ? 0 : i; };
    return multi_attach_rerank(
        m,
        [&](size_t i) {
            gb::DenseView ev;
            gb::SumElements se;
            return check_rerank_sum(m->parts[i], elements_bytes[image(i)], elements_len[image(i)], embeddings_bytes,
                                    embeddings_len, &ev, &se);
        },
        [&](size_t i) {
            return granne_b200_set_rerank_embeddings(m->parts[i], elements_bytes[image(i)], elements_len[image(i)],
                                                     embeddings_bytes, embeddings_len);
        });
}

// RANGE_PARTITIONED: every shard re-ranks its own candidates; the shard lists are sorted by (distance, local id) and
// a shard's local ids are monotone in the global ids, so the (distance, global id) merge of multi_batch equals the
// re-rank of the union of the shards' candidate sets.
int granne_b200_multi_search_rerank_batch(granne_b200_multi* m, const float* queries, size_t nq, int query_format,
                                          uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                          uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_rerank(m->parts[0], queries, nq, query_format, max_search, num_candidates, num_neighbors,
                             out_ids, out_dists);
    if (rc || nq == 0) return rc;
    return multi_batch(m, queries, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                       [&](size_t i, size_t, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                           return granne_b200_search_rerank_batch(m->parts[i], static_cast<const float*>(q), cnt,
                                                                  query_format, max_search, num_candidates,
                                                                  num_neighbors, ids, ds, c, nullptr);
                       });
}

}  // extern "C"

namespace {

// The diverse search of a RANGE_PARTITIONED handle (arguments checked, nq > 0).  The candidates are the shards'
// max_search lists merged by (distance, global id), as granne_b200_multi_search_batch merges them, without the query's
// own global id for QUERY_ID_EXCLUDING.  select_neighbors then runs over the global container: the merged candidates'
// element rows are read from the shards that own them and staged on part 0's device as a temporary container (f32 rows
// re-laid out by permute_rows_f32_kernel, i8 rows padded by pad_rows_i8_kernel; a SumEmbeddings shard's materialised
// rows as angular f32 rows, whose f32 angular distances are its own), and the lists select there.
int multi_diverse_partitioned(granne_b200_multi* m, const void* queries, size_t nq, int fmt, uint32_t ms, uint32_t k,
                              uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
    return guarded([&] {
        const uint64_t* gids = by_id(fmt) ? static_cast<const uint64_t*>(queries) : nullptr;
        std::vector<uint8_t> id_rows;
        const void* rows = queries;
        int qfmt = fmt;
        int rc;
        if (gids) {
            MultiIds mi;
            if ((rc = multi_ids(m, gids, nq, &mi)) || (rc = multi_id_rows(m, mi, nq, &id_rows))) return rc;
            rows = id_rows.data();
            qfmt = GRANNE_B200_QUERY_ELEMENT;
        }
        std::vector<uint64_t> cand(nq * ms);
        std::vector<float> cd(nq * ms);
        std::vector<uint32_t> cc(nq);
        if ((rc = multi_batch(m, rows, nq, qfmt, ms, cand.data(), cd.data(), cc.data(),
                              [&](size_t i, size_t, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                                  return granne_b200_search_batch(m->parts[i], q, cnt, qfmt, ms, ms, ids, ds, c,
                                                                  nullptr);
                              })))
            return rc;
        // the lists as rows of the gathered container, each merged candidate once
        std::map<uint64_t, uint32_t> row_of;
        std::vector<uint64_t> gid_of;
        std::vector<uint32_t> lid(nq * ms, gb::kUnusedId);
        for (size_t q = 0; q < nq; ++q) {
            uint32_t r = 0;
            for (uint32_t j = 0; j < cc[q]; ++j) {
                const uint64_t g = cand[q * ms + j];
                if (fmt == GRANNE_B200_QUERY_ID_EXCLUDING && g == gids[q]) continue;
                const auto it = row_of.emplace(g, (uint32_t)gid_of.size()).first;
                if (it->second == gid_of.size()) gid_of.push_back(g);
                lid[q * ms + r] = it->second;
                cd[q * ms + r] = cd[q * ms + j];
                ++r;
            }
            cc[q] = r;
        }
        const uint64_t n = gid_of.size();
        const int kind = m->kind == GRANNE_B200_ANGULAR_INT ? GRANNE_B200_ANGULAR_INT : GRANNE_B200_ANGULAR;
        const size_t row = query_row_bytes(m->kind, m->dim, GRANNE_B200_QUERY_ELEMENT);
        std::vector<uint8_t> host_rows(std::max<uint64_t>(n, 1) * row);
        std::vector<uint32_t> local;
        std::vector<uint64_t> at;
        std::vector<uint8_t> part_rows;
        for (size_t s = 0; s < m->parts.size(); ++s) {
            local.clear();
            at.clear();
            for (uint64_t r = 0; r < n; ++r)
                if (gid_of[r] >= m->base[s] && gid_of[r] - m->base[s] < m->parts[s]->index_len &&
                    (s + 1 == m->parts.size() || gid_of[r] < m->base[s + 1])) {
                    local.push_back((uint32_t)(gid_of[r] - m->base[s]));
                    at.push_back(r);
                }
            if (local.empty()) continue;
            part_rows.resize(local.size() * row);
            if ((rc = granne_b200_get_elements(m->parts[s], local.data(), local.size(), part_rows.data()))) return rc;
            for (size_t j = 0; j < at.size(); ++j)
                std::memcpy(host_rows.data() + at[j] * row, part_rows.data() + j * row, row);
        }
        std::vector<uint32_t> sel(nq * k);
        std::vector<uint32_t> sc(nq, 0);
        if (n > 0) {
            DeviceGuard on(m->parts[0]->device);
            GB_CUDA(on.err);
            Buffer<uint8_t> d_rows;
            if ((rc = d_rows.grow(n * row, nullptr))) return rc;
            GB_CUDA(cudaMemcpy(d_rows.get(), host_rows.data(), n * row, cudaMemcpyHostToDevice));
            DeviceGuard guard;
            std::unique_ptr<Handle> t;
            if ((rc = new_handle(&guard, m->parts[0]->device, kind, nullptr, 0, nullptr, 0, d_rows.get(), n, m->dim,
                                 &t)))
                return rc;
            t->index_len = n;
            rc = granne_b200_select_neighbors_batch(t.get(), lid.data(), cd.data(), cc.data(), nq, ms, k, sel.data(),
                                                    out_dists, sc.data());
            GB_CUDA(cudaDeviceSynchronize());  // the temporary handle's work is done before it is freed
            if (rc) return rc;
        } else {
            std::fill(out_dists, out_dists + nq * k, std::numeric_limits<float>::infinity());
        }
        for (size_t q = 0; q < nq; ++q)
            for (uint32_t j = 0; j < k; ++j)
                out_ids[q * k + j] = j < sc[q] ? gid_of[sel[q * k + j]] : ~0ull;
        if (out_counts) std::memcpy(out_counts, sc.data(), nq * 4);
        return (int)GRANNE_B200_OK;
    });
}

}  // namespace

extern "C" {

// REPLICATED: each device runs granne_b200_search_diverse_batch on its slice of the queries (by id: the global ids are
// its local ids, so QUERY_ID_EXCLUDING drops the element itself on the device).  RANGE_PARTITIONED:
// multi_diverse_partitioned.
int granne_b200_multi_search_diverse_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids,
                                           float* out_dists, uint32_t* out_counts) {
    if (!m) return fail(GRANNE_B200_ERR_INVALID_ARGUMENT, "multi handle is null");
    int rc = validate_diverse(m->parts[0], queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists);
    if (rc || nq == 0) return rc;
    if (m->mode == GRANNE_B200_MODE_RANGE_PARTITIONED)
        return multi_diverse_partitioned(m, queries, nq, query_format, max_search, num_neighbors, out_ids, out_dists,
                                         out_counts);
    return guarded([&] {
        std::vector<uint32_t> local;
        const void* rows = queries;
        if (by_id(query_format)) {
            const uint64_t* gids = static_cast<const uint64_t*>(queries);
            MultiIds mi;
            const int e = multi_ids(m, gids, nq, &mi);
            if (e) return e;
            local.assign(gids, gids + nq);  // every id is < Index::len here
            rows = local.data();
        }
        return multi_batch(m, rows, nq, query_format, num_neighbors, out_ids, out_dists, out_counts,
                           [&](size_t i, size_t, const void* q, size_t cnt, uint32_t* ids, float* ds, uint32_t* c) {
                               return granne_b200_search_diverse_batch(m->parts[i], q, cnt, query_format, max_search,
                                                                       num_neighbors, ids, ds, c, nullptr);
                           });
    });
}

}  // extern "C"
