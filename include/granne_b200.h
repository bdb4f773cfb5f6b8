/* granne_b200.h — C ABI of the H100-native drop-in for granne's search path.
 *
 * granne (Rust, v0.5.2) exposes no C FFI; its boundary is the generic Rust API re-exported in src/lib.rs:80-86 and the
 * rust-cpython module in py/src/lib.rs.  This header is what a `extern "C"` shim on the reference side binds (see
 * INTEGRATION.md for the Rust/ctypes stubs).  Every entry point cites the reference interface it replaces; paths are
 * relative to the reference repository root.
 *
 * Conventions
 *  - plain pointers and sizes only; no C++/torch types; nothing unwinds across this boundary.
 *  - every function returning `int` returns GRANNE_B200_OK (0) or a negative status; a human readable message for
 *    the calling thread's last failure is available from granne_b200_last_error().
 *    The reference panics where this ABI returns a status (malformed file: src/index/io.rs:73; NaN distance:
 *    src/elements/angular.rs:70; max_search == 0: src/index/mod.rs:1019).
 *  - input buffers stay owned by the caller and may be released as soon as the call returns (the reference borrows
 *    them for the index lifetime, src/index/mod.rs:108-113); outputs are caller-allocated.
 *  - ids are u32 on this boundary (granne limits an index to 2^32-2 elements: src/lib.rs:7, src/index/mod.rs:27-28,420).
 *  - a handle may be used from several host threads for concurrent search calls; open/close must not race with them.
 *  - the CUDA device is mandatory: there is no CPU fallback behind this ABI.
 *  - every call runs on its handle's device and restores the calling thread's current CUDA device before it returns.
 */
#ifndef GRANNE_B200_H
#define GRANNE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GRANNE_B200_ABI_VERSION 2 /* 2: GRANNE_B200_STAT_FLAGS reports the answering pass; device-resident containers; multi handle */

/* status codes */
#define GRANNE_B200_OK 0
#define GRANNE_B200_ERR_INVALID_ARGUMENT (-1) /* null pointer, dim mismatch, max_search == 0, bad enum ... */
#define GRANNE_B200_ERR_FORMAT (-2)           /* not a granne index / elements file, or truncated */
#define GRANNE_B200_ERR_IO (-3)               /* file could not be opened/read */
#define GRANNE_B200_ERR_CUDA (-4)             /* CUDA runtime failure (message carries cudaGetErrorString) */
#define GRANNE_B200_ERR_NO_DEVICE (-5)        /* no usable sm_90 device: the library never falls back to the CPU */
#define GRANNE_B200_ERR_NOT_FINITE (-6)       /* a NaN distance occurred (the reference panics: angular.rs:70) */
#define GRANNE_B200_ERR_CAPACITY (-7)         /* exact-search workspace exhausted even on the slow path */
#define GRANNE_B200_ERR_OUT_OF_RANGE (-8)     /* idx / layer out of range */

/* Element kinds — the three ElementContainer implementations granne ships (src/elements/mod.rs:17-45):
 * angular::Vectors (src/elements/angular.rs), angular_int::Vectors (src/elements/angular_int.rs),
 * embeddings::SumEmbeddings (src/elements/embeddings/mod.rs:41-44).  Same strings as the Python binding's
 * `element_type` (py/src/lib.rs:186-208). */
#define GRANNE_B200_ANGULAR 0     /* "angular":     f32 rows, normalised                                  */
#define GRANNE_B200_ANGULAR_INT 1 /* "angular_int": i8 rows (quantised)                                   */
#define GRANNE_B200_EMBEDDINGS 2  /* "embeddings":  element = list of embedding ids, vector = normalised sum */

/* Query formats for search. */
#define GRANNE_B200_QUERY_RAW_F32 0 /* caller's raw f32 vector; the library builds the Element exactly like
                                       `Vector::from(Vec<f32>)`: normalise (angular.rs:55-61, math.rs:124-150) or
                                       quantise (angular_int.rs:19-45) — what the Python binding does per call
                                       (py/src/variants/index.rs:15-16,32-33,103-108). */
#define GRANNE_B200_QUERY_ELEMENT 1 /* already an `Elements::Element`: normalised f32 (angular, embeddings) or i8
                                       (angular_int) — what Rust callers of Granne::search pass. */

/* Per-query counters written to `out_stats` (4 x u64 per query).  n_dist / n_expand are exactly the number of
 * `dist_to_element` (src/index/mod.rs:1012,1027) and `get_neighbors` (:1025) calls the reference makes for the
 * same query, all layers included; they are parity-checked against the oracle and feed the roofline. */
#define GRANNE_B200_STAT_N_DIST 0
#define GRANNE_B200_STAT_N_EXPAND 1
#define GRANNE_B200_STAT_N_NEIGHBORS_READ 2 /* sum of the degrees of the expanded nodes */
#define GRANNE_B200_STAT_FLAGS 3            /* which pass answered the query: 0 = fast pass, 1 = retry pass (longer
                                               list, larger visited table), 2 = exact slow pass (global workspaces) */
#define GRANNE_B200_STATS_PER_QUERY 4

typedef struct granne_b200_index granne_b200_index; /* opaque: owns all device + host memory */

/* ABI version of the loaded library (== GRANNE_B200_ABI_VERSION). */
int granne_b200_abi_version(void);

/* Message describing the calling thread's most recent failure ("" if none). Never NULL. */
const char* granne_b200_last_error(void);

/* Replaces Granne::from_bytes(index, elements) (src/index/mod.rs:108-113) together with
 * Vectors::from_bytes (src/elements/dense_vector.rs:50-52) / SumEmbeddings::from_bytes
 * (src/elements/embeddings/mod.rs:56-61).
 *   index_bytes     granne index file image (src/index/io.rs:11-113)
 *   element_kind    GRANNE_B200_ANGULAR | _ANGULAR_INT | _EMBEDDINGS
 *   elements_bytes  elements file image: FixedWidthSliceVector<f32|i8> (src/slice_vector/mod.rs:213-221,460-466) or,
 *                   for EMBEDDINGS, VariableWidthSliceVector<ThreeByteInt,FiveByteInt> (:623-676)
 *   embeddings_*    EMBEDDINGS only: the FixedWidthSliceVector<f32> embedding table, else NULL/0
 *   device          CUDA device ordinal the index is staged on (layer graph + vectors are copied to HBM)
 * Like the reference, the index may cover fewer elements than the container holds (src/index/mod.rs:74-83). */
int granne_b200_open(const void* index_bytes, size_t index_len, int element_kind, const void* elements_bytes,
                     size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                     granne_b200_index** out);

/* Replaces Granne::from_file (src/index/mod.rs:122-135) + Vectors::from_file (dense_vector.rs:61-63) /
 * SumEmbeddings::from_files (embeddings/mod.rs:75-86); same argument order as the Python constructor
 * Granne(index_path, element_type, elements_path, embeddings_path) (py/src/lib.rs:175-211). */
int granne_b200_open_files(const char* index_path, int element_kind, const char* elements_path,
                           const char* embeddings_path, int device, granne_b200_index** out);

/* Drop of a `Granne` value. NULL is accepted. */
void granne_b200_close(granne_b200_index* h);

/* Index trait (src/index/mod.rs:54-104). */
uint64_t granne_b200_len(const granne_b200_index* h);                        /* Index::len        :76-83 */
uint64_t granne_b200_num_layers(const granne_b200_index* h);                 /* Index::num_layers :86-88 */
uint64_t granne_b200_layer_len(const granne_b200_index* h, uint64_t layer);  /* Index::layer_len  :91-93 */
/* Index::get_neighbors(index, layer) :96-98 — ascending ids, as MultiSetVector returns them. */
int granne_b200_get_neighbors(const granne_b200_index* h, uint64_t idx, uint64_t layer, uint32_t* out, size_t cap,
                              size_t* out_n);

/* ElementContainer (src/elements/mod.rs:17-45). */
uint64_t granne_b200_num_elements(const granne_b200_index* h); /* ElementContainer::len (may exceed Index::len) */
uint64_t granne_b200_dim(const granne_b200_index* h);          /* Vectors::dim (dense_vector.rs:107-109)        */
int granne_b200_element_kind(const granne_b200_index* h);
/* Granne::get_element (src/index/mod.rs:153-155) == ElementContainer::get: writes dim f32 (ANGULAR: the stored row;
 * EMBEDDINGS: the normalised sum, embeddings/mod.rs:164-166) or dim i8 (ANGULAR_INT) to `out`. */
int granne_b200_get_element(const granne_b200_index* h, uint64_t idx, void* out);

/* Replaces Granne::search(&self, &element, max_search, num_neighbors) -> Vec<(usize, f32)>
 * (src/index/mod.rs:140-150, 962-1037), for a batch of `nq` independent queries (the reference has no batch API;
 * a batch is nq sequential `search` calls, and a single query is nq == 1).
 *   queries        HOST pointer, nq x dim, row-major; f32 (RAW_F32, or ELEMENT for ANGULAR/EMBEDDINGS) or
 *                  i8 (ELEMENT for ANGULAR_INT)
 *   max_search     >= 1 (0 panics in the reference, src/index/mod.rs:1019)
 *   num_neighbors  results kept per query; like the reference at most max_search results exist (:974-977)
 *   out_ids        nq x num_neighbors u32, ascending by (distance, id); padded with 0xFFFFFFFF
 *   out_dists      nq x num_neighbors f32; padded with +inf
 *   out_counts     nq u32: number of valid results of each query (may be NULL)
 *   out_stats      nq x GRANNE_B200_STATS_PER_QUERY u64 (may be NULL)
 * Host<->device copies happen inside the call. Results are bit-identical to the reference algorithm (ids and f32
 * distances). */
int granne_b200_search_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                             uint32_t max_search, uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                             uint32_t* out_counts, uint64_t* out_stats);

/* Same, with DEVICE pointers (on the index's device) and an optional cudaStream_t (NULL = the default stream);
 * asynchronous with respect to the host: the caller synchronises the stream before reading the outputs and before
 * calling granne_b200_stream_status(). */
int granne_b200_search_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                    uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids,
                                    float* d_out_dists, uint32_t* d_out_counts, uint64_t* d_out_stats,
                                    void* cuda_stream);

/* Multi-GPU result gather fused into the search kernels (replicated index, query batch sharded over GPUs, SURVEY.md §8e
 * mode 1).  `ids[p]` / `dists[p]` are device pointers, valid on THIS device, to the gathered result buffers of peer p
 * (peer-mapped memory, e.g. torch symmetric memory or cudaIpc/cuMem mappings; entry `my_rank` is this GPU's own
 * buffer), each [total_queries][num_neighbors].  The kernels store the rows of this call at row `row_offset + i` of
 * every peer buffer over NVLink — no collective, no rendezvous — and, when every store is done, release
 * `flags[p][my_rank] = seq` system-wide. */
#define GRANNE_B200_MAX_PEERS 8
typedef struct granne_b200_peer_gather {
    uint32_t n_peers; /* 1..8 */
    uint32_t my_rank;
    uint64_t row_offset;
    uint32_t seq;
    uint32_t reserved;
    void* ids[GRANNE_B200_MAX_PEERS];   /* u32 [total_queries][k] */
    void* dists[GRANNE_B200_MAX_PEERS]; /* f32 [total_queries][k] */
    void* flags[GRANNE_B200_MAX_PEERS]; /* u32 [n_peers] per peer */
} granne_b200_peer_gather;
/* granne_b200_search_batch_device with the results delivered through `gather` instead of d_out_ids/d_out_dists. */
int granne_b200_search_batch_device_gather(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_neighbors,
                                           const granne_b200_peer_gather* gather, uint32_t* d_out_counts,
                                           uint64_t* d_out_stats, void* cuda_stream);

/* The device-pointer calls keep one workspace per distinct caller stream (status words, per-warp visited tables) until
 * granne_b200_close.  A caller that retires a stream returns its workspace with this call (it synchronises the stream;
 * an error raised by its last batches is reported by the next granne_b200_stream_status). */
int granne_b200_release_stream(granne_b200_index* h, void* cuda_stream);

/* After synchronising a stream used with granne_b200_search_batch_device: GRANNE_B200_OK, or the first error
 * (ERR_NOT_FINITE / ERR_CAPACITY) any query of the calls issued since the previous check raised. */
int granne_b200_stream_status(granne_b200_index* h);

/* Range-partitioned mode (SURVEY.md §8e mode 2; granne shards elements into independent indexes,
 * src/elements/embeddings/parsing.rs:63-100): merges `num_parts` per-shard result tiles into the global top-k, ordered by
 * (distance, global id) — the tuple order of into_sorted_vec (src/index/mod.rs:1036).
 *   d_part_ids/dists  DEVICE, [num_parts][nq][k]; ids are shard-local, padded with 0xFFFFFFFF
 *   part_base         HOST, num_parts u64: global id of each shard's element 0
 *   d_out_ids         DEVICE, [nq][k] u64 global ids (padded with UINT64_MAX); d_out_dists [nq][k] f32 */
int granne_b200_merge_topk_device(int device, const uint32_t* d_part_ids, const float* d_part_dists,
                                  const uint64_t* part_base, size_t num_parts, size_t nq, uint32_t k,
                                  uint64_t* d_out_ids, float* d_out_dists, void* cuda_stream);

/* ---- several GPUs behind one handle (SURVEY.md §8b "Load" row: device list + mode; §8e) ------------------------------
 * For callers without torch / NCCL (a Rust or C++ host): one process drives all the devices.  Queries are independent
 * (`search` takes &self, src/index/mod.rs:140-150), so neither mode has a data-path collective.
 *   GRANNE_B200_MODE_REPLICATED        one index image, staged on every listed device; a query batch is split into
 *                                      contiguous slices, one per device; results are identical to a single device.
 *   GRANNE_B200_MODE_RANGE_PARTITIONED num_shards independent (index, elements) pairs — granne's own sharding of the
 *                                      element set (src/elements/embeddings/parsing.rs:63-100) — shard s staged on
 *                                      devices[s % num_devices]; every query is searched on every shard and the
 *                                      per-shard lists are merged by (distance, global id), the order of
 *                                      into_sorted_vec (src/index/mod.rs:1036); global id = shard_base[s] + local id.
 * `devices` may name a device more than once (several shards per GPU).  index/elements arrays hold num_shards
 * entries (1 for REPLICATED); the embeddings table (EMBEDDINGS kind) is shared by all shards. */
#define GRANNE_B200_MODE_REPLICATED 0
#define GRANNE_B200_MODE_RANGE_PARTITIONED 1
typedef struct granne_b200_multi granne_b200_multi;
int granne_b200_multi_open(int mode, const int* devices, size_t num_devices, int element_kind,
                           const void* const* index_bytes, const size_t* index_len,
                           const void* const* elements_bytes, const size_t* elements_len, size_t num_shards,
                           const void* embeddings_bytes, size_t embeddings_len, granne_b200_multi** out);
void granne_b200_multi_close(granne_b200_multi* m);
/* Index::len over all shards (replicated: of the one index). */
uint64_t granne_b200_multi_len(const granne_b200_multi* m);
/* number of staged single-device handles (devices for REPLICATED, shards for RANGE_PARTITIONED) */
size_t granne_b200_multi_num_parts(const granne_b200_multi* m);
/* global id of shard s's element 0 (0 for REPLICATED) */
uint64_t granne_b200_multi_shard_base(const granne_b200_multi* m, size_t s);
/* Granne::search for nq queries (HOST buffers, as granne_b200_search_batch); out_ids are u64 GLOBAL ids padded with
 * UINT64_MAX, out_dists padded with +inf, out_counts may be NULL.  Thread-safe like the single-device call. */
int granne_b200_multi_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                   uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                   uint32_t* out_counts);

/* Host-only helpers (no device needed): the loader's view of an index image.
 * granne_b200_inspect_index replaces io::read_layer_sizes + Index::num_layers/layer_len on raw bytes
 * (src/index/io.rs:89-113): writes the number of layers and, for up to `cap` layers, the node count, the maximum
 * out-degree and the staging row width (u32 per row, padded with 0xFFFFFFFF).
 * granne_b200_decode_layer decodes every neighbour list of one layer (MultiSetVector::get, set_vector.rs:57-115)
 * into fixed-width rows — exactly the layout that is copied to HBM.  `rows` must hold layer_len*width u32. */
int granne_b200_inspect_index(const void* index_bytes, size_t index_len, uint64_t* out_num_layers,
                              uint64_t* out_layer_len, uint32_t* out_max_degree, uint32_t* out_row_width, size_t cap);
int granne_b200_decode_layer(const void* index_bytes, size_t index_len, uint64_t layer, uint32_t* rows,
                             size_t rows_cap_u32);

/* ---- GranneBuilder (SURVEY.md §8f rows 1-2) --------------------------------------------------------------------------
 * GPU-side construction of the index: the reference's GranneBuilder (src/index/mod.rs:295-531, 645-960) with the
 * insertions of a layer issued in batches (the reference issues them through rayon, :773-783).  Candidate search is
 * the same kernel that serves granne_b200_search_batch; select_neighbors / connect_nodes / add_and_limit_neighbors run
 * as device kernels with the reference's exact arithmetic.  As with the reference's default (multi-threaded) build the
 * graph depends on the interleaving of concurrent insertions.  Two environment variables, read on every build call,
 * make it deterministic for testing:
 *   GRANNE_B200_BUILD_MAX_BATCH (default 4096) caps the insertion batch; at 1 every insertion sees all earlier links,
 *     and the build equals the oracle's single-threaded one (the reference's `singlethreaded` order) byte for byte.
 *   GRANNE_B200_BUILD_LINK_WARPS (default num_sms x 8) caps the warps that link a batch in; at 1 the batched build
 *     equals the oracle's model of this batch schedule byte for byte.
 * The default concurrent link phase also equals that model exactly when no row overflows and no selection drops a
 * candidate; with overflow it is checked through row invariants and recall. */

/* BuildConfig (src/index/mod.rs:198-291); granne_b200_build_config_default() fills the reference defaults (:220-231). */
typedef struct granne_b200_build_config {
    float layer_multiplier;        /* 15.0 */
    int64_t expected_num_elements; /* < 0 == None */
    uint32_t num_neighbors;        /* 30; 1..255 (the file format counts a list in one byte) */
    uint32_t max_search;           /* 200 */
    int32_t reinsert_elements;     /* 1 */
    int32_t show_progress;         /* accepted for compatibility, ignored */
} granne_b200_build_config;
void granne_b200_build_config_default(granne_b200_build_config* cfg);

typedef struct granne_b200_builder granne_b200_builder;

/* GranneBuilder::new(config, elements) (:419-426).  Element buffers as in granne_b200_open. */
int granne_b200_builder_new(const granne_b200_build_config* cfg, int element_kind, const void* elements_bytes,
                            size_t elements_len, const void* embeddings_bytes, size_t embeddings_len, int device,
                            granne_b200_builder** out);
/* GranneBuilder::new(config, elements) with the element container given as device rows (see "device-resident element
 * containers" below: row-major elements, num_elements x dim, memory of `device`). */
int granne_b200_builder_new_device_elements(const granne_b200_build_config* cfg, int element_kind,
                                            const void* d_element_rows, uint64_t num_elements, uint32_t dim,
                                            int device, granne_b200_builder** out);
/* GranneBuilder::push (src/index/mod.rs:512-531; py GranneBuilder.append, py/src/lib.rs:474-476): appends the
 * elements of an elements file image of the builder's own kind to its container; they are indexed by the next build.
 * angular / angular_int: rows of the same width (ExtendableElementContainer for Vectors, dense_vector.rs:120-136);
 * embeddings: term lists over the unchanged embedding table (SumEmbeddings::push, embeddings/mod.rs:97-100,177-189).
 * Not concurrent with other calls on `b`. */
int granne_b200_builder_append(granne_b200_builder* b, const void* elements_bytes, size_t elements_len);
/* Builder::build_partial(num_elements) (:374-402); num_elements == 0 means Builder::build() (all elements, :366-368). */
int granne_b200_builder_build(granne_b200_builder* b, uint64_t num_elements);
uint64_t granne_b200_builder_len(const granne_b200_builder* b);        /* Index::len for the builder (:329-331) */
uint64_t granne_b200_builder_num_layers(const granne_b200_builder* b); /* :334-336 */
uint64_t granne_b200_builder_layer_len(const granne_b200_builder* b, uint64_t layer);
/* Builder::num_elements (src/index/mod.rs:404-406): elements held by the builder, indexed or not. */
uint64_t granne_b200_builder_num_elements(const granne_b200_builder* b);
/* Index::get_neighbors for the builder (:339-349); same contract as granne_b200_get_neighbors. */
int granne_b200_builder_get_neighbors(const granne_b200_builder* b, uint64_t idx, uint64_t layer, uint32_t* out,
                                      size_t cap, size_t* n_out);
/* Index::write_index (:358-361, src/index/io.rs:11-70): the granne index file image (compressed layers).  Call with
 * out == NULL to query the size; the image is readable by granne itself and by granne_b200_open. */
int granne_b200_builder_write_index(granne_b200_builder* b, void* out, size_t cap, size_t* out_len);
/* GranneBuilder::get_index (:483-488): a searchable snapshot sharing the staged elements (no file round trip).
 * Close it with granne_b200_close; it stays valid after further builder calls and after the builder is freed. */
int granne_b200_builder_get_index(granne_b200_builder* b, granne_b200_index** out);
void granne_b200_builder_free(granne_b200_builder* b);

/* Element construction on the device: `angular::Vector::from(Vec<f32>)` per row — normalise (angular.rs:55-61,
 * math.rs:124-150) or quantise to i8 (angular_int.rs:28-45) — written as an elements file image
 * (FixedWidthSliceVector::write, src/slice_vector/mod.rs:460-466: u64 dim + rows).  kind: ANGULAR or ANGULAR_INT.
 * Call with out == NULL to query the size. */
int granne_b200_elements_from_raw(int element_kind, const float* raw, uint64_t n, uint32_t dim, int device, void* out,
                                  size_t cap, size_t* out_len);

/* ---- device-resident element containers ---------------------------------------------------------------------------
 * The reference borrows its element container from the caller (`Vectors::from_slice`, src/elements/dense_vector.rs:
 * 66-72; `Granne::from_bytes(index, &elements)`, src/index/mod.rs:108-113).  When the rows are already in HBM (made
 * by another kernel, or too large to bounce through the host: 100M x 128 f32 = 51 GB) these variants take them as a
 * device pointer: row-major ELEMENTS (normalised f32 for ANGULAR, i8 for ANGULAR_INT), num_elements x dim, memory of
 * `device`.  The rows are copied into the staged layout during the call; the caller keeps its buffer. */

/* Vector::from per row (angular.rs:55-61 / angular_int.rs:28-45), device to device, asynchronous on `cuda_stream`:
 * d_raw = n x dim raw f32 rows, d_out = n x dim elements (f32 or i8). */
int granne_b200_elements_from_raw_device(int element_kind, const float* d_raw, uint64_t n, uint32_t dim, int device,
                                         void* d_out, void* cuda_stream);

/* Granne::from_bytes (src/index/mod.rs:108-113) with the element container given as device rows. */
int granne_b200_open_device_elements(const void* index_bytes, size_t index_len, int element_kind,
                                     const void* d_element_rows, uint64_t num_elements, uint32_t dim, int device,
                                     granne_b200_index** out);

/* compute_distance (py/src/lib.rs:71-89) for n pairs: out[i] = Vector::from(a_i).dist(&Vector::from(b_i)) for
 * GRANNE_B200_ANGULAR (src/elements/angular.rs:55-74) or GRANNE_B200_ANGULAR_INT (angular_int.rs:19-59); `a`, `b` are
 * n x dim raw f32 rows on the host.  A NaN distance (the reference panics) returns GRANNE_B200_ERR_NOT_FINITE. */
int granne_b200_compute_distances(int element_kind, const float* a, const float* b, uint64_t n, uint32_t dim, int device,
                                  float* out);

/* Index::write_index (src/index/io.rs:11-70; py Granne.save_index, py/src/lib.rs:325-329) for a loaded or
 * builder-snapshot index: the granne index file image written from the staged rows.  out == NULL queries the size. */
int granne_b200_write_index(const granne_b200_index* h, void* out, size_t cap, size_t* out_len);

/* Host-only: decodes an index image and writes it again with this library's writer (Index::write_index,
 * src/index/io.rs:11-70).  For an image written by granne (sorted lists, same coding rules) the output is byte-identical
 * to the input; used to test the writer without a device.  Call with out == NULL to query the size. */
int granne_b200_reencode_index(const void* index_bytes, size_t index_len, void* out, size_t cap, size_t* out_len);

/* ---- Granne::reorder / reorder_by_keys (src/index/reorder.rs:59-174) ---------------------------------------------
 * An order is `order[i] == j`: the node and element at old index j move to index i (reorder.rs:66-67). */

/* Granne::compute_order (reorder.rs:126-174): for every element above the first layer, the trail of closest nodes in
 * the layers above it (find_entrypoint_trail, reorder.rs:180-207 — max_search = 1 searches from node 0), computed as
 * batches of the search kernel; then the per-layer sort by (trail, idx).  `order_out` holds Index::len entries.  Like
 * the reference's `&mut self`, not to be called concurrently with searches on `h`. */
int granne_b200_compute_order(granne_b200_index* h, uint64_t* order_out, uint64_t cap);

/* Host-only.  The sort half of compute_order (reorder.rs:133-166) for trails computed elsewhere: `trails` is n rows of
 * 8 node ids, row idx = find_entrypoint_trail of element idx (entries past min(8, first layer of idx) ignored). */
int granne_b200_order_from_trails(const uint64_t* layer_lens, uint32_t num_layers, const uint32_t* trails, uint64_t n,
                                  uint64_t* order_out);

/* Host-only.  The ordering part of Granne::reorder_by_keys (reorder.rs:96-108): a layer-preserving sort by
 * (key, idx); `keys` is num_keys rows of key_width u64 compared lexicographically. */
int granne_b200_order_by_keys(const void* index_bytes, size_t index_len, const uint64_t* keys, uint64_t num_keys,
                              uint32_t key_width, uint64_t* order_out);

/* Host-only.  embeddings::compute_keys_for_reordering (src/elements/embeddings/reorder.rs:31-58): keys_out holds
 * num_elements rows of 8 u64 (embedding ids by decreasing norm, zero padded). */
int granne_b200_embedding_reorder_keys(const void* elements_bytes, size_t elements_len, const void* embeddings_bytes,
                                       size_t embeddings_len, uint64_t* keys_out);

/* Host-only.  reorder_layers (reorder.rs:209-292) + Permutable::permute (src/slice_vector/mod.rs:437-458,
 * src/elements/embeddings/mod.rs:191-217): writes the reordered index file image and the permuted elements file image.
 * Call with both output pointers NULL to query the sizes.  An order that is not a layer-preserving permutation (the
 * reference panics) returns GRANNE_B200_ERR_INVALID_ARGUMENT. */
int granne_b200_apply_order(const void* index_bytes, size_t index_len, int element_kind, const void* elements_bytes,
                            size_t elements_len, const uint64_t* order, uint64_t n, void* out_index, size_t index_cap,
                            size_t* index_out_len, void* out_elements, size_t elements_cap, size_t* elements_out_len);

/* Number of kernels this library launched on behalf of `h` since it was opened (bench.py's gpu_launches). */
uint64_t granne_b200_launch_count(const granne_b200_index* h);

/* Bytes of device memory the staged index occupies (layer graph + vectors). */
uint64_t granne_b200_device_bytes(const granne_b200_index* h);

#ifdef __cplusplus
}
#endif
#endif /* GRANNE_B200_H */
