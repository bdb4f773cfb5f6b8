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
#define GRANNE_B200_QUERY_ID 2      /* nq u32 element ids (u64 global ids on a multi handle): the query of row q is
                                       Granne::get_element(ids[q]) (src/index/mod.rs:153-155), how the reference's
                                       examples and self-recall tests search (examples/glove.rs).  The result is
                                       bit-identical to the same call with those rows as QUERY_ELEMENT (ids, distance
                                       bits, counts, stats columns 0..2).  An id must be < granne_b200_num_elements
                                       (the container: ids in [Index::len, num_elements) of a builder snapshot are valid
                                       queries).  Host calls check every id before any device call and return
                                       GRANNE_B200_ERR_OUT_OF_RANGE; in device calls a query with a bad id gets count 0,
                                       padding and zero stats, the others are unaffected, and granne_b200_stream_status
                                       reports ERR_OUT_OF_RANGE.  Accepted by search_batch, exact_search_batch,
                                       exact_search_within_batch, search_filtered_batch,
                                       exact_search_filtered_batch, exact_range_count and exact_range_search (host
                                       and device forms, and their multi-handle forms) and search_diverse_batch (host
                                       and device forms, and its multi-handle form);
                                       search_batch_device_gather and the two-stage calls reject it as an unknown
                                       format. */
#define GRANNE_B200_QUERY_ID_EXCLUDING 3 /* QUERY_ID without the element itself: the call's result for the same query
                                       with num_neighbors = k + 1, the entry whose id is ids[q] removed, cut to the first
                                       k.  Other elements at distance 0 (duplicates) stay.  Stats columns 0..2 are
                                       QUERY_ID's.  The calls capped at GRANNE_B200_EXACT_MAX_K then take k <= 1023.
                                       The range calls remove ids[q] from the query's range if it is there (its count
                                       and segment shrink by one); other elements at distance 0 stay. */

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
/* granne_b200_get_element for n ids in one launch: row i of `out` (n x dim, f32 or i8 as above) is bit for bit what
 * granne_b200_get_element writes for ids[i].  Every id must be < granne_b200_num_elements(h): the host call checks them
 * all before any device call (GRANNE_B200_ERR_OUT_OF_RANGE).  n == 0 is valid; ids and out may be NULL then. */
int granne_b200_get_elements(granne_b200_index* h, const uint32_t* ids, size_t n, void* out);
/* Same with DEVICE pointers on cuda_stream (NULL = the default stream), asynchronous like
 * granne_b200_search_batch_device.  The kernel checks the ids: a bad id's row is zeros and granne_b200_stream_status
 * reports ERR_OUT_OF_RANGE. */
int granne_b200_get_elements_device(granne_b200_index* h, const uint32_t* d_ids, size_t n, void* d_out,
                                    void* cuda_stream);

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
 * `flags[p][my_rank] = seq` system-wide.  Every successful call publishes `seq`, including one with nq == 0 (no row is
 * stored) or num_neighbors == 0 (no column is stored); a call rejected for its arguments touches no buffer or flag. */
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

/* ---- exact k-nearest neighbours -------------------------------------------------------------------------------------
 * NOT a reference function: the reference's distance and result order applied to every element, the ground truth the
 * approximate search is measured against (recall).  For n = granne_b200_len(h) (Index::len) and a query q the result is
 * the first min(k, n) entries of
 *     sort ascending { (dist_to_element(q, i), i) : 0 <= i < n }
 * with dist_to_element the reference's distance of the handle's element kind (src/index/mod.rs:1012; angular.rs:63-74,
 * math.rs:16-42; angular_int.rs:47-59; embeddings/mod.rs:164-174), bit for bit, and the (NotNan<f32>, usize) order of
 * into_sorted_vec (src/index/mod.rs:1036).  Elements past Index::len (a container larger than the index) are never
 * returned: this is the set granne_b200_search_batch can return.  If max_search >= n and every bottom-layer node is
 * reachable from the entry point, the reference's search expands every node and returns exactly this answer.
 *   queries        as granne_b200_search_batch (RAW_F32 normalised / quantised, or ELEMENT); there is no max_search
 *   num_neighbors  k, 0..GRANNE_B200_EXACT_MAX_K; more is ERR_INVALID_ARGUMENT
 *   out_ids        nq x k u32, padded with 0xFFFFFFFF; out_dists nq x k f32, padded with +inf
 *   out_counts     nq u32 (may be NULL): min(k, n), so 0 when k == 0 or n == 0
 * nq == 0, k == 0 and n == 0 are valid; no element is read when k == 0 or n == 0.  A NaN distance returns
 * GRANNE_B200_ERR_NOT_FINITE, as in search; the exact scan meets every element, so a single NaN element makes every call
 * with nq > 0, k > 0 fail (search may step around it).  Argument checks run on the host before any device call.  Safe
 * concurrently with the search calls on the same handle. */
#define GRANNE_B200_EXACT_MAX_K 1024
int granne_b200_exact_search_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                   uint32_t num_neighbors, uint32_t* out_ids, float* out_dists, uint32_t* out_counts);
/* Same with DEVICE pointers and an optional cudaStream_t (NULL = the default stream), asynchronous like
 * granne_b200_search_batch_device: it uses that stream's workspace, and ERR_NOT_FINITE is reported by
 * granne_b200_stream_status after the stream is synchronised. */
int granne_b200_exact_search_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                          uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                          uint32_t* d_out_counts, void* cuda_stream);

/* ---- exact search within caller-given candidate lists ---------------------------------------------------------------
 * NOT a reference function: the exact answer within a list of ids per query — a restricted search (ids admitted by a
 * category, tenant, time range or ACL), the ranking of a lexical engine's candidates, the union of several indexes'
 * results, or ground truth inside a subset.  For n = granne_b200_len(h) (Index::len), a query q and its list L_q of
 * u32 ids the result is the first min(k, |set(L_q)|) entries of
 *     sort ascending { (dist_to_element(q, i), i) : i in set(L_q) }
 * with dist_to_element and the order exactly as in granne_b200_exact_search_batch (an angular_int handle ranks by its
 * i8 distance).  The result depends only on the set of ids, not on their order or multiplicity.  L_q = [0, n) gives
 * granne_b200_exact_search_batch(q, k); L_q = the ids of granne_b200_search_batch(q, ef, ef) gives
 * granne_b200_search_batch(q, ef, k) for k <= ef.
 *   queries        as granne_b200_exact_search_batch (RAW_F32 or ELEMENT)
 *   offsets        nq + 1 u64, offsets[0] == 0, non-decreasing: L_q = ids[offsets[q], offsets[q + 1])
 *   ids            offsets[nq] u32 ids, each < n (ids in [n, num_elements) of a container larger than its index are
 *                  rejected too); may be NULL when offsets[nq] == 0
 *   num_neighbors  k, 0..GRANNE_B200_EXACT_MAX_K
 *   out_*          as granne_b200_exact_search_batch; out_counts[q] = min(k, |set(L_q)|)
 * nq == 0, k == 0 and empty lists are valid.  Only listed elements are read: a NaN distance of a listed element (or a
 * NaN query with a non-empty list and k > 0) returns ERR_NOT_FINITE; one of an element no list names does not.
 * ERR_INVALID_ARGUMENT, in this order: a rule of granne_b200_exact_search_batch; offsets NULL with nq > 0; ids NULL with
 * offsets[nq] > 0; offsets that do not start at 0 or go backwards; an id >= n.  The host call checks all of them on
 * the host before any device call; its lists are copied to the device with the queries, in the one round trip of the
 * call, into memory held only until the call's kernels have run.  Workspace is bounded (query chunks of 1024, k keys per query) whatever the lists' lengths. */
int granne_b200_exact_search_within_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                          const uint64_t* offsets, const uint32_t* ids, uint32_t num_neighbors,
                                          uint32_t* out_ids, float* out_dists, uint32_t* out_counts);
/* Same with DEVICE pointers (queries, offsets, ids, outputs) on cuda_stream (NULL = the default stream), asynchronous
 * like granne_b200_exact_search_batch_device and without a host synchronisation.  The host checks the arguments up to
 * offsets NULL; the kernels check the offsets and the ids: a bad list writes count 0 and padding for its query, and
 * granne_b200_stream_status reports ERR_INVALID_ARGUMENT (ERR_NOT_FINITE for a NaN distance). */
int granne_b200_exact_search_within_batch_device(granne_b200_index* h, const void* d_queries, size_t nq,
                                                 int query_format, const uint64_t* d_offsets, const uint32_t* d_ids,
                                                 uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                                 uint32_t* d_out_counts, void* cuda_stream);

/* ---- filtered search: the k nearest admitted elements among those the graph search scores ---------------------------
 * NOT a reference function: granne_b200_search_batch's traversal, unchanged, with its scored candidates filtered by an
 * id bitmap — a tenant's, a category's or an ACL's ids.  For a query q let B be the bottom layer and S(q) the elements
 * whose distance granne_b200_search_batch(q, max_search) computes in B: B's entry point and every layer-B neighbour of
 * every element its layer-B search expands.  With A the ids the query's filter admits, the result is the first
 * min(k, |S(q) ∩ A|) elements of S(q) ∩ A ordered by (distance, id), distances as the handle's search computes them,
 * bit for bit.  The expansions, the visited set and stats columns 0..2 (n_dist, n_expand, n_nbr) are
 * granne_b200_search_batch's for the same query and max_search, whatever the filter; a larger max_search widens S(q).
 * Every element of S(q) strictly closer than the last of search_batch(q, max_search, max_search) is among its results,
 * so an all-admitting filter returns search_batch(q, max_search, k) (k <= max_search) whenever that call's k-th
 * distance is strictly below its max_search-th, or it returns fewer than max_search results.  There
 * is no exact fallback: a selective filter may return fewer than k (granne_b200_exact_search_filtered_batch returns
 * the exact answer over the same bitmaps).
 *   filters        num_filters bitmaps of filter_words u32 words each, bitmap f at filters + f * filter_words; id i is
 *                  admitted by filter f iff bit i % 32 (LSB first) of word i / 32 of bitmap f is set.  Bits at or
 *                  beyond Index::len are ignored.
 *   filter_words   >= ceil(Index::len / 32)
 *   query_filter   nq u32 in [0, num_filters): the filter of each query; NULL: every query uses filter 0
 *   num_neighbors  k, 0..GRANNE_B200_EXACT_MAX_K; k may exceed max_search
 *   out_*          as granne_b200_search_batch (ids padded with 0xFFFFFFFF, dists with +inf); out_stats' column 3 is
 *                  the answering pass of the filtered call's own ladder
 * ERR_INVALID_ARGUMENT, in this order: the handle is NULL; an unknown query format; max_search == 0; k >
 * GRANNE_B200_EXACT_MAX_K; nq above the batch limit; a NULL queries or output buffer; then, when nq > 0: filters NULL or
 * num_filters == 0; filter_words < ceil(Index::len / 32); and (host call) a query_filter entry >= num_filters.  The
 * host call checks all of them before any device call and copies the filters and query_filter to the device in its one
 * round trip, into memory held only until its kernels have run.  ERR_NOT_FINITE / ERR_CAPACITY as in search. */
int granne_b200_search_filtered_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                      uint32_t max_search, uint32_t num_neighbors, const uint32_t* filters,
                                      uint32_t num_filters, uint64_t filter_words, const uint32_t* query_filter,
                                      uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint64_t* out_stats);
/* Same with DEVICE pointers (queries, filters, query_filter, outputs) on cuda_stream (NULL = the default stream),
 * asynchronous like granne_b200_search_batch_device.  The host checks the rules up to filter_words; the kernel checks
 * query_filter: a query whose entry is >= num_filters gets count 0 and padding, and granne_b200_stream_status reports
 * ERR_INVALID_ARGUMENT. */
int granne_b200_search_filtered_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                             uint32_t max_search, uint32_t num_neighbors, const uint32_t* d_filters,
                                             uint32_t num_filters, uint64_t filter_words,
                                             const uint32_t* d_query_filter, uint32_t* d_out_ids, float* d_out_dists,
                                             uint32_t* d_out_counts, uint64_t* d_out_stats, void* cuda_stream);

/* ---- exact filtered k-nearest neighbours: the k nearest elements an id bitmap admits --------------------------------
 * NOT a reference function: the exact answer of a filtered search — a small tenant's, a rare category's or an ACL's
 * nearest elements, and the ground truth filtered search is measured against.  For n = granne_b200_len(h)
 * (Index::len), a query q with filter f(q) (query_filter[q], or 0 when query_filter is NULL) and
 *     A_f = { i < n : bit i of bitmap f is set }
 * (filtered search's bitmaps, bit order and layout; bits at or beyond n are ignored) the result of q is the first
 * min(k, |A_f(q)|) entries of
 *     sort ascending { (dist_to_element(q, i), i) : i in A_f(q) }
 * with granne_b200_exact_search_batch's distance bits and (distance, id) order.  An all-admitting filter gives
 * granne_b200_exact_search_batch(q, k); the bitmap of a list L gives granne_b200_exact_search_within_batch(q, L, k).
 * Ids in [n, num_elements) of a container larger than its index are never returned.
 *   queries        as granne_b200_exact_search_batch (RAW_F32, ELEMENT, QUERY_ID or QUERY_ID_EXCLUDING; the last runs
 *                  k + 1 and drops the query's own id, which is there only when its filter admits it)
 *   filters, num_filters, filter_words, query_filter   as granne_b200_search_filtered_batch
 *   num_neighbors  k, 0..GRANNE_B200_EXACT_MAX_K; there is no max_search
 *   out_*          as granne_b200_exact_search_batch; out_counts[q] = min(k, |A_f(q)|)
 * nq == 0, k == 0 and empty filters are valid.  Only rows admitted by a filter some query of the call uses are read.
 * ERR_NOT_FINITE when some query q has a NaN distance to an element of A_f(q) (for angular_int: a NaN raw query with a
 * non-empty A_f(q)); a NaN element no query's filter admits, or a NaN query whose A_f(q) is empty, does not fail the
 * call.  ERR_INVALID_ARGUMENT, in this order: the handle is NULL; an unknown query format; k >
 * GRANNE_B200_EXACT_MAX_K; nq above the batch limit; a NULL queries or output buffer; then, when nq > 0: filters NULL
 * or num_filters == 0; QUERY_ID_EXCLUDING with k > 1023; filter_words < ceil(n / 32); and (host call) a query_filter
 * entry >= num_filters.  The host call checks them all before any device call and copies filters and query_filter up
 * in its one round trip, into memory held only until its kernels have run.
 * Cost: per query chunk (1024 queries) the rows of U, the union of the filters the chunk's queries name, plus 2F x n /
 * 32 bitmap words (F = the distinct filters the chunk names) and three small launches per list of up to a slab of ids
 * (65536 for a chunk of 1024 queries; ceil(n / (slab - 31)) lists, of which those past U's last id are empty) — not
 * the n rows of granne_b200_exact_search_batch.  A chunk whose queries share one filter scans exactly its admitted
 * rows, so callers with many distinct filters get the best grouping by ordering their queries by filter.  Workspace
 * is exact_search_batch's plus one list of ids per chunk, whatever n and the density. */
int granne_b200_exact_search_filtered_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                            const uint32_t* filters, uint32_t num_filters, uint64_t filter_words,
                                            const uint32_t* query_filter, uint32_t num_neighbors, uint32_t* out_ids,
                                            float* out_dists, uint32_t* out_counts);
/* Same with DEVICE pointers (queries, filters, query_filter, outputs) on cuda_stream (NULL = the default stream),
 * asynchronous like granne_b200_exact_search_batch_device and without a host synchronisation (the admitted counts stay
 * on the device).  The host checks the rules up to filter_words; the kernels check query_filter: a query whose entry
 * is >= num_filters gets count 0 and padding (its entry is never used as an index), the other queries are answered,
 * and granne_b200_stream_status reports ERR_INVALID_ARGUMENT. */
int granne_b200_exact_search_filtered_batch_device(granne_b200_index* h, const void* d_queries, size_t nq,
                                                   int query_format, const uint32_t* d_filters, uint32_t num_filters,
                                                   uint64_t filter_words, const uint32_t* d_query_filter,
                                                   uint32_t num_neighbors, uint32_t* d_out_ids, float* d_out_dists,
                                                   uint32_t* d_out_counts, void* cuda_stream);

/* ---- exact range search: every element within a distance bound -------------------------------------------------------
 * NOT a reference function: near-duplicate detection, threshold matching, density counts.  For n = granne_b200_len(h)
 * (Index::len), d(q, i) the distance of granne_b200_exact_search_batch (the same bits) and a radius r (f32):
 *     R(q) = { i : 0 <= i < n, d(q, i) <= r }
 * with IEEE <=, so r = +-0.0 admits distance 0 and r = +inf admits every element.  The result of q is R(q) sorted
 * ascending by (distance, id), the order of into_sorted_vec (src/index/mod.rs:1036), with no cap on its size; its first
 * min(k, |R(q)|) entries are the entries of granne_b200_exact_search_batch(q, k) whose distance is <= r.
 * Two phases, one radius per call:
 *   granne_b200_exact_range_count   counts[q] = |R(q)| (nq u64)
 *   granne_b200_exact_range_search  R(q) into ids[offsets[q], offsets[q + 1]) (u32) and dists[...] (f32), offsets being
 *                                   nq + 1 u64, offsets[0] == 0, non-decreasing: normally the exclusive prefix sum of
 *                                   the counts.  Distances are deterministic bit for bit, so both phases see the same
 *                                   sets.  A segment whose length differs from its query's count is padded whole with
 *                                   0xFFFFFFFF / +inf and the call reports ERR_INVALID_ARGUMENT (a device call through
 *                                   granne_b200_stream_status); nothing is written outside a query's own segment.
 * Queries are RAW_F32, ELEMENT, QUERY_ID or QUERY_ID_EXCLUDING (see GRANNE_B200_QUERY_ID).  With nq > 0 and n > 0 the
 * scan runs whatever r is, so a NaN distance returns ERR_NOT_FINITE as in granne_b200_exact_search_batch.  nq == 0 and
 * n == 0 are valid (all counts 0).  Argument checks run on the host before any device call; ERR_INVALID_ARGUMENT, in
 * this order: the handle is NULL; an unknown query format; a NaN radius; nq above the batch limit; queries NULL with
 * nq > 0; then, with nq > 0, counts NULL (count) or offsets NULL (search); and for the host search offsets that do not
 * start at 0 or go backwards, then ids or dists NULL with offsets[nq] > 0.  Then (host calls) an id >= num_elements is
 * ERR_OUT_OF_RANGE.
 * The scan is granne_b200_exact_search_batch's (query chunks of 1024, bounded row slabs, embeddings windows), so a
 * count costs about one exact scan and a search one more.  The search writes its entries straight into the caller's
 * segments and sorts each segment there, so its workspace is bounded (8 bytes per query of a chunk besides the scan's)
 * whatever the number of results; the host search stages its results in the handle's workspace, 8 bytes per result. */
int granne_b200_exact_range_count(granne_b200_index* h, const void* queries, size_t nq, int query_format, float radius,
                                  uint64_t* counts);
/* Same with DEVICE pointers on cuda_stream (NULL = the default stream), asynchronous like
 * granne_b200_exact_search_batch_device, with that stream's workspace and no host synchronisation.  A bad id gives its
 * query count 0 and granne_b200_stream_status reports ERR_OUT_OF_RANGE. */
int granne_b200_exact_range_count_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                         float radius, uint64_t* d_counts, void* cuda_stream);
int granne_b200_exact_range_search(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                   float radius, const uint64_t* offsets, uint32_t* ids, float* dists);
/* Same with DEVICE pointers (queries, offsets, outputs) on cuda_stream, asynchronous like
 * granne_b200_exact_range_count_device.  The kernels check the segments: offsets that go backwards write nothing,
 * NULL ids or dists take only empty segments, and either is reported as a length mismatch.  A bad id gives its query
 * an empty range (its segment must be empty) and granne_b200_stream_status reports ERR_OUT_OF_RANGE. */
int granne_b200_exact_range_search_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                          float radius, const uint64_t* d_offsets, uint32_t* d_ids, float* d_dists,
                                          void* cuda_stream);

/* ---- two-stage search: traverse angular_int rows, re-rank by exact f32 angular distance ----------------------------
 * NOT a reference function: what a user of granne assembles by hand from two containers over one index.  For an
 * angular_int handle h with an attached container F (angular rows or SumEmbeddings) and a raw f32 query q:
 *   1. S = Granne<angular_int::Vectors>::search(&angular_int::Vector::from(q), max_search, C), i.e. exactly
 *      granne_b200_search_batch(h, q, RAW_F32, max_search, C): at most min(C, max_search) ids;
 *   2. d_i = F.dist_to_element(i, &angular::Vector::from(q)) for i in S, over the attached container (angular rows or
 *      SumEmbeddings), the reference's f32 angular distance bit for bit (angular.rs:63-74, math.rs:16-42; for
 *      SumEmbeddings the ordered term sum and normalize_f32 first, embeddings/mod.rs:124-143,164-174, math.rs:92-150);
 *   3. the first min(k, |S|) entries of sort ascending { (d_i, i) }, the order of into_sorted_vec (src/index/mod.rs:1036).
 * The result depends only on the set S.  Per query, its intersection with the exact f32 top-k equals S's, so its
 * recall is the candidate set's and never below the i8 search's.  Output layout as granne_b200_search_batch.
 *
 * Attach F once, before searching; one container per handle, of either kind, with no replacement while searches may
 * be in flight, and an attach concurrent with a search on h is not supported.  Concurrent attaches on h are
 * serialised: one attaches its container, the others return ERR_INVALID_ARGUMENT.  The container is copied into HBM
 * (counted by granne_b200_device_bytes): angular rows in the layout the search path's f32 engine for their width
 * reads, a SumEmbeddings container as an EMBEDDINGS index stages it (table, offsets, term ids).
 * ERR_INVALID_ARGUMENT: h is not ANGULAR_INT, a container is already attached, its width differs from the index's, or
 * it holds fewer than granne_b200_len(h) elements.  ERR_FORMAT: a malformed image.  Every image check runs on the host
 * before any device call.
 *   elements_bytes   an angular elements file image (u64 dim | normalised f32 rows)
 *   d_rows           n x dim normalised f32 rows in device memory of h's device */
#define GRANNE_B200_RERANK_MAX_CANDIDATES 1024
int granne_b200_set_rerank_elements(granne_b200_index* h, const void* elements_bytes, size_t elements_len);
int granne_b200_set_rerank_elements_device(granne_b200_index* h, const float* d_rows, uint64_t n, uint32_t dim);
/* Attaches a SumEmbeddings container: the two images granne_b200_open takes for GRANNE_B200_EMBEDDINGS (the element
 * term lists, the embedding table).  Besides the rules above, ERR_INVALID_ARGUMENT for a table wider than 4096, and
 * ERR_FORMAT for a term id past the table.  A NaN distance in stage 2 returns ERR_NOT_FINITE from the search. */
int granne_b200_set_rerank_embeddings(granne_b200_index* h, const void* elements_bytes, size_t elements_len,
                                      const void* embeddings_bytes, size_t embeddings_len);
/* The two-stage search for nq raw f32 queries (host buffers).  ERR_INVALID_ARGUMENT, before any device call, when
 * query_format is not RAW_F32, no rows are attached, num_candidates is 0 or above GRANNE_B200_RERANK_MAX_CANDIDATES,
 * num_neighbors > num_candidates, or a rule of granne_b200_search_batch is broken.  out_stats (may be NULL) holds stage
 * 1's counters as granne_b200_search_batch writes them.  A NaN distance in either stage returns ERR_NOT_FINITE. */
int granne_b200_search_rerank_batch(granne_b200_index* h, const float* queries, size_t nq, int query_format,
                                    uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                    uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint64_t* out_stats);
/* Same with DEVICE pointers on cuda_stream (NULL = the default stream), asynchronous like
 * granne_b200_search_batch_device; ERR_NOT_FINITE is reported by granne_b200_stream_status. */
int granne_b200_search_rerank_batch_device(granne_b200_index* h, const float* d_queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                           uint32_t* d_out_ids, float* d_out_dists, uint32_t* d_out_counts,
                                           uint64_t* d_out_stats, void* cuda_stream);

/* ---- diverse search: the neighbours granne would link the query to -------------------------------------------------
 * NOT a reference function: GranneBuilder::select_neighbors (src/index/mod.rs:849-883) applied to a query's search
 * list, i.e. what index_element (:805-846) links an inserted element to.  For a query q:
 *   1. C = granne_b200_search_batch(h, q, max_search, max_search): at most max_search (id, distance) candidates in
 *      (distance, id) order; QUERY_ID_EXCLUDING drops the element itself (index_element's filter(id != idx), :822);
 *   2. if |C| <= k the result is C unpruned (:856-858); otherwise the candidates are walked in order and candidate j is
 *      kept when d(q, j) <= dist_to_element(s, get(j)) for every s kept before it, until k are kept (:864-880).
 * The result is up to k ids with their stage-1 distance bits, in candidate order, and a count; the k nearest that are
 * not near-duplicates of nearer ones, so on clustered data the answers differ from one another.  Output layout as
 * granne_b200_search_batch (padded with 0xFFFFFFFF / +inf); out_stats (may be NULL) holds stage 1's counters.  The
 * pair distances are the handle's own, bit for bit.  Costs stage 1 plus at most k x |C| pair distances per query.
 *   queries        every format of granne_b200_search_batch (QUERY_ID / QUERY_ID_EXCLUDING included)
 *   max_search     1..GRANNE_B200_DIVERSE_MAX_CANDIDATES
 * ERR_INVALID_ARGUMENT, in this order, before any device call: the handle is NULL; an unknown query format;
 * max_search == 0 or above GRANNE_B200_DIVERSE_MAX_CANDIDATES; nq above the batch limit; a NULL queries or output
 * buffer.  Then (host call) an id >= num_elements is ERR_OUT_OF_RANGE.  A NaN distance in either stage returns
 * ERR_NOT_FINITE (the query gets count 0). */
#define GRANNE_B200_DIVERSE_MAX_CANDIDATES 1024
int granne_b200_search_diverse_batch(granne_b200_index* h, const void* queries, size_t nq, int query_format,
                                     uint32_t max_search, uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                                     uint32_t* out_counts, uint64_t* out_stats);
/* Same with DEVICE pointers on cuda_stream (NULL = the default stream), asynchronous like
 * granne_b200_search_batch_device; errors are reported by granne_b200_stream_status. */
int granne_b200_search_diverse_batch_device(granne_b200_index* h, const void* d_queries, size_t nq, int query_format,
                                            uint32_t max_search, uint32_t num_neighbors, uint32_t* d_out_ids,
                                            float* d_out_dists, uint32_t* d_out_counts, uint64_t* d_out_stats,
                                            void* cuda_stream);
/* select_neighbors(list_q, k) over nq caller lists, the rule of granne_b200_search_diverse_batch's step 2: it composes
 * with the output of every query call (exact_search_batch(q, C) gives the exact diverse answer, the filtered calls a
 * diverse filtered one, exact_search_within_batch a diverse ranking of caller candidates).  List q is
 * cand_ids / cand_dists[q * stride, q * stride + cand_counts[q]): ids < granne_b200_len(h), distances ascending (taken
 * as given; the reference requires the order, :860-863).  Outputs as granne_b200_search_diverse_batch.
 * ERR_INVALID_ARGUMENT, in this order, before any device call: the handle is NULL; stride above
 * GRANNE_B200_DIVERSE_MAX_CANDIDATES; nq above the batch limit; with nq > 0, cand_counts NULL, an output NULL with
 * k > 0, or cand_ids / cand_dists NULL with stride > 0; then (host call) a count > stride, an id >= granne_b200_len(h),
 * or a list whose distances are not ascending (a NaN included).  nq == 0, k == 0 and empty lists are valid.  A NaN
 * pair distance returns ERR_NOT_FINITE. */
int granne_b200_select_neighbors_batch(granne_b200_index* h, const uint32_t* cand_ids, const float* cand_dists,
                                       const uint32_t* cand_counts, size_t nq, uint32_t stride,
                                       uint32_t num_neighbors, uint32_t* out_ids, float* out_dists,
                                       uint32_t* out_counts);
/* Same with DEVICE pointers on cuda_stream, asynchronous; it takes the (ids, dists, counts) outputs of any device query
 * call as they are (stride = that call's k).  The kernel checks the lists: a bad list gets count 0 and padding, and
 * granne_b200_stream_status reports ERR_INVALID_ARGUMENT. */
int granne_b200_select_neighbors_batch_device(granne_b200_index* h, const uint32_t* d_cand_ids,
                                              const float* d_cand_dists, const uint32_t* d_cand_counts, size_t nq,
                                              uint32_t stride, uint32_t num_neighbors, uint32_t* d_out_ids,
                                              float* d_out_dists, uint32_t* d_out_counts, void* cuda_stream);

/* The device-pointer calls keep one workspace per distinct caller stream (status words, per-warp visited tables) until
 * granne_b200_close.  A caller that retires a stream returns its workspace with this call (it synchronises the stream;
 * an error raised by its last batches is reported by the next granne_b200_stream_status). */
int granne_b200_release_stream(granne_b200_index* h, void* cuda_stream);

/* After synchronising a stream used with granne_b200_search_batch_device: GRANNE_B200_OK, or the first error
 * (ERR_NOT_FINITE / ERR_CAPACITY, or ERR_INVALID_ARGUMENT for a bad candidate list of
 * granne_b200_exact_search_within_batch_device or granne_b200_select_neighbors_batch_device, or a range search segment
 * whose length is not its count, or
 * ERR_OUT_OF_RANGE for an element id >= num_elements of a
 * GRANNE_B200_QUERY_ID* call or of granne_b200_get_elements_device) any query of the calls issued since the previous
 * check raised. */
int granne_b200_stream_status(granne_b200_index* h);
/* granne_b200_stream_status for one caller stream: synchronises cuda_stream only, and reports and clears the errors of
 * the calls issued on it since its previous check (GRANNE_B200_OK for a stream the handle has no workspace for).  The
 * other streams' errors stay for their own check, so a caller that shares the handle with other threads checks its
 * own work without consuming theirs. */
int granne_b200_stream_status_of(granne_b200_index* h, void* cuda_stream);

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
/* Index::len of part s (REPLICATED: every part's is the index's); its global ids are [shard_base, shard_base + this). */
uint64_t granne_b200_multi_part_len(const granne_b200_multi* m, size_t s);
/* Granne::search for nq queries (HOST buffers, as granne_b200_search_batch); out_ids are u64 GLOBAL ids padded with
 * UINT64_MAX, out_dists padded with +inf, out_counts may be NULL.  Thread-safe like the single-device call.
 * GRANNE_B200_QUERY_ID* queries on this and the three calls below are nq u64 GLOBAL ids, each in some part's
 * [shard_base, shard_base + Index::len) range (else ERR_OUT_OF_RANGE, checked on the host before any device call):
 * each query's row is read from the part that owns it and the call runs as QUERY_ELEMENT (with k + 1 columns and the
 * query's own global id removed for QUERY_ID_EXCLUDING). */
int granne_b200_multi_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                   uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                   uint32_t* out_counts);
/* granne_b200_exact_search_batch over a multi handle, with u64 GLOBAL ids like granne_b200_multi_search_batch.
 * REPLICATED slices the queries over the devices; RANGE_PARTITIONED runs the exact scan on every shard and merges by
 * (distance, global id): the exact answer over the union of the shards' Index::len ranges. */
int granne_b200_multi_exact_search_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                         uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                         uint32_t* out_counts);
/* granne_b200_exact_search_within_batch over a multi handle: u64 GLOBAL ids in the lists and in the results.
 * REPLICATED slices the queries together with their lists over the devices; RANGE_PARTITIONED routes each id to the
 * shard that owns it (shard_base[s] <= id < shard_base[s] + that shard's Index::len), runs every shard on its local
 * lists and merges by (distance, global id).  An id >= granne_b200_multi_len(m), or one in no shard's Index::len range,
 * is ERR_INVALID_ARGUMENT, checked on the host before any device call. */
int granne_b200_multi_exact_search_within_batch(granne_b200_multi* m, const void* queries, size_t nq,
                                                int query_format, const uint64_t* offsets, const uint64_t* ids,
                                                uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                                uint32_t* out_counts);
/* granne_b200_exact_range_count / granne_b200_exact_range_search over a multi handle (HOST buffers), with u64 GLOBAL
 * ids in QUERY_ID* queries (as granne_b200_multi_search_batch) and in the results.  Argument rules as the single-device
 * calls.  REPLICATED slices the queries over the devices (a search with each slice's offsets rebased into the caller's
 * arrays).  RANGE_PARTITIONED counts every query on every shard and sums the counts; a search counts every shard first
 * (so it scans each shard twice), fills each shard's runs and merges them per query by (distance, global id) into the
 * caller's segment on the host.  QUERY_ID_EXCLUDING on a range-partitioned handle also asks the owning shard for the
 * query's distance to itself (one exact within-list call). */
int granne_b200_multi_exact_range_count(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                        float radius, uint64_t* counts);
int granne_b200_multi_exact_range_search(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                         float radius, const uint64_t* offsets, uint64_t* ids, float* dists);
/* granne_b200_search_filtered_batch over a multi handle: the bitmaps are over GLOBAL ids, results are u64 GLOBAL ids.
 * REPLICATED slices the queries together with their query_filter entries over the devices; RANGE_PARTITIONED runs
 * every query on every shard, shard s reading bit shard_base[s] + local id of the same bitmaps, and merges the shard
 * lists by (distance, global id).  filter_words must cover every part's ids: >= ceil(max_s(shard_base[s] + Index::len
 * of shard s) / 32) (REPLICATED: ceil(Index::len / 32)).  The rules and their order are the single-device call's,
 * with "multi handle is null" first; all are checked on the host before any device call. */
int granne_b200_multi_search_filtered_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                            uint32_t max_search, uint32_t num_neighbors, const uint32_t* filters,
                                            uint32_t num_filters, uint64_t filter_words, const uint32_t* query_filter,
                                            uint64_t* out_ids, float* out_dists, uint32_t* out_counts);
/* granne_b200_exact_search_filtered_batch over a multi handle, with granne_b200_multi_search_filtered_batch's bitmaps
 * over GLOBAL ids, filter_words rule and split: REPLICATED slices the queries with their query_filter entries;
 * RANGE_PARTITIONED runs every query on every shard, shard s reading bit shard_base[s] + local id (shard bases need not
 * be multiples of 32), and merges the shards' exact lists by (distance, global id).  Results are u64 GLOBAL ids. */
int granne_b200_multi_exact_search_filtered_batch(granne_b200_multi* m, const void* queries, size_t nq,
                                                  int query_format, const uint32_t* filters, uint32_t num_filters,
                                                  uint64_t filter_words, const uint32_t* query_filter,
                                                  uint32_t num_neighbors, uint64_t* out_ids, float* out_dists,
                                                  uint32_t* out_counts);
/* granne_b200_set_rerank_elements on every part: REPLICATED takes one image (elements_bytes[0]) and stages it on every
 * device; RANGE_PARTITIONED takes one image per shard.  Every image is checked before any is staged; if a part then fails to
 * stage its rows (a device error), the parts this call attached release theirs again, so the call can be repeated. */
int granne_b200_multi_set_rerank_elements(granne_b200_multi* m, const void* const* elements_bytes,
                                          const size_t* elements_len);
/* granne_b200_set_rerank_embeddings on every part: REPLICATED takes one term-list image (elements_bytes[0]),
 * RANGE_PARTITIONED one per shard; the one embedding table is shared by all parts, as granne_b200_multi_open shares
 * it.  Images are checked and a failed attach is undone as in granne_b200_multi_set_rerank_elements. */
int granne_b200_multi_set_rerank_embeddings(granne_b200_multi* m, const void* const* elements_bytes,
                                            const size_t* elements_len, const void* embeddings_bytes,
                                            size_t embeddings_len);
/* granne_b200_search_rerank_batch over a multi handle, with u64 GLOBAL ids like granne_b200_multi_search_batch.
 * RANGE_PARTITIONED: every shard re-ranks its own candidates and the lists are merged by (distance, global id), which
 * equals re-ranking the union of the shards' candidate sets. */
int granne_b200_multi_search_rerank_batch(granne_b200_multi* m, const float* queries, size_t nq, int query_format,
                                          uint32_t max_search, uint32_t num_candidates, uint32_t num_neighbors,
                                          uint64_t* out_ids, float* out_dists, uint32_t* out_counts);
/* granne_b200_search_diverse_batch over a multi handle, with u64 GLOBAL ids like granne_b200_multi_search_batch (every
 * query format; an id must lie in some part's [shard_base, shard_base + Index::len)).  REPLICATED slices the queries
 * over the devices.  RANGE_PARTITIONED: the candidates are the shards' max_search lists merged by (distance, global id)
 * as granne_b200_multi_search_batch merges them (without the query's own global id for QUERY_ID_EXCLUDING), and
 * select_neighbors runs over the global container: the candidates' element rows are gathered onto part 0's device and
 * selected there (a SumEmbeddings shard's materialised rows as angular f32 rows, whose distances are the same bits).
 * Argument rules as granne_b200_search_diverse_batch; no stats. */
int granne_b200_multi_search_diverse_batch(granne_b200_multi* m, const void* queries, size_t nq, int query_format,
                                           uint32_t max_search, uint32_t num_neighbors, uint64_t* out_ids,
                                           float* out_dists, uint32_t* out_counts);

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
/* GranneBuilder::from_bytes(config, index, elements) (src/index/mod.rs:428-461): a builder that continues from an
 * index file image over the elements it was built from (or more of them).  Every loaded neighbour list keeps its ids
 * in stored (ascending) order and is truncated to the first cfg->num_neighbors ids or padded, exactly as the reference
 * does; the next build indexes only the elements beyond the loaded last layer.  The config is checked as in
 * granne_b200_builder_new, then the image is decoded and checked before any device call: a malformed image or one with
 * more than 24 layers gives GRANNE_B200_ERR_FORMAT even without a device.  An image whose last layer holds more nodes
 * than the container holds elements gives GRANNE_B200_ERR_FORMAT too (checked once the elements are staged).  An
 * image without layers gives the same builder as granne_b200_builder_new.  Element buffers as in granne_b200_open. */
int granne_b200_builder_from_index(const granne_b200_build_config* cfg, const void* index_bytes, size_t index_len,
                                   int element_kind, const void* elements_bytes, size_t elements_len,
                                   const void* embeddings_bytes, size_t embeddings_len, int device,
                                   granne_b200_builder** out);
/* granne_b200_builder_from_index with the element container given as device rows (as in
 * granne_b200_builder_new_device_elements). */
int granne_b200_builder_from_index_device_elements(const granne_b200_build_config* cfg, const void* index_bytes,
                                                   size_t index_len, int element_kind, const void* d_element_rows,
                                                   uint64_t num_elements, uint32_t dim, int device,
                                                   granne_b200_builder** out);
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
 * dim is 1..12000: a row is staged in the kernel's default 48 KB of shared memory (wider rows: ERR_INVALID_ARGUMENT).
 * granne_b200_compute_distances shares the limit.  Call with out == NULL to query the size. */
int granne_b200_elements_from_raw(int element_kind, const float* raw, uint64_t n, uint32_t dim, int device, void* out,
                                  size_t cap, size_t* out_len);

/* ---- device-resident element containers ---------------------------------------------------------------------------
 * The reference borrows its element container from the caller (`Vectors::from_slice`, src/elements/dense_vector.rs:
 * 66-72; `Granne::from_bytes(index, &elements)`, src/index/mod.rs:108-113).  When the rows are already in HBM (made
 * by another kernel, or too large to bounce through the host: 100M x 128 f32 = 51 GB) these variants take them as a
 * device pointer: row-major ELEMENTS (normalised f32 for ANGULAR, i8 for ANGULAR_INT), num_elements x dim, memory of
 * `device`.  The rows are copied into the staged layout during the call; the caller keeps its buffer. */

/* Vector::from per row (angular.rs:55-61 / angular_int.rs:28-45), device to device, asynchronous on `cuda_stream`:
 * d_raw = n x dim raw f32 rows, d_out = n x dim elements (f32 or i8); dim 1..12000 as in granne_b200_elements_from_raw. */
int granne_b200_elements_from_raw_device(int element_kind, const float* d_raw, uint64_t n, uint32_t dim, int device,
                                         void* d_out, void* cuda_stream);

/* compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152) as an elements file image: for every
 * element of a SumEmbeddings container (elements_bytes, embeddings_bytes as in granne_b200_open), its raw sum of
 * embeddings (embeddings/mod.rs:112-143) made into a vector.  kind ANGULAR_INT is the reference function:
 * angular_int::Vector::from(sum), the quantised raw sum (angular_int.rs:19-45).  kind ANGULAR is SumEmbeddings::get
 * per element (embeddings/mod.rs:164-166): the normalised sum, so searching these rows searches the SumEmbeddings
 * container.  The image is FixedWidthSliceVector::write (u64 width | rows); with no element, or a table without rows,
 * it is the 8-byte header of width 0.  Every argument and image check runs on the host before any device call
 * (ERR_FORMAT as in granne_b200_open; ERR_INVALID_ARGUMENT for a bad kind, a null pointer, a table wider than 4096 or
 * too small a `cap`).  A sum holding NaN (ANGULAR_INT; the reference panics) or any non-finite value (ANGULAR)
 * returns ERR_NOT_FINITE.  The device holds the table and a fixed window of elements, whatever their number.
 * out == NULL queries the size (no device needed). */
int granne_b200_compute_embeddings(int element_kind, const void* elements_bytes, size_t elements_len,
                                   const void* embeddings_bytes, size_t embeddings_len, int device, void* out,
                                   size_t cap, size_t* out_len);
/* The same rows, device-resident (n x dim, f32 or i8, memory of `device`) for granne_b200_open_device_elements /
 * granne_b200_builder_new_device_elements.  d_out == NULL writes n and dim only.  Synchronises cuda_stream (NULL = the
 * default stream) before returning, so that ERR_NOT_FINITE can be reported. */
int granne_b200_compute_embeddings_device(int element_kind, const void* elements_bytes, size_t elements_len,
                                          const void* embeddings_bytes, size_t embeddings_len, int device,
                                          void* d_out, uint64_t* out_n, uint32_t* out_dim, void* cuda_stream);

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

/* Bytes of device memory the staged index occupies: layer rows + element container + attached re-rank container, for
 * every way a handle is made (granne_b200_open*, granne_b200_builder_get_index).  Memory a handle shares with a
 * builder or another snapshot is counted by every handle that holds it.  Workspaces are not counted. */
uint64_t granne_b200_device_bytes(const granne_b200_index* h);

#ifdef __cplusplus
}
#endif
#endif /* GRANNE_B200_H */
