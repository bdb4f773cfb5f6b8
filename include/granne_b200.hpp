// granne_b200.hpp — C++17 host-side mirror of granne's Rust API over the C ABI in granne_b200.h (header only).
//
// granne is a Rust crate and this image has no Rust toolchain, so the host side above the C ABI is C++: the classes
// below keep the reference's names, argument meaning and error behaviour so that client code and tests read like the
// reference's (`src/index/tests.rs`):
//
//   granne::Granne::from_bytes / from_file, search, Index::{len, num_layers, layer_len, get_neighbors}, get_element
//                                                      (src/index/mod.rs:38-160)        -> granne_b200::Granne
//   granne::BuildConfig (fluent setters, src/index/mod.rs:198-291)                      -> granne_b200::BuildConfig
//   granne::GranneBuilder::{new, from_bytes, from_file, build, build_partial, push, get_index,
//                           write_index, num_elements} (src/index/mod.rs:295-531)       -> granne_b200::GranneBuilder
//   angular::Vectors / angular_int::Vectors / embeddings::SumEmbeddings file images     -> granne_b200::Elements
//   Granne::reorder / reorder_by_keys (src/index/reorder.rs:59-124)                     -> Granne::reorder*
//
// Where the reference panics (malformed file, NaN distance, max_search == 0, fewer elements than already indexed)
// these classes throw granne_b200::Error carrying the C ABI status and message.  There is no CPU fallback: without an
// sm_90 device every constructor that stages data throws Error{GRANNE_B200_ERR_NO_DEVICE}.
#pragma once

#include <algorithm>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "granne_b200.h"

namespace granne_b200 {

class Error : public std::runtime_error {
public:
    Error(int code, const std::string& what) : std::runtime_error(what), code_(code) {}
    int code() const { return code_; }

private:
    int code_;
};

inline void check(int rc) {
    if (rc != GRANNE_B200_OK) throw Error(rc, granne_b200_last_error());
}

enum class ElementKind : int {
    Angular = GRANNE_B200_ANGULAR,        // angular::Vectors      (f32, normalised)
    AngularInt = GRANNE_B200_ANGULAR_INT, // angular_int::Vectors  (i8, quantised)
    Embeddings = GRANNE_B200_EMBEDDINGS,  // embeddings::SumEmbeddings
};

inline std::vector<uint8_t> read_file(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw Error(GRANNE_B200_ERR_IO, "could not open " + path);
    return std::vector<uint8_t>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

namespace detail {

// The bytes of a C ABI call that reports the size of what it writes and writes only into a buffer it is given:
// `call(out, cap, &len)` once without a buffer for the size, once with one of that size.
template <class Call>
std::vector<uint8_t> sized_bytes(Call&& call) {
    size_t need = 0;
    check(call(nullptr, 0, &need));
    std::vector<uint8_t> out(need);
    check(call(out.data(), out.size(), &need));
    out.resize(need);
    return out;
}

// One result list per query from the C ABI's (ids, dists, counts) with k slots per query: its first counts[q] pairs.
// Range results in CSR form (offsets [nq + 1], ids, dists) as one list per query.
template <class Result, class Id>
std::vector<Result> csr_lists(const std::vector<uint64_t>& offsets, const std::vector<Id>& ids,
                              const std::vector<float>& dists) {
    std::vector<Result> out(offsets.empty() ? 0 : offsets.size() - 1);
    for (size_t q = 0; q < out.size(); ++q)
        for (uint64_t j = offsets[q]; j < offsets[q + 1]; ++j) out[q].emplace_back(ids[j], dists[j]);
    return out;
}

// Count, prefix sum, fill: the two phases of a range search into CSR arrays.
template <class Id, class Count, class Fill>
void range_csr(size_t nq, Count&& count, Fill&& fill, std::vector<uint64_t>* offsets, std::vector<Id>* ids,
               std::vector<float>* dists) {
    std::vector<uint64_t> counts(nq);
    count(counts.data());
    offsets->assign(nq + 1, 0);
    for (size_t q = 0; q < nq; ++q) (*offsets)[q + 1] = (*offsets)[q] + counts[q];
    ids->resize(offsets->back());
    dists->resize(offsets->back());
    fill(offsets->data(), ids->data(), dists->data());
}

template <class Result, class Id>
std::vector<Result> result_lists(const std::vector<Id>& ids, const std::vector<float>& dists,
                                 const std::vector<uint32_t>& counts, size_t k) {
    std::vector<Result> out(counts.size());
    for (size_t q = 0; q < counts.size(); ++q)
        for (uint32_t j = 0; j < counts[q]; ++j) out[q].emplace_back(ids[q * k + j], dists[q * k + j]);
    return out;
}

}  // namespace detail

// An element container as the file image granne writes (`ElementContainer` + `io::Writeable`): u64 width + rows for
// the vector types; offsets + 3-byte ids (and the embeddings table) for SumEmbeddings.
struct Elements {
    ElementKind kind = ElementKind::Angular;
    std::vector<uint8_t> bytes;
    std::vector<uint8_t> embeddings;  // SumEmbeddings only

    // `rows.map(Vector::from).collect()`: normalise (angular.rs:55-61) or quantise (angular_int.rs:19-45) n raw rows
    static Elements from_raw(ElementKind kind, const float* rows, uint64_t n, uint32_t dim, int device = 0) {
        Elements e;
        e.kind = kind;
        e.bytes = detail::sized_bytes([&](void* out, size_t cap, size_t* len) {
            return granne_b200_elements_from_raw(static_cast<int>(kind), rows, n, dim, device, out, cap, len);
        });
        return e;
    }
    // compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152): the sum of embeddings of every
    // element of a SumEmbeddings container as an AngularInt (quantised raw sum, what the reference writes) or Angular
    // (normalised sum: SumEmbeddings::get) container
    static Elements compute_embeddings(ElementKind kind, const Elements& sum, int device = 0) {
        Elements e;
        e.kind = kind;
        e.bytes = detail::sized_bytes([&](void* out, size_t cap, size_t* len) {
            return granne_b200_compute_embeddings(static_cast<int>(kind), sum.bytes.data(), sum.bytes.size(),
                                                  sum.embeddings.data(), sum.embeddings.size(), device, out, cap, len);
        });
        return e;
    }
    // Vectors::from_file / SumEmbeddings::from_files
    static Elements from_files(ElementKind kind, const std::string& elements_path,
                               const std::string& embeddings_path = std::string()) {
        Elements e;
        e.kind = kind;
        e.bytes = read_file(elements_path);
        if (kind == ElementKind::Embeddings) e.embeddings = read_file(embeddings_path);
        return e;
    }
    uint64_t dim() const {  // meaningful for the vector types
        uint64_t w = 0;
        for (int b = 0; b < 8 && b < static_cast<int>(bytes.size()); ++b) w |= static_cast<uint64_t>(bytes[b]) << (8 * b);
        return w;
    }
    uint64_t len() const {  // ElementContainer::len
        if (bytes.size() < 8) return 0;
        if (kind == ElementKind::Embeddings) return dim();  // the leading u64 is the element count
        const uint64_t row = dim() * (kind == ElementKind::Angular ? 4 : 1);
        return row ? (bytes.size() - 8) / row : 0;
    }
};

using SearchResult = std::vector<std::pair<size_t, float>>;  // Vec<(usize, f32)>

// granne::Granne (src/index/mod.rs:38-160).  Move-only; owns the staged index.
class Granne {
public:
    Granne() = default;
    Granne(const Granne&) = delete;
    Granne& operator=(const Granne&) = delete;
    Granne(Granne&& o) noexcept { swap(o); }
    Granne& operator=(Granne&& o) noexcept {
        if (this != &o) {
            close();
            swap(o);
        }
        return *this;
    }
    ~Granne() { close(); }

    // Granne::from_bytes(index, elements) (:108-113)
    static Granne from_bytes(const void* index, size_t index_len, const Elements& elements, int device = 0) {
        Granne g;
        check(granne_b200_open(index, index_len, static_cast<int>(elements.kind), elements.bytes.data(),
                               elements.bytes.size(), elements.embeddings.empty() ? nullptr : elements.embeddings.data(),
                               elements.embeddings.size(), device, &g.h_));
        g.elements_ = elements;
        g.device_ = device;
        return g;
    }
    static Granne from_bytes(const std::vector<uint8_t>& index, const Elements& elements, int device = 0) {
        return from_bytes(index.data(), index.size(), elements, device);
    }
    // Granne::from_file(&file, elements) (:122-135)
    static Granne from_file(const std::string& index_path, const Elements& elements, int device = 0) {
        return from_bytes(read_file(index_path), elements, device);
    }

    // Index trait (:54-104)
    size_t len() const { return static_cast<size_t>(granne_b200_len(h_)); }
    size_t num_layers() const { return static_cast<size_t>(granne_b200_num_layers(h_)); }
    size_t layer_len(size_t layer) const { return static_cast<size_t>(granne_b200_layer_len(h_, layer)); }
    std::vector<size_t> get_neighbors(size_t idx, size_t layer) const {
        uint32_t buf[256];
        size_t n = 0;
        check(granne_b200_get_neighbors(h_, idx, layer, buf, 256, &n));
        return std::vector<size_t>(buf, buf + n);
    }
    std::vector<uint8_t> write_index() const {  // Index::write_index (io.rs:11-70)
        return detail::sized_bytes(
            [&](void* out, size_t cap, size_t* len) { return granne_b200_write_index(h_, out, cap, len); });
    }

    // ElementContainer
    size_t dim() const { return static_cast<size_t>(granne_b200_dim(h_)); }
    ElementKind kind() const { return static_cast<ElementKind>(granne_b200_element_kind(h_)); }
    const Elements& get_elements() const { return elements_; }
    std::vector<float> get_element(size_t idx) const {  // Granne::get_element (:153-155), f32 element types
        if (kind() == ElementKind::AngularInt) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "use get_element_i8");
        std::vector<float> out(dim());
        check(granne_b200_get_element(h_, idx, out.data()));
        return out;
    }
    std::vector<int8_t> get_element_i8(size_t idx) const {
        if (kind() != ElementKind::AngularInt) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "use get_element");
        std::vector<int8_t> out(dim());
        check(granne_b200_get_element(h_, idx, out.data()));
        return out;
    }
    // get_element for every id in one launch (granne_b200_get_elements): ids.size() x dim() values, row-major
    std::vector<float> get_elements(const std::vector<uint32_t>& ids) const {
        if (kind() == ElementKind::AngularInt) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "use get_elements_i8");
        std::vector<float> out(ids.size() * dim());
        check(granne_b200_get_elements(h_, ids.data(), ids.size(), out.data()));
        return out;
    }
    std::vector<int8_t> get_elements_i8(const std::vector<uint32_t>& ids) const {
        if (kind() != ElementKind::AngularInt) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "use get_elements");
        std::vector<int8_t> out(ids.size() * dim());
        check(granne_b200_get_elements(h_, ids.data(), ids.size(), out.data()));
        return out;
    }

    // Granne::search(&get_element(id), max_search, num_neighbors) for every id in one call (GRANNE_B200_QUERY_ID);
    // with exclude_self each id's own entry is dropped from its k + 1 results (GRANNE_B200_QUERY_ID_EXCLUDING).
    // exact_search_by_id is the same for exact_search_batch.  exact_search_within and search_filtered take ids the same
    // way: pass ids.data(), ids.size() and GRANNE_B200_QUERY_ID or GRANNE_B200_QUERY_ID_EXCLUDING as their queries.
    std::vector<SearchResult> search_by_id(const std::vector<uint32_t>& ids, size_t max_search, size_t num_neighbors,
                                           bool exclude_self = false) const {
        return search_batch(ids.data(), ids.size(), exclude_self ? GRANNE_B200_QUERY_ID_EXCLUDING : GRANNE_B200_QUERY_ID,
                            max_search, num_neighbors);
    }
    std::vector<SearchResult> exact_search_by_id(const std::vector<uint32_t>& ids, size_t num_neighbors,
                                                 bool exclude_self = false) const {
        return exact_search_batch(ids.data(), ids.size(),
                                  exclude_self ? GRANNE_B200_QUERY_ID_EXCLUDING : GRANNE_B200_QUERY_ID, num_neighbors);
    }
    // The k-nearest-neighbour graph: search_by_id (or exact_search_batch by id, `exact`) of every element of [0, len())
    // in chunks of `chunk` ids; entry i is element i's list.
    std::vector<SearchResult> knn_graph(size_t max_search, size_t num_neighbors, bool exclude_self = true,
                                        bool exact = false, size_t chunk = 65536) const {
        if (chunk == 0) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "chunk must be >= 1");
        std::vector<SearchResult> graph;
        const int fmt = exclude_self ? GRANNE_B200_QUERY_ID_EXCLUDING : GRANNE_B200_QUERY_ID;
        for (size_t c0 = 0; c0 < len(); c0 += chunk) {
            std::vector<uint32_t> ids(std::min(chunk, len() - c0));
            for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<uint32_t>(c0 + i);
            std::vector<SearchResult> part = exact ? exact_search_batch(ids.data(), ids.size(), fmt, num_neighbors)
                                                   : search_batch(ids.data(), ids.size(), fmt, max_search, num_neighbors);
            for (auto& r : part) graph.push_back(std::move(r));
        }
        return graph;
    }

    // Granne::search(&element, max_search, num_neighbors) (:140-150); `element` is an Elements::Element
    // (normalised f32 for angular / embeddings, i8 for angular_int) exactly as in the reference.
    SearchResult search(const std::vector<float>& element, size_t max_search, size_t num_neighbors) const {
        return search_batch(element.data(), 1, GRANNE_B200_QUERY_ELEMENT, max_search, num_neighbors).at(0);
    }
    SearchResult search(const std::vector<int8_t>& element, size_t max_search, size_t num_neighbors) const {
        return search_batch(element.data(), 1, GRANNE_B200_QUERY_ELEMENT, max_search, num_neighbors).at(0);
    }
    // search(&Vector::from(raw), ...): the raw vector is normalised / quantised by the library like Vector::from
    SearchResult search_raw(const std::vector<float>& raw, size_t max_search, size_t num_neighbors) const {
        return search_batch(raw.data(), 1, GRANNE_B200_QUERY_RAW_F32, max_search, num_neighbors).at(0);
    }
    // nq independent searches in one launch; `queries` holds nq rows of dim() values in `query_format`
    std::vector<SearchResult> search_batch(const void* queries, size_t nq, int query_format, size_t max_search,
                                           size_t num_neighbors) const {
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_search_batch(h_, queries, nq, query_format, static_cast<uint32_t>(max_search),
                                       static_cast<uint32_t>(num_neighbors), ids.data(), dists.data(), counts.data(),
                                       nullptr));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }
    // Exact k nearest neighbours (granne_b200_exact_search_batch): the first min(k, len()) elements by (distance, id),
    // the reference's distance bit for bit.  Not a reference function: the ground truth of recall.
    std::vector<SearchResult> exact_search_batch(const void* queries, size_t nq, int query_format,
                                                 size_t num_neighbors) const {
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_exact_search_batch(h_, queries, nq, query_format, static_cast<uint32_t>(num_neighbors),
                                             ids.data(), dists.data(), counts.data()));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }
    // Exact range search (granne_b200_exact_range_count, then granne_b200_exact_range_search): every element of
    // [0, len()) whose distance to the query is <= radius, sorted by (distance, id), the reference's distance bit for
    // bit.  Not a reference function.  Queries in any format, ids included.
    std::vector<SearchResult> exact_range_search(const void* queries, size_t nq, int query_format, float radius) const {
        std::vector<uint64_t> offsets;
        std::vector<uint32_t> ids;
        std::vector<float> dists;
        detail::range_csr(
            nq, [&](uint64_t* c) { check(granne_b200_exact_range_count(h_, queries, nq, query_format, radius, c)); },
            [&](const uint64_t* o, uint32_t* i, float* d) {
                check(granne_b200_exact_range_search(h_, queries, nq, query_format, radius, o, i, d));
            },
            &offsets, &ids, &dists);
        return detail::csr_lists<SearchResult>(offsets, ids, dists);
    }
    // Exact k nearest neighbours of each query within its own candidate list (granne_b200_exact_search_within_batch):
    // lists[q] holds query q's ids (< len(); duplicates count once); the first min(k, |set(lists[q])|) by (distance,
    // id), the reference's distance bit for bit.  Not a reference function.
    std::vector<SearchResult> exact_search_within(const void* queries, size_t nq, int query_format,
                                                  const std::vector<std::vector<uint32_t>>& lists,
                                                  size_t num_neighbors) const {
        if (lists.size() != nq) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "one candidate list per query");
        std::vector<uint64_t> offsets(1, 0);
        std::vector<uint32_t> cand;
        for (const auto& l : lists) {
            cand.insert(cand.end(), l.begin(), l.end());
            offsets.push_back(cand.size());
        }
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_exact_search_within_batch(h_, queries, nq, query_format, offsets.data(), cand.data(),
                                                    static_cast<uint32_t>(num_neighbors), ids.data(), dists.data(),
                                                    counts.data()));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }
    // Filtered search (granne_b200_search_filtered_batch): search_batch's traversal, unchanged, keeping the first k
    // elements by (distance, id) among those it scores in the bottom layer that the query's filter admits.  `filters`
    // holds num_filters bitmaps of filter_words u32 words (id i: bit i % 32 of word i / 32, filter_words >=
    // ceil(len() / 32)); query_filter (may be null) picks each query's bitmap.  k <= GRANNE_B200_EXACT_MAX_K.  Not a
    // reference function.
    std::vector<SearchResult> search_filtered(const void* queries, size_t nq, int query_format, size_t max_search,
                                              size_t num_neighbors, const uint32_t* filters, uint32_t num_filters,
                                              uint64_t filter_words, const uint32_t* query_filter = nullptr) const {
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_search_filtered_batch(h_, queries, nq, query_format, static_cast<uint32_t>(max_search),
                                                static_cast<uint32_t>(num_neighbors), filters, num_filters,
                                                filter_words, query_filter, ids.data(), dists.data(), counts.data(),
                                                nullptr));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }
    // Exact filtered k-NN (granne_b200_exact_search_filtered_batch): the first min(k, |A|) of the ids < len() the
    // query's filter admits, by (distance, id), with exact_search's distances.  Filters as in search_filtered; there is
    // no max_search.  k <= GRANNE_B200_EXACT_MAX_K.  Not a reference function.
    std::vector<SearchResult> exact_search_filtered(const void* queries, size_t nq, int query_format,
                                                    size_t num_neighbors, const uint32_t* filters,
                                                    uint32_t num_filters, uint64_t filter_words,
                                                    const uint32_t* query_filter = nullptr) const {
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_exact_search_filtered_batch(h_, queries, nq, query_format, filters, num_filters,
                                                      filter_words, query_filter,
                                                      static_cast<uint32_t>(num_neighbors), ids.data(), dists.data(),
                                                      counts.data()));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }

    // Two-stage search (granne_b200_search_rerank_batch): attach the container of this angular_int index's elements
    // once (angular f32 rows, or the SumEmbeddings container the rows were computed from), then search_rerank
    // returns, for nq raw f32 queries, the first num_candidates results of the i8 search re-ranked by their exact f32
    // angular distance over that container.  Not a reference function.
    void set_rerank_elements(const Elements& container) {
        if (container.kind == ElementKind::Angular) {
            check(granne_b200_set_rerank_elements(h_, container.bytes.data(), container.bytes.size()));
        } else if (container.kind == ElementKind::Embeddings) {
            check(granne_b200_set_rerank_embeddings(h_, container.bytes.data(), container.bytes.size(),
                                                    container.embeddings.data(), container.embeddings.size()));
        } else {
            throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "re-rank containers are angular or SumEmbeddings elements");
        }
    }
    std::vector<SearchResult> search_rerank(const float* queries, size_t nq, size_t max_search, size_t num_candidates,
                                            size_t num_neighbors) const {
        std::vector<uint32_t> ids(nq * num_neighbors), counts(nq);
        std::vector<float> dists(nq * num_neighbors);
        check(granne_b200_search_rerank_batch(h_, queries, nq, GRANNE_B200_QUERY_RAW_F32,
                                              static_cast<uint32_t>(max_search), static_cast<uint32_t>(num_candidates),
                                              static_cast<uint32_t>(num_neighbors), ids.data(), dists.data(),
                                              counts.data(), nullptr));
        return detail::result_lists<SearchResult>(ids, dists, counts, num_neighbors);
    }

    // Granne::reorder (reorder.rs:59-82) / reorder_by_keys (:89-124): reorders index and elements, returns the order
    // (`order[i] == j`: element j moved to i).
    std::vector<size_t> reorder(bool /*show_progress*/ = false) {
        std::vector<uint64_t> order(len());
        check(granne_b200_compute_order(h_, order.data(), order.size()));
        return apply(order);
    }
    std::vector<size_t> reorder_by_keys(const std::vector<uint64_t>& keys, uint32_t key_width = 1,
                                        bool /*show_progress*/ = false) {
        const std::vector<uint8_t> image = write_index();
        std::vector<uint64_t> order(len());
        check(granne_b200_order_by_keys(image.data(), image.size(), keys.data(), keys.size() / key_width, key_width,
                                        order.data()));
        return apply(order);
    }

    granne_b200_index* handle() const { return h_; }

private:
    friend class GranneBuilder;
    std::vector<size_t> apply(const std::vector<uint64_t>& order) {
        const std::vector<uint8_t> image = write_index();
        size_t ni = 0, ne = 0;
        check(granne_b200_apply_order(image.data(), image.size(), static_cast<int>(elements_.kind), elements_.bytes.data(),
                                      elements_.bytes.size(), order.data(), order.size(), nullptr, 0, &ni, nullptr, 0,
                                      &ne));
        std::vector<uint8_t> new_index(ni);
        Elements new_elements = elements_;
        new_elements.bytes.resize(ne);
        check(granne_b200_apply_order(image.data(), image.size(), static_cast<int>(elements_.kind), elements_.bytes.data(),
                                      elements_.bytes.size(), order.data(), order.size(), new_index.data(), ni, &ni,
                                      new_elements.bytes.data(), ne, &ne));
        Granne fresh = from_bytes(new_index, new_elements, device_);
        *this = std::move(fresh);
        return std::vector<size_t>(order.begin(), order.end());
    }
    void close() {
        if (h_) granne_b200_close(h_);
        h_ = nullptr;
    }
    void swap(Granne& o) {
        std::swap(h_, o.h_);
        std::swap(elements_, o.elements_);
        std::swap(device_, o.device_);
    }
    granne_b200_index* h_ = nullptr;
    Elements elements_;
    int device_ = 0;
};

// Several GPUs of this process behind one handle (granne_b200_multi_*): `Granne::from_bytes` + `search` with the index
// replicated on every device (query batches are sliced) or range-partitioned into independent shards (every shard is
// searched, results merged by (distance, global id) — the order of into_sorted_vec, src/index/mod.rs:1036).
class MultiGranne {
public:
    using Result = std::vector<std::pair<uint64_t, float>>;  // (global id, distance)
    MultiGranne() = default;
    MultiGranne(const MultiGranne&) = delete;
    MultiGranne& operator=(const MultiGranne&) = delete;
    MultiGranne(MultiGranne&& o) noexcept { std::swap(h_, o.h_); std::swap(dim_, o.dim_); std::swap(kind_, o.kind_); }
    ~MultiGranne() { if (h_) granne_b200_multi_close(h_); }

    static MultiGranne replicated(const std::vector<uint8_t>& index, const Elements& elements,
                                  const std::vector<int>& devices) {
        const void* ip[1] = {index.data()};
        const size_t il[1] = {index.size()};
        const void* ep[1] = {elements.bytes.data()};
        const size_t el[1] = {elements.bytes.size()};
        MultiGranne m;
        check(granne_b200_multi_open(GRANNE_B200_MODE_REPLICATED, devices.data(), devices.size(),
                                     static_cast<int>(elements.kind), ip, il, ep, el, 1,
                                     elements.embeddings.empty() ? nullptr : elements.embeddings.data(),
                                     elements.embeddings.size(), &m.h_));
        m.dim_ = elements.dim();
        m.kind_ = elements.kind;
        return m;
    }
    // one (index, elements) pair per shard; shard s lives on devices[s % devices.size()]
    static MultiGranne partitioned(const std::vector<std::vector<uint8_t>>& indexes, const std::vector<Elements>& shards,
                                   const std::vector<int>& devices) {
        if (indexes.size() != shards.size() || shards.empty())
            throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "one index per shard");
        std::vector<const void*> ip, ep;
        std::vector<size_t> il, el;
        for (size_t s = 0; s < shards.size(); ++s) {
            ip.push_back(indexes[s].data());
            il.push_back(indexes[s].size());
            ep.push_back(shards[s].bytes.data());
            el.push_back(shards[s].bytes.size());
        }
        MultiGranne m;
        check(granne_b200_multi_open(GRANNE_B200_MODE_RANGE_PARTITIONED, devices.data(), devices.size(),
                                     static_cast<int>(shards[0].kind), ip.data(), il.data(), ep.data(), el.data(),
                                     shards.size(), shards[0].embeddings.empty() ? nullptr : shards[0].embeddings.data(),
                                     shards[0].embeddings.size(), &m.h_));
        m.dim_ = shards[0].dim();
        m.kind_ = shards[0].kind;
        return m;
    }
    uint64_t len() const { return granne_b200_multi_len(h_); }
    size_t num_parts() const { return granne_b200_multi_num_parts(h_); }
    uint64_t shard_base(size_t s) const { return granne_b200_multi_shard_base(h_, s); }

    // search(&Vector::from(raw), max_search, num_neighbors) for nq raw f32 queries (nq x dim, row-major)
    std::vector<Result> search_batch_raw(const std::vector<float>& queries, size_t max_search,
                                         size_t num_neighbors) const {
        const size_t nq = dim_ ? queries.size() / dim_ : 0;
        std::vector<uint64_t> ids(nq * num_neighbors);
        std::vector<float> d(nq * num_neighbors);
        std::vector<uint32_t> c(nq);
        check(granne_b200_multi_search_batch(h_, queries.data(), nq, GRANNE_B200_QUERY_RAW_F32,
                                             static_cast<uint32_t>(max_search), static_cast<uint32_t>(num_neighbors),
                                             ids.data(), d.data(), c.data()));
        return detail::result_lists<Result>(ids, d, c, num_neighbors);
    }
    // exact k nearest neighbours over every shard for nq raw f32 queries (granne_b200_multi_exact_search_batch)
    std::vector<Result> exact_search_batch_raw(const std::vector<float>& queries, size_t num_neighbors) const {
        const size_t nq = dim_ ? queries.size() / dim_ : 0;
        std::vector<uint64_t> ids(nq * num_neighbors);
        std::vector<float> d(nq * num_neighbors);
        std::vector<uint32_t> c(nq);
        check(granne_b200_multi_exact_search_batch(h_, queries.data(), nq, GRANNE_B200_QUERY_RAW_F32,
                                                   static_cast<uint32_t>(num_neighbors), ids.data(), d.data(),
                                                   c.data()));
        return detail::result_lists<Result>(ids, d, c, num_neighbors);
    }
    // Granne::exact_range_search over every part (granne_b200_multi_exact_range_count, then _search): GLOBAL ids in
    // the results, and as queries of the QUERY_ID* formats (u64)
    std::vector<Result> exact_range_search(const void* queries, size_t nq, int query_format, float radius) const {
        std::vector<uint64_t> offsets, ids;
        std::vector<float> dists;
        detail::range_csr(
            nq,
            [&](uint64_t* c) { check(granne_b200_multi_exact_range_count(h_, queries, nq, query_format, radius, c)); },
            [&](const uint64_t* o, uint64_t* i, float* d) {
                check(granne_b200_multi_exact_range_search(h_, queries, nq, query_format, radius, o, i, d));
            },
            &offsets, &ids, &dists);
        return detail::csr_lists<Result>(offsets, ids, dists);
    }
    // Granne::exact_search_within over every part for nq raw f32 queries (nq x dim, row-major, as the *_raw calls
    // take them), GLOBAL ids in the lists and the results (granne_b200_multi_exact_search_within_batch)
    std::vector<Result> exact_search_within(const std::vector<float>& queries,
                                                const std::vector<std::vector<uint64_t>>& lists,
                                                size_t num_neighbors) const {
        const size_t nq = dim_ ? queries.size() / dim_ : 0;
        if (lists.size() != nq) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "one candidate list per query");
        std::vector<uint64_t> offsets(1, 0), cand;
        for (const auto& l : lists) {
            cand.insert(cand.end(), l.begin(), l.end());
            offsets.push_back(cand.size());
        }
        std::vector<uint64_t> ids(nq * num_neighbors);
        std::vector<float> d(nq * num_neighbors);
        std::vector<uint32_t> c(nq);
        check(granne_b200_multi_exact_search_within_batch(h_, queries.data(), nq, GRANNE_B200_QUERY_RAW_F32,
                                                          offsets.data(), cand.data(),
                                                          static_cast<uint32_t>(num_neighbors), ids.data(), d.data(),
                                                          c.data()));
        return detail::result_lists<Result>(ids, d, c, num_neighbors);
    }
    // Granne::search_filtered over every part for nq raw f32 queries: the bitmaps are over GLOBAL ids, and so are the
    // results (granne_b200_multi_search_filtered_batch)
    std::vector<Result> search_filtered(const std::vector<float>& queries, size_t max_search, size_t num_neighbors,
                                        const uint32_t* filters, uint32_t num_filters, uint64_t filter_words,
                                        const uint32_t* query_filter = nullptr) const {
        const size_t nq = dim_ ? queries.size() / dim_ : 0;
        std::vector<uint64_t> ids(nq * num_neighbors);
        std::vector<float> d(nq * num_neighbors);
        std::vector<uint32_t> c(nq);
        check(granne_b200_multi_search_filtered_batch(h_, queries.data(), nq, GRANNE_B200_QUERY_RAW_F32,
                                                      static_cast<uint32_t>(max_search),
                                                      static_cast<uint32_t>(num_neighbors), filters, num_filters,
                                                      filter_words, query_filter, ids.data(), d.data(), c.data()));
        return detail::result_lists<Result>(ids, d, c, num_neighbors);
    }
    // Granne::exact_search_filtered over every part for nq raw f32 queries: bitmaps over GLOBAL ids, GLOBAL ids in the
    // results (granne_b200_multi_exact_search_filtered_batch)
    std::vector<Result> exact_search_filtered(const std::vector<float>& queries, size_t num_neighbors,
                                              const uint32_t* filters, uint32_t num_filters, uint64_t filter_words,
                                              const uint32_t* query_filter = nullptr) const {
        const size_t nq = dim_ ? queries.size() / dim_ : 0;
        std::vector<uint64_t> ids(nq * num_neighbors);
        std::vector<float> d(nq * num_neighbors);
        std::vector<uint32_t> c(nq);
        check(granne_b200_multi_exact_search_filtered_batch(h_, queries.data(), nq, GRANNE_B200_QUERY_RAW_F32, filters,
                                                            num_filters, filter_words, query_filter,
                                                            static_cast<uint32_t>(num_neighbors), ids.data(),
                                                            d.data(), c.data()));
        return detail::result_lists<Result>(ids, d, c, num_neighbors);
    }

private:
    granne_b200_multi* h_ = nullptr;
    uint64_t dim_ = 0;
    ElementKind kind_ = ElementKind::Angular;
};

// granne::BuildConfig (src/index/mod.rs:198-291): `BuildConfig::default().num_neighbors(20).max_search(5)`
class BuildConfig {
public:
    BuildConfig() { granne_b200_build_config_default(&c_); }  // layer_multiplier 15, num_neighbors 30, max_search 200
    BuildConfig layer_multiplier(float v) const { BuildConfig r = *this; r.c_.layer_multiplier = v; return r; }
    BuildConfig expected_num_elements(size_t v) const { BuildConfig r = *this; r.c_.expected_num_elements = static_cast<int64_t>(v); return r; }
    BuildConfig num_neighbors(size_t v) const { BuildConfig r = *this; r.c_.num_neighbors = static_cast<uint32_t>(v); return r; }
    BuildConfig max_search(size_t v) const { BuildConfig r = *this; r.c_.max_search = static_cast<uint32_t>(v); return r; }
    BuildConfig reinsert_elements(bool v) const { BuildConfig r = *this; r.c_.reinsert_elements = v ? 1 : 0; return r; }
    BuildConfig show_progress(bool v) const { BuildConfig r = *this; r.c_.show_progress = v ? 1 : 0; return r; }
    const granne_b200_build_config& raw() const { return c_; }

private:
    granne_b200_build_config c_{};
};

// granne::GranneBuilder (src/index/mod.rs:295-531).  Move-only.
class GranneBuilder {
public:
    // GranneBuilder::new(config, elements) (:303-315)
    GranneBuilder(const BuildConfig& config, const Elements& elements, int device = 0) : elements_(elements), device_(device) {
        check(granne_b200_builder_new(&config.raw(), static_cast<int>(elements.kind), elements.bytes.data(),
                                      elements.bytes.size(), elements.embeddings.empty() ? nullptr : elements.embeddings.data(),
                                      elements.embeddings.size(), device, &b_));
    }
    // GranneBuilder::from_bytes(config, index, elements) (:428-461): continues from an index built over `elements`
    // (or over a prefix of them); every neighbour list is truncated or padded to config's num_neighbors
    static GranneBuilder from_bytes(const BuildConfig& config, const void* index, size_t index_len,
                                    const Elements& elements, int device = 0) {
        GranneBuilder g;
        check(granne_b200_builder_from_index(&config.raw(), index, index_len, static_cast<int>(elements.kind),
                                             elements.bytes.data(), elements.bytes.size(),
                                             elements.embeddings.empty() ? nullptr : elements.embeddings.data(),
                                             elements.embeddings.size(), device, &g.b_));
        g.elements_ = elements;
        g.device_ = device;
        return g;
    }
    static GranneBuilder from_bytes(const BuildConfig& config, const std::vector<uint8_t>& index,
                                    const Elements& elements, int device = 0) {
        return from_bytes(config, index.data(), index.size(), elements, device);
    }
    // GranneBuilder::from_file(config, &file, elements) (:463-469)
    static GranneBuilder from_file(const BuildConfig& config, const std::string& index_path, const Elements& elements,
                                   int device = 0) {
        return from_bytes(config, read_file(index_path), elements, device);
    }
    GranneBuilder(const GranneBuilder&) = delete;
    GranneBuilder& operator=(const GranneBuilder&) = delete;
    GranneBuilder(GranneBuilder&& o) noexcept : b_(o.b_), elements_(std::move(o.elements_)), device_(o.device_) { o.b_ = nullptr; }
    ~GranneBuilder() {
        if (b_) granne_b200_builder_free(b_);
    }

    void build() { check(granne_b200_builder_build(b_, 0)); }                              // Builder::build (:366-368)
    void build_partial(size_t num_elements) {                                             // :374-402
        if (num_elements == 0) return;  // indexes nothing (the C ABI reserves 0 for "all")
        check(granne_b200_builder_build(b_, num_elements));
    }
    // GranneBuilder::push for every row of `more` (:512-531): same element type and width
    void push(const Elements& more) {
        check(granne_b200_builder_append(b_, more.bytes.data(), more.bytes.size()));
        elements_.bytes.insert(elements_.bytes.end(), more.bytes.begin() + 8, more.bytes.end());
    }
    size_t len() const { return static_cast<size_t>(granne_b200_builder_len(b_)); }        // Index::len (:329-331)
    size_t num_elements() const { return static_cast<size_t>(granne_b200_builder_num_elements(b_)); }  // :404-406
    size_t num_layers() const { return static_cast<size_t>(granne_b200_builder_num_layers(b_)); }
    size_t layer_len(size_t layer) const { return static_cast<size_t>(granne_b200_builder_layer_len(b_, layer)); }
    std::vector<size_t> get_neighbors(size_t idx, size_t layer) const {
        uint32_t buf[256];
        size_t n = 0;
        check(granne_b200_builder_get_neighbors(b_, idx, layer, buf, 256, &n));
        return std::vector<size_t>(buf, buf + n);
    }
    std::vector<uint8_t> write_index() const {  // Index::write_index (:358-361)
        return detail::sized_bytes(
            [&](void* out, size_t cap, size_t* len) { return granne_b200_builder_write_index(b_, out, cap, len); });
    }
    const Elements& get_elements() const { return elements_; }
    Granne get_index() const {  // GranneBuilder::get_index (:483-488): a searchable snapshot
        Granne g;
        check(granne_b200_builder_get_index(b_, &g.h_));
        g.elements_ = elements_;
        g.device_ = device_;
        return g;
    }

private:
    GranneBuilder() = default;
    granne_b200_builder* b_ = nullptr;
    Elements elements_;
    int device_ = 0;
};

// compute_distance (py/src/lib.rs:71-89): Vector::from(a).dist(&Vector::from(b))
inline float compute_distance(ElementKind kind, const std::vector<float>& a, const std::vector<float>& b, int device = 0) {
    if (a.size() != b.size()) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "vectors differ in length");
    float out = 0.0f;
    check(granne_b200_compute_distances(static_cast<int>(kind), a.data(), b.data(), 1, static_cast<uint32_t>(a.size()),
                                        device, &out));
    return out;
}

}  // namespace granne_b200
