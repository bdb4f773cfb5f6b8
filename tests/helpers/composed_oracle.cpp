// composed_oracle.cpp — checkers composed from the CPU oracle's own pieces, one entry point per GPU call family.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// It compiles the CPU oracle (oracle/granne_oracle.cpp) unchanged and adds three entry points beside it.  Loaded
// through tests/helpers/composed_oracle.py.
//
// orc_exact_search — brute-force k nearest neighbours, the checker of granne_b200_exact_search_batch: for every query,
// the oracle's own Elements::dist_to_element (src/index/mod.rs:1012) for every element i < index_len, then a stable
// partial sort by (distance, id) — the order of into_sorted_vec (:1036).
//
// orc_filtered_search — filtered search, the checker of granne_b200_search_filtered_batch.  Per query:
//   1. the oracle's upper-layer descent (search_for_neighbors with max_search = 1 per layer, as index_search does);
//   2. the oracle's search_for_neighbors on the bottom layer B with the caller's max_search, through a GetNeighbors
//      that records every neighbour it returns.  It is called exactly once per expansion, and every neighbour it
//      returns is scored unless already visited, so the recorded ids plus the entrypoint are S(q), the elements whose
//      distance the search computes in B;
//   3. the filter applied to S(q), and Elements::dist_to_element for each admitted id;
//   4. a sort by (distance, id) — the order of into_sorted_vec (src/index/mod.rs:1036) — and the first k.
//
// orc_compute_embeddings — CPU restatement of compute_embeddings_and_save_to_disk
// (src/elements/embeddings/parsing.rs:102-152), the checker of granne_b200_compute_embeddings.  The sum
// (Elements::raw_embedding), quantize_i8 and normalize_f32 it uses are the oracle's own.
#include "../../oracle/granne_oracle.cpp"

extern "C" {

// `p`: an oracle element container.  queries: nq rows of raw f32 (already_element = 0: made into elements like the
// reference's Python binding), or elements (already_element = 1: normalised f32, or i8 rows in queries_i8 for
// angular_int).  Writes nq x k ids (UNUSED padded), distances (+inf padded) and counts = min(k, index_len).  Returns 0,
// or -1 when a distance is NaN (the reference panics).
int orc_exact_search(void* p, uint64_t index_len, const float* queries, const int8_t* queries_i8, uint64_t nq,
                     int already_element, uint64_t k, int threads, uint32_t* out_ids, float* out_dists,
                     uint32_t* out_counts) {
    const Elements& e = *(const Elements*)p;
    const size_t dim = e.dim;
    std::atomic<bool> bad{false};
    auto run = [&](size_t t) {
        Query q;
        std::vector<std::pair<float, u64>> all(index_len);
        for (size_t i = t; i < nq; i += (size_t)threads) {
            if (e.kind == KIND_I8 && already_element)
                q.q.assign(queries_i8 + i * dim, queries_i8 + (i + 1) * dim);
            else
                e.make_query(queries + i * dim, already_element != 0, &q);
            std::vector<float> x(dim);
            for (u64 j = 0; j < index_len; ++j) {
                const float d = e.dist_to_element(j, q);
                // angular_dist_f32 maps the NaN of 1 - dot to 0 where the reference panics (angular.rs:70): the
                // f32 kinds' dot is recomputed to see it
                if (e.kind != KIND_I8) {
                    const float* row = e.f32.data() + j * dim;
                    if (e.kind == KIND_SUM) {
                        e.raw_embedding(j, x.data());
                        normalize_f32(x.data(), dim);
                        row = x.data();
                    }
                    if (std::isnan(1.0f - dot_product_f32(row, q.f.data(), dim))) bad = true;
                }
                all[j] = {d, j};
            }
            const size_t m = std::min<u64>(k, index_len);
            std::partial_sort(all.begin(), all.begin() + m, all.end());  // (distance, id): keys are unique
            for (size_t r = 0; r < k; ++r) {
                out_ids[i * k + r] = r < m ? (u32)all[r].second : UNUSED;
                out_dists[i * k + r] = r < m ? all[r].first : INFINITY;
            }
            out_counts[i] = (u32)m;
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(run, (size_t)t);
    run(0);
    for (auto& th : pool) th.join();
    if (bad) {
        g_err = "NaN distance (the reference panics)";
        return -1;
    }
    return 0;
}

// `index`, `elements`: oracle objects (orc_index_from_bytes / orc_elements_from_bytes).  queries as orc_search_batch.
// filters: num_filters bitmaps of filter_words u32 words; query q uses bitmap query_filter[q] (null: 0) and admits id i
// iff bit (bit_base + i) is set.  Writes nq x k ids (UNUSED padded), distances (+inf padded), counts and, when stats is
// not null, nq x 3 {n_dist, n_expand, n_nbr_read} of the unfiltered search.  Returns 0, or -1 when a distance the search
// computes is NaN (the reference panics).
int orc_filtered_search(void* index, void* elements, const float* queries, const int8_t* queries_i8, uint64_t nq,
                        int already_element, uint64_t max_search, uint64_t k, const uint32_t* filters,
                        uint64_t filter_words, const uint32_t* query_filter, uint64_t bit_base, int threads,
                        uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint64_t* stats) {
    const Index& ix = *(const Index*)index;
    const Elements& el = *(const Elements*)elements;
    const size_t dim = el.dim, layers = ix.num_layers();
    std::atomic<bool> bad{false};
    auto run = [&](size_t t) {
        Query q;
        std::vector<float> x(dim);
        for (size_t i = t; i < nq; i += (size_t)threads) {
            if (el.kind == KIND_I8 && already_element)
                q.q.assign(queries_i8 + i * dim, queries_i8 + (i + 1) * dim);
            else
                el.make_query(queries + i * dim, already_element != 0, &q);
            SearchStats st;
            std::vector<u64> scored;
            if (layers > 0) {
                u64 entrypoint = 0;
                for (size_t l = 0; l + 1 < layers; ++l)
                    entrypoint = search_for_neighbors([&](size_t n, std::vector<u32>& o) { ix.get_neighbors(l, n, o); },
                                                      entrypoint, el, q, 1, &st)[0].first;
                scored.push_back(entrypoint);
                search_for_neighbors(
                    [&](size_t n, std::vector<u32>& o) {
                        ix.get_neighbors(layers - 1, n, o);
                        scored.insert(scored.end(), o.begin(), o.end());
                    },
                    entrypoint, el, q, max_search, &st);
            }
            std::sort(scored.begin(), scored.end());
            scored.erase(std::unique(scored.begin(), scored.end()), scored.end());
            // a NaN distance anywhere in the search: the reference panics (angular_dist_f32 maps the NaN of 1 - dot to
            // 0, so the f32 kinds' dot is recomputed to see it, as orc_exact_search does)
            if (el.kind != KIND_I8)
                for (u64 j : scored) {
                    const float* row = el.f32.data() + j * dim;
                    if (el.kind == KIND_SUM) {
                        el.raw_embedding(j, x.data());
                        normalize_f32(x.data(), dim);
                        row = x.data();
                    }
                    if (std::isnan(1.0f - dot_product_f32(row, q.f.data(), dim))) bad = true;
                }
            const uint32_t* bits = filters + (size_t)(query_filter ? query_filter[i] : 0) * filter_words;
            std::vector<std::pair<float, u64>> adm;
            for (u64 j : scored) {
                const u64 b = bit_base + j;
                if ((bits[b / 32] >> (b % 32)) & 1u) adm.emplace_back(el.dist_to_element(j, q), j);
            }
            std::sort(adm.begin(), adm.end());  // (distance, id): keys are unique
            const size_t m = std::min<size_t>(k, adm.size());
            for (size_t r = 0; r < k; ++r) {
                out_ids[i * k + r] = r < m ? (u32)adm[r].second : UNUSED;
                out_dists[i * k + r] = r < m ? adm[r].first : INFINITY;
            }
            out_counts[i] = (u32)m;
            if (stats) {
                stats[i * 3 + 0] = st.n_dist;
                stats[i * 3 + 1] = st.n_expand;
                stats[i * 3 + 2] = st.n_nbr_read;
            }
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(run, (size_t)t);
    run(0);
    for (auto& th : pool) th.join();
    if (bad) {
        g_err = "NaN distance (the reference panics)";
        return -1;
    }
    return 0;
}

// kind 0 (angular): angular::Vector::from(get_embedding(i)) = SumEmbeddings::get(i) (embeddings/mod.rs:164-166),
// normalize_f32 of the sum (angular.rs:55-61).  kind 1 (angular_int): angular_int::Vector::from(get_embedding(i)),
// quantize of the raw sum (parsing.rs:133-134, angular_int.rs:19-45), what the reference writes.
//
// `p` is a SumEmbeddings oracle container; `threads` stands for rayon's par_iter over a chunk (parsing.rs:133-134).
// Writes the file image to `out` (cap bytes, at least 8 + n * dim * {4|1}) and returns its length, or -1 where the
// reference panics (a NaN in an angular_int sum: NotNan::new(s.abs()).unwrap(), angular_int.rs:31) or where an angular
// row would hold NaN after normalising (a non-finite sum; every later distance to it panics, angular.rs:70).
int64_t orc_compute_embeddings(void* p, int kind, int threads, uint8_t* out, uint64_t cap) {
    const Elements& e = *(const Elements*)p;
    const size_t n = e.len();
    // get_embedding_internal (embeddings/mod.rs:124-143): an element without terms is zeros of the table width, or
    // the empty vector when the table has no rows
    const size_t width = e.num_embeddings > 0 ? e.dim : 0;
    const size_t esz = kind == 0 ? 4 : 1;
    std::atomic<bool> bad{false};
    uint64_t pos = 0;
    auto write = [&](const void* src, size_t len) {
        if (pos + len <= cap) std::memcpy(out + pos, src, len);
        pos += len;
    };
    // generate vectors in chunks to limit memory usage (parsing.rs:127-151)
    const size_t num_chunks = 100;
    const size_t chunk_size = (n + num_chunks - 1) / num_chunks;
    for (size_t i = 0; i < num_chunks; ++i) {
        const size_t begin = i * chunk_size, end = std::min((i + 1) * chunk_size, n);
        const size_t len = end > begin ? end - begin : 0;
        // chunk.par_iter().map(|&i| elements.get_embedding(i).into()).collect()
        std::vector<u8> vectors(len * width * esz);
        auto work = [&](size_t t) {
            std::vector<float> raw(e.dim);
            for (size_t j = t; j < len; j += (size_t)threads) {
                if (width == 0) continue;
                e.raw_embedding(begin + j, raw.data());
                for (size_t k = 0; k < width; ++k)
                    if (kind == 0 ? !std::isfinite(raw[k]) : std::isnan(raw[k])) bad = true;
                if (kind == 0) {
                    normalize_f32(raw.data(), width);
                    std::memcpy(&vectors[j * width * 4], raw.data(), width * 4);
                } else {
                    quantize_i8(raw.data(), width, reinterpret_cast<int8_t*>(&vectors[j * width]));
                }
            }
        };
        std::vector<std::thread> pool;
        for (int t = 1; t < threads; ++t) pool.emplace_back(work, (size_t)t);
        work(0);
        for (auto& th : pool) th.join();
        if (bad) {
            g_err = kind == 0 ? "a sum of embeddings is not finite" : "NaN in a sum of embeddings (the reference panics)";
            return -1;
        }
        // angular_int::Vectors::new() + push: the width of the first vector pushed, 0 for an empty chunk
        if (i == 0) {
            u8 header[8];
            write_uint_le(header, len > 0 ? width : 0, 8);
            write(header, 8);  // vectors.write(&mut file)
        }
        write(vectors.data(), vectors.size());  // write_as_bytes(vectors.as_slice())
    }
    return (int64_t)pos;
}

}  // extern "C"
