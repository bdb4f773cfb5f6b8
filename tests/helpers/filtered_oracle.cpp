// filtered_oracle.cpp — filtered search composed from the CPU oracle's own pieces, the checker of
// granne_b200_search_filtered_batch.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// It compiles the CPU oracle (oracle/granne_oracle.cpp) unchanged and adds one entry point beside it.  Per query:
//   1. the oracle's upper-layer descent (search_for_neighbors with max_search = 1 per layer, as index_search does);
//   2. the oracle's search_for_neighbors on the bottom layer B with the caller's max_search, through a GetNeighbors
//      that records every neighbour it returns.  It is called exactly once per expansion, and every neighbour it
//      returns is scored unless already visited, so the recorded ids plus the entrypoint are S(q), the elements whose
//      distance the search computes in B;
//   3. the filter applied to S(q), and Elements::dist_to_element for each admitted id;
//   4. a sort by (distance, id) — the order of into_sorted_vec (src/index/mod.rs:1036) — and the first k.
// Loaded through tests/helpers/filtered_oracle.py.
#include "../../oracle/granne_oracle.cpp"

extern "C" {

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
            // 0, so the f32 kinds' dot is recomputed to see it, as exact_oracle.cpp does)
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

}  // extern "C"
