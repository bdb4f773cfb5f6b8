// exact_oracle.cpp — brute-force k nearest neighbours over the CPU oracle, the checker of
// granne_b200_exact_search_batch.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// It compiles the CPU oracle (oracle/granne_oracle.cpp) unchanged and adds one entry point beside it: for every query,
// the oracle's own Elements::dist_to_element (src/index/mod.rs:1012) for every element i < index_len, then a stable
// partial sort by (distance, id) — the order of into_sorted_vec (:1036).  Loaded through tests/helpers/exact_oracle.py.
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

}  // extern "C"
