// cxx_diverse_client.cpp — a C++ client of granne_b200_search_diverse_batch and granne_b200_select_neighbors_batch
// through the C header (include/granne_b200.h).
//
// Usage: cxx_diverse_client <index file> <angular elements file> <queries file> <nq> <max_search> <k>
// The queries file holds nq raw f32 rows of the elements' width.  Prints each query's diverse ids on one line (the
// caller compares them with the Python binding), after checking that the selection over search_batch(q, max_search,
// max_search) gives the same lists and that max_search above GRANNE_B200_DIVERSE_MAX_CANDIDATES is rejected.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "granne_b200.h"

int main(int argc, char** argv) {
    if (argc != 7) return 2;
    const size_t nq = std::strtoull(argv[4], nullptr, 10);
    const uint32_t ef = (uint32_t)std::strtoul(argv[5], nullptr, 10), k = (uint32_t)std::strtoul(argv[6], nullptr, 10);
    granne_b200_index* h = nullptr;
    if (granne_b200_open_files(argv[1], GRANNE_B200_ANGULAR, argv[2], nullptr, 0, &h) != GRANNE_B200_OK) return 3;
    const size_t dim = granne_b200_dim(h);
    std::vector<float> q(nq * dim);
    FILE* f = std::fopen(argv[3], "rb");
    if (!f || std::fread(q.data(), 4, q.size(), f) != q.size()) return 4;
    std::fclose(f);
    std::vector<uint32_t> ids(nq * k), counts(nq), ci(nq * ef), cc(nq), si(nq * k), sc(nq);
    std::vector<float> d(nq * k), cd(nq * ef), sd(nq * k);
    if (granne_b200_search_diverse_batch(h, q.data(), nq, GRANNE_B200_QUERY_RAW_F32, ef, k, ids.data(), d.data(),
                                         counts.data(), nullptr) != GRANNE_B200_OK)
        return 5;
    if (granne_b200_search_batch(h, q.data(), nq, GRANNE_B200_QUERY_RAW_F32, ef, ef, ci.data(), cd.data(), cc.data(),
                                 nullptr) != GRANNE_B200_OK ||
        granne_b200_select_neighbors_batch(h, ci.data(), cd.data(), cc.data(), nq, ef, k, si.data(), sd.data(),
                                           sc.data()) != GRANNE_B200_OK)
        return 6;
    if (si != ids || sc != counts) return 7;
    if (granne_b200_search_diverse_batch(h, q.data(), nq, GRANNE_B200_QUERY_RAW_F32,
                                         GRANNE_B200_DIVERSE_MAX_CANDIDATES + 1, k, ids.data(), d.data(),
                                         counts.data(), nullptr) != GRANNE_B200_ERR_INVALID_ARGUMENT)
        return 8;
    for (size_t i = 0; i < nq; ++i) {
        for (uint32_t j = 0; j < sc[i]; ++j) std::printf(j ? " %u" : "%u", si[i * k + j]);
        std::printf("\n");
    }
    granne_b200_close(h);
    return 0;
}
