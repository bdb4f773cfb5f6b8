// cxx_rerank_sum_client.cpp — a C++ client of Granne::set_rerank_elements with a SumEmbeddings container and
// search_rerank (include/granne_b200.hpp).
//
// Usage: cxx_rerank_sum_client <index file> <angular_int elements file> <term-list file> <embeddings file> <queries file>
// The angular_int elements are the compute_embeddings rows of the SumEmbeddings container (term lists, embeddings);
// the queries file holds raw f32 rows of the elements' width.  Searches them with max_search 50, 20 candidates and
// k = 5, and prints "id distance" per result, one per line (the caller compares them with the oracle).  Also checks
// that a second attach, of either kind, throws.
#include <cstdio>
#include <cstring>
#include <vector>

#include "granne_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 6) return 2;
    using namespace granne_b200;
    const Elements i8 = Elements::from_files(ElementKind::AngularInt, argv[2]);
    const Elements sum = Elements::from_files(ElementKind::Embeddings, argv[3], argv[4]);
    Granne g = Granne::from_file(argv[1], i8);
    g.set_rerank_elements(sum);
    const std::vector<uint8_t> raw = read_file(argv[5]);
    std::vector<float> q(raw.size() / 4);
    std::memcpy(q.data(), raw.data(), q.size() * 4);
    const size_t nq = q.size() / g.dim();
    const auto res = g.search_rerank(q.data(), nq, 50, 20, 5);
    for (const auto& r : res) {
        if (r.size() != 5) return 3;
        for (const auto& p : r) std::printf("%zu %.9g\n", p.first, p.second);
    }
    try {
        g.set_rerank_elements(sum);
        return 4;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 5;
    }
    try {
        g.set_rerank_elements(Elements::compute_embeddings(ElementKind::Angular, sum));
        return 6;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 7;
    }
    try {
        g.set_rerank_elements(i8);  // an angular_int container re-ranks nothing
        return 8;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 9;
    }
    return 0;
}
