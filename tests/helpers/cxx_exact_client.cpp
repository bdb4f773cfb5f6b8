// cxx_exact_client.cpp — a C++ client of Granne::exact_search_batch (include/granne_b200.hpp).
//
// Usage: cxx_exact_client <index file> <angular elements file>
// Searches the first four elements as ELEMENT queries for their 5 exact nearest neighbours and prints the ids, one
// per line (the caller compares them with the oracle).  Also checks that k above GRANNE_B200_EXACT_MAX_K throws.
#include <cstdio>
#include <vector>

#include "granne_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    using namespace granne_b200;
    const Elements elements = Elements::from_files(ElementKind::Angular, argv[2]);
    const Granne g = Granne::from_file(argv[1], elements);
    const size_t dim = g.dim();
    std::vector<float> q;
    for (size_t i = 0; i < 4; ++i) {
        const std::vector<float> e = g.get_element(i);
        q.insert(q.end(), e.begin(), e.end());
    }
    const auto res = g.exact_search_batch(q.data(), 4, GRANNE_B200_QUERY_ELEMENT, 5);
    for (const auto& r : res) {
        if (r.size() != 5) return 3;
        for (const auto& p : r) std::printf("%zu\n", p.first);
    }
    try {
        g.exact_search_batch(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, GRANNE_B200_EXACT_MAX_K + 1);
        return 4;
    } catch (const Error&) {
    }
    (void)dim;
    return 0;
}
