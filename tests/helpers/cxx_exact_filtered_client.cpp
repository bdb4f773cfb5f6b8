// cxx_exact_filtered_client.cpp — a C++ client of Granne::exact_search_filtered (include/granne_b200.hpp).
//
// Usage: cxx_exact_filtered_client <index file> <angular elements file>
// Searches for element 7 as an ELEMENT query with k = 5 under the filter that admits the odd ids, and prints
// "id distance" per result, one per line (the caller compares them with the oracle).  Also checks that a bitmap
// narrower than ceil(len() / 32) words and a query_filter entry >= num_filters throw ERR_INVALID_ARGUMENT.
#include <cstdio>
#include <vector>

#include "granne_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    using namespace granne_b200;
    const Elements el = Elements::from_files(ElementKind::Angular, argv[2]);
    Granne g = Granne::from_file(argv[1], el);
    const std::vector<float> q = g.get_element(7);
    const uint64_t words = (g.len() + 31) / 32;
    const std::vector<uint32_t> odd(words, 0xAAAAAAAAu);
    const auto res = g.exact_search_filtered(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, 5, odd.data(), 1, words);
    if (res.size() != 1) return 3;
    for (const auto& p : res[0]) std::printf("%zu %.9g\n", p.first, p.second);
    try {
        g.exact_search_filtered(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, 5, odd.data(), 1, words - 1);
        return 4;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 5;
    }
    const uint32_t bad = 1;
    try {
        g.exact_search_filtered(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, 5, odd.data(), 1, words, &bad);
        return 6;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 7;
    }
    return 0;
}
