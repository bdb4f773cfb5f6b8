// cxx_within_client.cpp — a C++ client of Granne::exact_search_within (include/granne_b200.hpp).
//
// Usage: cxx_within_client <index file> <angular elements file>
// Ranks the overlapping list 0..99, 50..149 for element 7 as an ELEMENT query with k = 5 and prints "id distance"
// per result, one per line (the caller compares them with the oracle).  Also checks that an id >= len() and a list
// count other than nq throw ERR_INVALID_ARGUMENT.
#include <cstdio>
#include <vector>

#include "granne_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    using namespace granne_b200;
    const Elements el = Elements::from_files(ElementKind::Angular, argv[2]);
    Granne g = Granne::from_file(argv[1], el);
    const std::vector<float> q = g.get_element(7);
    std::vector<uint32_t> list;
    for (uint32_t i = 0; i < 100; ++i) list.push_back(i);
    for (uint32_t i = 50; i < 150; ++i) list.push_back(i);
    const auto res = g.exact_search_within(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, {list}, 5);
    if (res.size() != 1 || res[0].size() != 5) return 3;
    for (const auto& p : res[0]) std::printf("%zu %.9g\n", p.first, p.second);
    try {
        g.exact_search_within(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, {{static_cast<uint32_t>(g.len())}}, 5);
        return 4;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 5;
    }
    try {
        g.exact_search_within(q.data(), 1, GRANNE_B200_QUERY_ELEMENT, {}, 5);
        return 6;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 7;
    }
    return 0;
}
