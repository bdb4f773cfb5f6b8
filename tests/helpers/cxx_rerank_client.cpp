// cxx_rerank_client.cpp — a C++ client of Granne::set_rerank_elements / search_rerank (include/granne_b200.hpp).
//
// Usage: cxx_rerank_client <index file> <angular_int elements file> <angular elements file> <queries file>
// The queries file holds raw f32 rows of the elements' width.  Searches them with max_search 50, 20 candidates and
// k = 5, and prints "id distance" per result, one per line (the caller compares them with the oracle).  Also checks
// that more than GRANNE_B200_RERANK_MAX_CANDIDATES candidates and a second attach throw.
#include <cstdio>
#include <cstring>
#include <vector>

#include "granne_b200.hpp"

int main(int argc, char** argv) {
    if (argc != 5) return 2;
    using namespace granne_b200;
    const Elements i8 = Elements::from_files(ElementKind::AngularInt, argv[2]);
    const Elements f32 = Elements::from_files(ElementKind::Angular, argv[3]);
    Granne g = Granne::from_file(argv[1], i8);
    g.set_rerank_elements(f32);
    const std::vector<uint8_t> raw = read_file(argv[4]);
    std::vector<float> q(raw.size() / 4);
    std::memcpy(q.data(), raw.data(), q.size() * 4);
    const size_t nq = q.size() / g.dim();
    const auto res = g.search_rerank(q.data(), nq, 50, 20, 5);
    for (const auto& r : res) {
        if (r.size() != 5) return 3;
        for (const auto& p : r) std::printf("%zu %.9g\n", p.first, p.second);
    }
    try {
        g.search_rerank(q.data(), 1, 2000, GRANNE_B200_RERANK_MAX_CANDIDATES + 1, 5);
        return 4;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 5;
    }
    try {
        g.set_rerank_elements(f32);
        return 6;
    } catch (const Error& e) {
        if (e.code() != GRANNE_B200_ERR_INVALID_ARGUMENT) return 7;
    }
    return 0;
}
