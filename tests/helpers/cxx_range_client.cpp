// C++ client of the exact range search: for every element as a query (by id), the range at the radius given is
// checked against exact_search_batch's first k entries within it (the identity the range search keeps), and the
// excluding form against the same list without the query's own id.
// Usage: cxx_range_client <index file> <angular elements file> <radius>; prints "entries <n>" and "ok".
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "granne_b200.hpp"

namespace gb = granne_b200;

#define REQUIRE(c)                                                   \
    do {                                                             \
        if (!(c)) {                                                  \
            std::fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                \
        }                                                            \
    } while (0)

int main(int argc, char** argv) {
    if (argc != 4) return 2;
    try {
        const gb::Elements elements = gb::Elements::from_files(gb::ElementKind::Angular, argv[2]);
        const gb::Granne index = gb::Granne::from_bytes(gb::read_file(argv[1]), elements);
        const float radius = std::strtof(argv[3], nullptr);
        std::vector<uint32_t> ids(index.len());
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<uint32_t>(i);
        const auto range = index.exact_range_search(ids.data(), ids.size(), GRANNE_B200_QUERY_ID, radius);
        const auto without = index.exact_range_search(ids.data(), ids.size(), GRANNE_B200_QUERY_ID_EXCLUDING, radius);
        const size_t k = 64;
        const auto top = index.exact_search_by_id(ids, k);
        size_t entries = 0;
        REQUIRE(range.size() == ids.size() && without.size() == ids.size());
        for (size_t i = 0; i < ids.size(); ++i) {
            gb::SearchResult cut;
            for (const auto& e : top[i])
                if (e.second <= radius) cut.push_back(e);
            const size_t m = std::min(k, range[i].size());
            REQUIRE(gb::SearchResult(range[i].begin(), range[i].begin() + m) == cut);
            gb::SearchResult rest;
            for (const auto& e : range[i])
                if (e.first != i) rest.push_back(e);
            REQUIRE(rest == without[i]);
            entries += range[i].size();
        }
        std::printf("entries %zu\nok\n", entries);
    } catch (const gb::Error& e) {
        std::fprintf(stderr, "error %d: %s\n", e.code(), e.what());
        return 1;
    }
    return 0;
}
