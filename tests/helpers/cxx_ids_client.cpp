// C++ client of the id queries (GRANNE_B200_QUERY_ID*): the reference's self-recall check (verify_search,
// src/index/tests.rs:50-62 — search(get_element(i), max_search, 1) for every i) as one batched call by id, checked
// against the per-element loop, and knn_graph without self.
// Usage: cxx_ids_client <index file> <angular elements file>; prints "recall <r>" and "ok".
#include <cstdio>

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
    if (argc != 3) return 2;
    try {
        const gb::Elements elements = gb::Elements::from_files(gb::ElementKind::Angular, argv[2]);
        const gb::Granne index = gb::Granne::from_bytes(gb::read_file(argv[1]), elements);
        std::vector<uint32_t> ids(index.len());
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<uint32_t>(i);
        const std::vector<gb::SearchResult> batched = index.search_by_id(ids, 100, 1);
        size_t found = 0;
        for (size_t i = 0; i < ids.size(); ++i) {
            REQUIRE(batched[i] == index.search(index.get_element(i), 100, 1));
            found += (!batched[i].empty() && batched[i][0].first == i) ? 1 : 0;
        }
        const std::vector<float> rows = index.get_elements(ids);
        REQUIRE(rows.size() == ids.size() * index.dim());
        REQUIRE(std::vector<float>(rows.begin(), rows.begin() + index.dim()) == index.get_element(0));
        const std::vector<gb::SearchResult> graph = index.knn_graph(100, 5, true, false, 333);
        REQUIRE(graph.size() == ids.size());
        for (size_t i = 0; i < graph.size(); ++i) {
            REQUIRE(graph[i] == index.search_by_id({ids[i]}, 100, 5, true).at(0));
            for (const auto& e : graph[i]) REQUIRE(e.first != i);
        }
        std::printf("recall %.6f\nok\n", ids.empty() ? 1.0 : static_cast<double>(found) / static_cast<double>(ids.size()));
    } catch (const gb::Error& e) {
        std::fprintf(stderr, "error %d: %s\n", e.code(), e.what());
        return 1;
    }
    return 0;
}
