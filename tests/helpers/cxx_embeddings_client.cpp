// C++ client of Elements::compute_embeddings in include/granne_b200.hpp (compute_embeddings_and_save_to_disk,
// src/elements/embeddings/parsing.rs:102-152).
//   cxx_embeddings_client gpu <dir>   <dir>/elements, <dir>/embeddings: a SumEmbeddings container.  Materialises it
//                                     as angular and angular_int vectors, writes <dir>/angular and <dir>/angular_int
//                                     for the caller to compare, builds an index over each and searches it with every
//                                     element's own row.
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "granne_b200.hpp"

namespace gb = granne_b200;

#define REQUIRE(cond)                                                      \
    do {                                                                   \
        if (!(cond)) {                                                     \
            std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);  \
            return 1;                                                      \
        }                                                                  \
    } while (0)

static void write_file(const std::string& path, const std::vector<uint8_t>& bytes) {
    std::ofstream f(path, std::ios::binary);
    f.write(reinterpret_cast<const char*>(bytes.data()), static_cast<std::streamsize>(bytes.size()));
    if (!f) throw gb::Error(GRANNE_B200_ERR_IO, "could not write " + path);
}

static int gpu(const std::string& dir) {
    const gb::Elements sum = gb::Elements::from_files(gb::ElementKind::Embeddings, dir + "/elements", dir + "/embeddings");
    const uint64_t n = sum.len();
    const uint64_t dim = gb::Elements::from_files(gb::ElementKind::Angular, dir + "/embeddings").dim();
    REQUIRE(n > 100);
    const gb::Elements angular = gb::Elements::compute_embeddings(gb::ElementKind::Angular, sum);
    const gb::Elements angular_int = gb::Elements::compute_embeddings(gb::ElementKind::AngularInt, sum);
    REQUIRE(angular.kind == gb::ElementKind::Angular && angular.len() == n && angular.dim() == dim);
    REQUIRE(angular_int.kind == gb::ElementKind::AngularInt && angular_int.len() == n && angular_int.dim() == dim);
    write_file(dir + "/angular", angular.bytes);
    write_file(dir + "/angular_int", angular_int.bytes);

    // every element finds itself among its nearest neighbours in both materialised containers
    for (const gb::Elements* el : {&angular, &angular_int}) {
        gb::GranneBuilder builder(gb::BuildConfig().max_search(50).num_neighbors(20), *el);
        builder.build();
        const gb::Granne index = gb::Granne::from_bytes(builder.write_index(), *el);
        REQUIRE(index.len() == n);
        size_t found = 0;
        for (uint64_t i = 0; i < n; ++i) {
            const gb::SearchResult r = el->kind == gb::ElementKind::Angular ? index.search(index.get_element(i), 50, 5)
                                                                           : index.search(index.get_element_i8(i), 50, 5);
            bool self = false;
            for (const auto& hit : r) self = self || hit.first == i || hit.second == 0.0f;  // or an equal row
            found += self;
        }
        REQUIRE(found >= n * 95 / 100);
    }
    std::printf("gpu ok\n");
    return 0;
}

int main(int argc, char** argv) {
    try {
        if (argc == 3 && std::string(argv[1]) == "gpu") return gpu(argv[2]);
    } catch (const gb::Error& e) {
        std::printf("FAILED: %s\n", e.what());
        return 1;
    }
    std::printf("usage: cxx_embeddings_client gpu <dir>\n");
    return 2;
}
