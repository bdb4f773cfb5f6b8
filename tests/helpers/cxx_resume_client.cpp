// C++ client of GranneBuilder::from_bytes / from_file in include/granne_b200.hpp, written like the reference's
// read_index_reduce_num_neighbors (src/index/tests.rs:243-290).
//   cxx_resume_client nodevice <index> <elements>   without a GPU: every call fails with the status it should
//   cxx_resume_client gpu <dir>                      <dir>/elements: 1000 angular elements of width 5.  Writes
//                                                    <dir>/half.index and <dir>/resumed.index for the caller to check
#include <algorithm>
#include <cstdio>
#include <cstring>
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

template <class F>
static int error_code_of(F&& f) {
    try {
        f();
    } catch (const gb::Error& e) {
        return e.code();
    }
    return GRANNE_B200_OK;
}

static void write_file(const std::string& path, const std::vector<uint8_t>& bytes) {
    std::ofstream f(path, std::ios::binary);
    f.write(reinterpret_cast<const char*>(bytes.data()), static_cast<std::streamsize>(bytes.size()));
    if (!f) throw gb::Error(GRANNE_B200_ERR_IO, "could not write " + path);
}

static int nodevice(const std::string& index_path, const std::string& elements_path) {
    const gb::Elements elements = gb::Elements::from_files(gb::ElementKind::Angular, elements_path);
    const std::vector<uint8_t> image = gb::read_file(index_path);
    const gb::BuildConfig config = gb::BuildConfig().max_search(10).num_neighbors(5);
    // the image is checked before the device: a damaged one is a format error even here
    const std::vector<uint8_t> cut(image.begin(), image.begin() + image.size() / 2);
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_bytes(config, cut, elements); }) == GRANNE_B200_ERR_FORMAT);
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_bytes(config.num_neighbors(0), image, elements); }) ==
            GRANNE_B200_ERR_INVALID_ARGUMENT);
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_file(config, "/nonexistent/granne", elements); }) ==
            GRANNE_B200_ERR_IO);
    // a valid image: no CPU fallback
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_bytes(config, image, elements); }) == GRANNE_B200_ERR_NO_DEVICE);
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_file(config, index_path, elements); }) ==
            GRANNE_B200_ERR_NO_DEVICE);
    std::printf("nodevice ok\n");
    return 0;
}

static int gpu(const std::string& dir) {
    const size_t num_elements = 1000;
    const gb::Elements elements = gb::Elements::from_files(gb::ElementKind::Angular, dir + "/elements");
    REQUIRE(elements.len() == num_elements && elements.dim() == 5);

    gb::GranneBuilder builder(gb::BuildConfig().max_search(10).num_neighbors(20), elements);
    builder.build_partial(num_elements / 2);
    const std::vector<uint8_t> image = builder.write_index();
    write_file(dir + "/half.index", image);
    // "not necessarily true, but should be valid"
    REQUIRE(builder.get_neighbors(0, builder.num_layers() - 1).size() > 5);

    // lower num_neighbors
    const gb::BuildConfig config = gb::BuildConfig().max_search(10).num_neighbors(5);
    gb::GranneBuilder owning_builder = gb::GranneBuilder::from_file(config, dir + "/half.index", elements);
    const gb::GranneBuilder from_bytes = gb::GranneBuilder::from_bytes(config, image, elements);
    REQUIRE(builder.len() == num_elements / 2);
    REQUIRE(owning_builder.len() == num_elements / 2 && from_bytes.len() == num_elements / 2);
    REQUIRE(owning_builder.num_layers() == builder.num_layers() && from_bytes.num_layers() == builder.num_layers());
    REQUIRE(owning_builder.write_index() == from_bytes.write_index());
    for (size_t layer = 0; layer < owning_builder.num_layers(); ++layer) {
        REQUIRE(owning_builder.layer_len(layer) == builder.layer_len(layer));
        for (size_t i = 0; i < owning_builder.layer_len(layer); ++i) {
            // the first five of the stored (ascending) ids
            std::vector<size_t> want = builder.get_neighbors(i, layer);
            std::sort(want.begin(), want.end());
            if (want.size() > 5) want.resize(5);
            REQUIRE(owning_builder.get_neighbors(i, layer) == want);
        }
    }

    owning_builder.build();
    REQUIRE(owning_builder.len() == num_elements);
    REQUIRE(owning_builder.get_neighbors(0, owning_builder.num_layers() - 1).size() <= 5);
    for (size_t layer = 0; layer < owning_builder.num_layers(); ++layer)
        for (size_t i = 0; i < owning_builder.layer_len(layer); ++i)
            REQUIRE(owning_builder.get_neighbors(i, layer).size() <= 5);
    write_file(dir + "/resumed.index", owning_builder.write_index());
    // "Cannot index fewer elements than already in index." (mod.rs:379-382)
    REQUIRE(error_code_of([&] { owning_builder.build_partial(10); }) == GRANNE_B200_ERR_INVALID_ARGUMENT);

    // an index over more elements than the container holds
    gb::Elements fewer = elements;
    fewer.bytes.resize(8 + 400 * 5 * 4);
    REQUIRE(fewer.len() == 400);
    REQUIRE(error_code_of([&] { gb::GranneBuilder::from_bytes(config, image, fewer); }) == GRANNE_B200_ERR_FORMAT);
    std::printf("gpu ok\n");
    return 0;
}

int main(int argc, char** argv) {
    try {
        if (argc > 2 && std::strcmp(argv[1], "gpu") == 0) return gpu(argv[2]);
        if (argc > 3 && std::strcmp(argv[1], "nodevice") == 0) return nodevice(argv[2], argv[3]);
        std::printf("usage: cxx_resume_client nodevice <index> <elements> | gpu <dir>\n");
        return 2;
    } catch (const gb::Error& e) {
        std::printf("granne_b200::Error %d: %s\n", e.code(), e.what());
        return 2;
    }
}
