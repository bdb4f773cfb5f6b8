// embeddings_oracle.cpp — CPU restatement of compute_embeddings_and_save_to_disk
// (src/elements/embeddings/parsing.rs:102-152), the checker of granne_b200_compute_embeddings.
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// It compiles the CPU oracle (oracle/granne_oracle.cpp) unchanged and adds this one entry point beside it, so that the
// sum (Elements::raw_embedding), quantize_i8 and normalize_f32 it uses are the oracle's own.  Loaded through
// tests/helpers/embeddings_oracle.py.
#include "../../oracle/granne_oracle.cpp"

extern "C" {

// kind 0 (angular): angular::Vector::from(get_embedding(i)) = SumEmbeddings::get(i) (embeddings/mod.rs:164-166),
// normalize_f32 of the sum (angular.rs:55-61).  kind 1 (angular_int): angular_int::Vector::from(get_embedding(i)),
// quantize of the raw sum (parsing.rs:133-134, angular_int.rs:19-45), what the reference writes.
//
// `p` is a SumEmbeddings oracle container; `threads` stands for rayon's par_iter over a chunk (parsing.rs:133-134).
// Writes the file image to `out` (cap bytes, at least 8 + n * dim * {4|1}) and returns its length, or -1 where the
// reference panics (a NaN in an angular_int sum: NotNan::new(s.abs()).unwrap(), angular_int.rs:31) or where an angular
// row would hold NaN after normalising (a non-finite sum; every later distance to it panics, angular.rs:70).
int64_t orc_compute_embeddings(void* p, int kind, int threads, uint8_t* out, uint64_t cap) {
    const Elements& e = *(const Elements*)p;
    const size_t n = e.len();
    // get_embedding_internal (embeddings/mod.rs:124-143): an element without terms is zeros of the table width, or
    // the empty vector when the table has no rows
    const size_t width = e.num_embeddings > 0 ? e.dim : 0;
    const size_t esz = kind == 0 ? 4 : 1;
    std::atomic<bool> bad{false};
    uint64_t pos = 0;
    auto write = [&](const void* src, size_t len) {
        if (pos + len <= cap) std::memcpy(out + pos, src, len);
        pos += len;
    };
    // generate vectors in chunks to limit memory usage (parsing.rs:127-151)
    const size_t num_chunks = 100;
    const size_t chunk_size = (n + num_chunks - 1) / num_chunks;
    for (size_t i = 0; i < num_chunks; ++i) {
        const size_t begin = i * chunk_size, end = std::min((i + 1) * chunk_size, n);
        const size_t len = end > begin ? end - begin : 0;
        // chunk.par_iter().map(|&i| elements.get_embedding(i).into()).collect()
        std::vector<u8> vectors(len * width * esz);
        auto work = [&](size_t t) {
            std::vector<float> raw(e.dim);
            for (size_t j = t; j < len; j += (size_t)threads) {
                if (width == 0) continue;
                e.raw_embedding(begin + j, raw.data());
                for (size_t k = 0; k < width; ++k)
                    if (kind == 0 ? !std::isfinite(raw[k]) : std::isnan(raw[k])) bad = true;
                if (kind == 0) {
                    normalize_f32(raw.data(), width);
                    std::memcpy(&vectors[j * width * 4], raw.data(), width * 4);
                } else {
                    quantize_i8(raw.data(), width, reinterpret_cast<int8_t*>(&vectors[j * width]));
                }
            }
        };
        std::vector<std::thread> pool;
        for (int t = 1; t < threads; ++t) pool.emplace_back(work, (size_t)t);
        work(0);
        for (auto& th : pool) th.join();
        if (bad) {
            g_err = kind == 0 ? "a sum of embeddings is not finite" : "NaN in a sum of embeddings (the reference panics)";
            return -1;
        }
        // angular_int::Vectors::new() + push: the width of the first vector pushed, 0 for an empty chunk
        if (i == 0) {
            u8 header[8];
            write_uint_le(header, len > 0 ? width : 0, 8);
            write(header, 8);  // vectors.write(&mut file)
        }
        write(vectors.data(), vectors.size());  // write_as_bytes(vectors.as_slice())
    }
    return (int64_t)pos;
}

}  // extern "C"
