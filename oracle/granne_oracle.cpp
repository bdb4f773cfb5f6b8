// granne_oracle.cpp — CPU restatement of granne's search path (and of the builder that feeds it).
//
// *** TEST INFRASTRUCTURE, NOT PRODUCT CODE. ***
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference` legs may load this
// library, and only as the checker / CPU baseline.  Nothing under granne_b200/ links, imports or calls it.
//
// Parity status: PARITY UNPINNED against a run of the reference — pinned only to the reference's own known-answer
// tests (below) and, for the Stream VByte bytes, to an independent third statement
// (tests/test_stream_vbyte_independent.py).  The reference is Rust (granne 0.5.2); there is no rustc/cargo in this image, so the reference
// itself cannot be compiled or run here, and its own tests use unseeded random data (src/test_helper.rs:3-18), so
// no golden *search results* exist.  The restatement is pinned against every known-answer test the reference holds
// for this path (tests/test_oracle_kat.py): layer sizes (src/index/tests.rs:305-335), delta coding
// (src/slice_vector/set_vector.rs:231-248), the raw-vs-vbyte size rule (set_vector.rs:275-283), odd-byte ints
// (src/odd_byte_int.rs:43-79), dot/sum/dist tolerances (src/math.rs:166-196, src/elements/angular.rs:97-126),
// self-recall > 0.95 (src/index/tests.rs:41-62,114-132) and format round-trips (src/index/tests.rs:337-451);
// tests/test_oracle_formats_kat.py adds Offsets (src/slice_vector/offsets.rs:302-351), the MultiSetVector writers
// (set_vector.rs:318-425), the variable-width element container, select_neighbors / empty_build / write_and_load /
// incremental builds (src/index/tests.rs:11-40,134-242,292-417); tests/test_oracle_reorder.py the reorder and
// permute tests (src/index/reorder.rs:294-334, src/slice_vector/mod.rs:1028-1092, embeddings/reorder.rs:60-102).
// Byte-level parity of the stream-vbyte coding (third-party crate stream-vbyte 0.3.2, Cargo.toml:42, not vendored
// under /root/reference) is restated from the published Stream VByte layout and is otherwise UNPINNED.
//
// Every function cites the reference file:line it follows (paths relative to /root/reference).
//
// Build: g++ -O3 -std=c++17 -mavx2 -mfma -ffp-contract=off -fPIC -shared -pthread (see oracle/Makefile).

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <queue>
#include <string>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

using u8 = uint8_t;
using u32 = uint32_t;
using u64 = uint64_t;

constexpr u32 UNUSED = 0xFFFFFFFFu;  // src/index/mod.rs:27-28

// ---------------------------------------------------------------------------------------------------------------
// math  (src/math.rs)
// ---------------------------------------------------------------------------------------------------------------

// src/math.rs:16-42  — 32 FMA accumulators over chunks_exact(32), ordered lane sum, FMA tail.
float dot_product_f32(const float* x, const float* y, size_t n) {
    constexpr size_t CHUNK = 32;
    float chunk[CHUNK];
    for (size_t i = 0; i < CHUNK; ++i) chunk[i] = 0.0f;
    size_t full = n / CHUNK;
    for (size_t c = 0; c < full; ++c) {
        const float* a = x + c * CHUNK;
        const float* b = y + c * CHUNK;
        for (size_t i = 0; i < CHUNK; ++i) chunk[i] = std::fmaf(a[i], b[i], chunk[i]);
    }
    float r = 0.0f;
    for (size_t i = 0; i < CHUNK; ++i) r += chunk[i];
    for (size_t i = full * CHUNK; i < n; ++i) r = std::fmaf(x[i], y[i], r);
    return r;
}

// src/math.rs:59-89 — exact i32 accumulation of r, dx, dy.
void dot_product_and_squared_norms_i8(const int8_t* x, const int8_t* y, size_t n, int32_t* r, int32_t* dx,
                                      int32_t* dy) {
    int32_t rr = 0, ddx = 0, ddy = 0;
    for (size_t i = 0; i < n; ++i) {
        int32_t xi = x[i], yi = y[i];
        rr += xi * yi;
        ddx += xi * xi;
        ddy += yi * yi;
    }
    *r = rr;
    *dx = ddx;
    *dy = ddy;
}

// src/math.rs:92-116
void sum_into_f32(float* x, const float* y, size_t n) {
    for (size_t i = 0; i < n; ++i) x[i] += y[i];
}

// src/math.rs:124-150 — norm = sqrt(dot(x,x)); if norm > 0 { x[i] /= norm }
void normalize_f32(float* x, size_t n) {
    float norm = std::sqrt(dot_product_f32(x, x, n));
    if (norm > 0.0f) {
        for (size_t i = 0; i < n; ++i) x[i] /= norm;
    }
}

// src/elements/angular.rs:63-74 — d = max(0, 1 - dot).  NaN panics in the reference (NotNan::new().unwrap()).
float angular_dist_f32(const float* x, const float* y, size_t n) {
    float r = dot_product_f32(x, y, n);
    float d = 1.0f - r;
    return (0.0f <= d) ? d : 0.0f;  // cmp::max(0.0, d) returns d when equal / greater
}

// src/elements/angular_int.rs:47-59
float angular_dist_i8(const int8_t* x, const int8_t* y, size_t n) {
    int32_t ri, dxi, dyi;
    dot_product_and_squared_norms_i8(x, y, n, &ri, &dxi, &dyi);
    float r = (float)ri, dx = (float)dxi, dy = (float)dyi;
    float q = r / (std::sqrt(dx) * std::sqrt(dy));
    if (std::isnan(q)) q = 0.0f;  // NotNan::new(..).unwrap_or_else(|_| 0.0)
    float d = 1.0f - q;
    return (0.0f <= d) ? d : 0.0f;
}

// src/elements/angular_int.rs:28-45 — vi = x * 127 / max|x|, `as i8` (truncate toward zero, saturating, NaN->0).
void quantize_i8(const float* s, size_t n, int8_t* out) {
    float max_value = 127.0f;  // unwrap_or_else for empty input
    bool any = false;
    for (size_t i = 0; i < n; ++i) {
        float a = std::fabs(s[i]);
        if (!any || a > max_value) {
            max_value = a;
            any = true;
        }
    }
    for (size_t i = 0; i < n; ++i) {
        float vi = s[i] * 127.0f / max_value;
        int8_t q;
        if (std::isnan(vi))
            q = 0;
        else if (vi >= 127.0f)
            q = 127;
        else if (vi <= -128.0f)
            q = -128;
        else
            q = (int8_t)(int32_t)vi;  // truncation toward zero
        out[i] = q;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// odd byte ints (src/odd_byte_int.rs:3-36)
// ---------------------------------------------------------------------------------------------------------------
u64 read_uint_le(const u8* p, int nbytes) {
    u64 v = 0;
    for (int i = 0; i < nbytes; ++i) v |= (u64)p[i] << (8 * i);
    return v;
}
void write_uint_le(u8* p, u64 v, int nbytes) {
    for (int i = 0; i < nbytes; ++i) p[i] = (u8)(v >> (8 * i));
}

// ---------------------------------------------------------------------------------------------------------------
// element containers (src/elements/mod.rs:17-45)
// ---------------------------------------------------------------------------------------------------------------
enum ElemKind { KIND_F32 = 0, KIND_I8 = 1, KIND_SUM = 2 };

struct Query {  // Elements::Element — a normalised f32 vector or an i8 vector
    std::vector<float> f;
    std::vector<int8_t> q;
};

struct Elements {
    int kind = KIND_F32;
    size_t dim = 0;
    size_t n = 0;
    std::vector<float> f32;  // KIND_F32 rows; KIND_SUM: embeddings rows
    std::vector<int8_t> i8;  // KIND_I8 rows
    // KIND_SUM (src/elements/embeddings/mod.rs:41-44): element -> list of embedding ids
    size_t num_embeddings = 0;
    std::vector<u64> offsets;  // n+1
    std::vector<u32> terms;

    size_t len() const { return n; }

    // src/elements/embeddings/mod.rs:124-143 (get_embedding_internal) — ordered sum of rows
    void raw_embedding(size_t idx, float* out) const {
        u64 b = offsets[idx], e = offsets[idx + 1];
        if (b == e) {
            for (size_t i = 0; i < dim; ++i) out[i] = 0.0f;
            return;
        }
        std::memcpy(out, &f32[(size_t)terms[b] * dim], dim * sizeof(float));
        for (u64 t = b + 1; t < e; ++t) sum_into_f32(out, &f32[(size_t)terms[t] * dim], dim);
    }

    // ElementContainer::get  (dense_vector.rs:141-143; embeddings/mod.rs:164-166)
    void get(size_t idx, Query* out) const {
        if (kind == KIND_F32) {
            out->f.assign(&f32[idx * dim], &f32[idx * dim] + dim);
        } else if (kind == KIND_I8) {
            out->q.assign(&i8[idx * dim], &i8[idx * dim] + dim);
        } else {
            out->f.resize(dim);
            raw_embedding(idx, out->f.data());
            normalize_f32(out->f.data(), dim);  // Vector::from(Vec<f32>) (angular.rs:55-61)
        }
    }

    // ElementContainer::dist_to_element (dense_vector.rs:149-151; embeddings/mod.rs:172-174)
    float dist_to_element(size_t idx, const Query& q) const {
        if (kind == KIND_F32) return angular_dist_f32(&f32[idx * dim], q.f.data(), dim);
        if (kind == KIND_I8) return angular_dist_i8(&i8[idx * dim], q.q.data(), dim);
        std::vector<float> tmp(dim);  // the reference allocates a Vec per call too
        raw_embedding(idx, tmp.data());
        normalize_f32(tmp.data(), dim);
        return angular_dist_f32(tmp.data(), q.f.data(), dim);
    }

    // ElementContainer::dist (elements/mod.rs:31-33 / dense_vector.rs:153-155)
    float dist(size_t i, size_t j) const {
        Query q;
        get(j, &q);
        return dist_to_element(i, q);
    }

    // Query construction from a caller's raw f32 vector: angular.rs:55-61 / angular_int.rs:19-45
    void make_query(const float* raw, bool already_element, Query* out) const {
        if (kind == KIND_I8) {
            out->q.resize(dim);
            quantize_i8(raw, dim, out->q.data());
        } else {
            out->f.assign(raw, raw + dim);
            if (!already_element) normalize_f32(out->f.data(), dim);
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Stream VByte (scalar) — third-party crate stream-vbyte 0.3.2; layout restated from the published format:
// ceil(n/4) control bytes, then data; 2-bit code = byte_length-1, number i of a quad in bits [2i,2i+1]; LE bytes.
// ---------------------------------------------------------------------------------------------------------------
size_t svb_encode(const u32* in, size_t n, std::vector<u8>& out) {
    size_t nctrl = (n + 3) / 4;
    size_t base = out.size();
    out.resize(base + nctrl, 0);
    for (size_t i = 0; i < n; ++i) {
        u32 v = in[i];
        int len = v < (1u << 8) ? 1 : v < (1u << 16) ? 2 : v < (1u << 24) ? 3 : 4;
        out[base + i / 4] |= (u8)((len - 1) << (2 * (i % 4)));
        for (int b = 0; b < len; ++b) out.push_back((u8)(v >> (8 * b)));
    }
    return out.size() - base;
}

size_t svb_decode(const u8* in, size_t n, u32* out) {
    size_t nctrl = (n + 3) / 4;
    const u8* data = in + nctrl;
    for (size_t i = 0; i < n; ++i) {
        int len = ((in[i / 4] >> (2 * (i % 4))) & 3) + 1;
        u32 v = 0;
        for (int b = 0; b < len; ++b) v |= (u32)data[b] << (8 * b);
        data += len;
        out[i] = v;
    }
    return (size_t)(data - in);
}

// ---------------------------------------------------------------------------------------------------------------
// MultiSetVector list coding (src/slice_vector/set_vector.rs)
// ---------------------------------------------------------------------------------------------------------------
constexpr size_t MIN_NUMBERS_TO_ENCODE = 4;  // set_vector.rs:12

// set_vector.rs:117-148
void set_encode(std::vector<u32> data, std::vector<u8>& encoded) {
    if (data.size() >= 255) data.resize(255, 0);
    for (size_t i = data.size(); i-- > 1;) data[i] -= data[i - 1];  // delta_encode :151-155
    size_t count = data.size();
    if (data.size() < MIN_NUMBERS_TO_ENCODE) data.resize(MIN_NUMBERS_TO_ENCODE, 0);
    std::vector<u8> enc;
    svb_encode(data.data(), data.size(), enc);
    if (enc.size() >= sizeof(u32) * count) {  // only use compression if it makes the data smaller
        enc.clear();
        for (size_t i = 0; i < count; ++i)
            for (int b = 0; b < 4; ++b) enc.push_back((u8)(data[i] >> (8 * b)));
    }
    encoded.clear();
    encoded.push_back((u8)count);
    encoded.insert(encoded.end(), enc.begin(), enc.end());
}

// set_vector.rs:91-115
void set_decode(const u8* enc, size_t len, std::vector<u32>& out) {
    size_t count = enc[0];
    out.clear();
    const u8* data = enc + 1;
    size_t dlen = len - 1;
    if (dlen != count * sizeof(u32)) {
        out.resize(std::max(MIN_NUMBERS_TO_ENCODE, count), 0);
        svb_decode(data, out.size(), out.data());
        out.resize(count, 0);
    } else {
        for (size_t i = 0; i < count; ++i) out.push_back((u32)read_uint_le(data + 4 * i, 4));
    }
    for (size_t i = 1; i < out.size(); ++i) out[i] += out[i - 1];  // delta_decode :158-162
}

// ---------------------------------------------------------------------------------------------------------------
// Offsets / Chunk (src/slice_vector/offsets.rs:148-296) and the compressed layer blob
// ---------------------------------------------------------------------------------------------------------------
constexpr size_t OFFSETS_PER_CHUNK = 60;  // offsets.rs:7
constexpr size_t CHUNK_BYTES = 128;       // repr(C) { usize initial; u16 deltas[60] }
constexpr uint16_t DELTA_UNUSED = 0xFFFF;

struct CompressedLayer {  // MultiSetVector over a borrowed byte range
    const u8* chunks = nullptr;
    size_t num_chunks = 0;
    const u8* data = nullptr;
    size_t data_len = 0;
    size_t n = 0;  // number of lists

    static u64 chunk_initial(const u8* c) { return read_uint_le(c, 8); }
    static uint16_t chunk_delta(const u8* c, size_t i) { return (uint16_t)read_uint_le(c + 8 + 2 * i, 2); }

    // offsets.rs:171-176 (Chunk::get)
    static u64 chunk_get(const u8* c, size_t index) {
        u64 res = 0;
        for (size_t i = 0; i <= index; ++i) res += chunk_delta(c, i);
        return res + chunk_initial(c);
    }
    u64 offset_get(size_t index) const {  // offsets.rs:245-247
        return chunk_get(chunks + (index / OFFSETS_PER_CHUNK) * CHUNK_BYTES, index % OFFSETS_PER_CHUNK);
    }
    // offsets.rs:249-259
    void get_consecutive(size_t index, u64* b, u64* e) const {
        if ((index + 1) % OFFSETS_PER_CHUNK == 0) {
            *b = offset_get(index);
            *e = offset_get(index + 1);
        } else {
            const u8* c = chunks + (index / OFFSETS_PER_CHUNK) * CHUNK_BYTES;
            *b = chunk_get(c, index % OFFSETS_PER_CHUNK);
            *e = *b + chunk_delta(c, index % OFFSETS_PER_CHUNK + 1);
        }
    }
    // offsets.rs:267-270 (Offsets::len) minus one (offsets.rs:63-67)
    static size_t count_lists(const u8* chunks, size_t num_chunks) {
        if (num_chunks == 0) return 0;
        const u8* last = chunks + (num_chunks - 1) * CHUNK_BYTES;
        size_t l = 0;
        while (l < OFFSETS_PER_CHUNK && chunk_delta(last, l) != DELTA_UNUSED) ++l;
        size_t offsets_len = OFFSETS_PER_CHUNK * (num_chunks - 1) + l;
        return offsets_len == 0 ? 0 : offsets_len - 1;
    }
    // offsets.rs:127-139 (load_mmap)
    bool load(const u8* blob, size_t len) {
        if (len < 8) return false;
        u64 nb = read_uint_le(blob, 8);
        if (8 + nb > len || nb % CHUNK_BYTES != 0) return false;
        chunks = blob + 8;
        num_chunks = nb / CHUNK_BYTES;
        data = blob + 8 + nb;
        data_len = len - 8 - nb;
        n = count_lists(chunks, num_chunks);
        return true;
    }
    // set_vector.rs:57-69 — allocates per call like the reference
    void get(size_t idx, std::vector<u32>& out) const {
        u64 b, e;
        get_consecutive(idx, &b, &e);
        set_decode(data + b, (size_t)(e - b), out);
    }
};

// write_as_multi_set_vector (set_vector.rs:169-221) + Offsets::push (offsets.rs:233-241)
// Offsets::new / push (offsets.rs:225-241) over Chunk::new / push (offsets.rs:158-204): chunks of 60 u16 deltas with
// a u64 `initial`; unused deltas are 0xFFFF; the first chunk starts with initial = 0.  `ok` turns false where the
// reference panics (offset below the previous one, offsets.rs:201; delta above u16::MAX, offsets.rs:203).
struct OffsetsWriter {
    std::vector<u8> chunks;
    size_t cur_len = 0;
    u64 last_offset = 0;  // Chunk::last() of the current chunk, or its `initial` while it is empty
    bool ok = true;

    OffsetsWriter() { new_chunk(0); }
    void new_chunk(u64 initial) {
        chunks.resize(chunks.size() + CHUNK_BYTES, 0xFF);
        write_uint_le(&chunks[chunks.size() - CHUNK_BYTES], initial, 8);
        cur_len = 0;
        last_offset = initial;
    }
    void push(u64 offset) {
        if (cur_len == OFFSETS_PER_CHUNK) new_chunk(offset);  // is_full -> Chunk::new(offset), then push(offset)
        if (offset < last_offset) {
            ok = false;
            return;
        }
        const u64 delta = offset - last_offset;
        if (delta > 0xFFFF) {
            ok = false;
            return;
        }
        write_uint_le(&chunks[chunks.size() - CHUNK_BYTES + 8 + 2 * cur_len], delta, 2);
        ++cur_len;
        last_offset = offset;
    }
};

void write_layer_blob(const std::vector<std::vector<u32>>& lists, std::vector<u8>& out) {
    size_t n = lists.size();
    size_t bytes_for_offsets = (1 + n / OFFSETS_PER_CHUNK) * CHUNK_BYTES;
    size_t base = out.size();
    out.resize(base + 8 + bytes_for_offsets, 0);
    write_uint_le(&out[base], bytes_for_offsets, 8);
    OffsetsWriter offsets;
    offsets.push(0);
    std::vector<u8> enc;
    u64 total = 0;
    for (size_t i = 0; i < n; ++i) {
        std::vector<u32> s = lists[i];
        std::sort(s.begin(), s.end());
        set_encode(s, enc);
        out.insert(out.end(), enc.begin(), enc.end());
        total += enc.size();
        offsets.push(total);
    }
    if (!offsets.ok || offsets.chunks.size() != bytes_for_offsets) {
        std::fprintf(stderr, "oracle: offsets do not fit (delta too large or chunk count mismatch)\n");
        std::abort();
    }
    std::memcpy(&out[base + 8], offsets.chunks.data(), bytes_for_offsets);
}

// ---------------------------------------------------------------------------------------------------------------
// index file (src/index/io.rs)
// ---------------------------------------------------------------------------------------------------------------
constexpr size_t METADATA_LEN = 1024;  // io.rs:7

// Minimal JSON: find `"key"` and parse the integer array / integer after the colon (serde_json parse in io.rs:89-113).
bool json_find(const std::string& s, const char* key, size_t* pos) {
    std::string k = std::string("\"") + key + "\"";
    size_t p = s.find(k);
    if (p == std::string::npos) return false;
    p = s.find(':', p + k.size());
    if (p == std::string::npos) return false;
    *pos = p + 1;
    return true;
}
bool json_int_array(const std::string& s, const char* key, std::vector<u64>& out) {
    size_t p;
    if (!json_find(s, key, &p)) return false;
    while (p < s.size() && std::isspace((unsigned char)s[p])) ++p;
    if (p >= s.size() || s[p] != '[') return false;
    ++p;
    out.clear();
    while (p < s.size()) {
        while (p < s.size() && (std::isspace((unsigned char)s[p]) || s[p] == ',')) ++p;
        if (p < s.size() && s[p] == ']') return true;
        if (p >= s.size() || !std::isdigit((unsigned char)s[p])) return false;
        u64 v = 0;
        while (p < s.size() && std::isdigit((unsigned char)s[p])) v = v * 10 + (u64)(s[p++] - '0');
        out.push_back(v);
    }
    return false;
}

struct Index {
    // Either compressed (borrowing `bytes`) or fixed-width rows (builder output / "strong" CPU variant).
    std::vector<u8> bytes;
    std::vector<CompressedLayer> compressed;
    // fixed-width representation: layers[l] = rows of width `width`, UNUSED padded (index/mod.rs:540-552)
    std::vector<std::vector<u32>> fixed;
    size_t width = 0;
    bool use_fixed = false;

    size_t num_layers() const { return use_fixed ? fixed.size() : compressed.size(); }
    size_t layer_len(size_t l) const { return use_fixed ? (width ? fixed[l].size() / width : 0) : compressed[l].n; }
    size_t len() const { return num_layers() ? layer_len(num_layers() - 1) : 0; }

    void get_neighbors(size_t layer, size_t idx, std::vector<u32>& out) const {
        if (use_fixed) {
            out.clear();
            const u32* row = &fixed[layer][idx * width];
            for (size_t i = 0; i < width && row[i] != UNUSED; ++i) out.push_back(row[i]);
        } else {
            compressed[layer].get(idx, out);
        }
    }
};

// io.rs:72-113 (load_layers / read_layer_sizes)
bool load_index_bytes(Index* ix, const u8* buf, size_t len, std::string* err) {
    if (len < METADATA_LEN || std::memcmp(buf, "granne", 6) != 0) {
        *err = "Library string missing";
        return false;
    }
    ix->bytes.assign(buf, buf + len);
    std::string meta((const char*)ix->bytes.data() + 6, METADATA_LEN - 6);
    std::vector<u64> layer_sizes, layer_counts;
    if (!json_int_array(meta, "layer_sizes", layer_sizes) || !json_int_array(meta, "layer_counts", layer_counts)) {
        *err = "Could not read metadata";
        return false;
    }
    if (layer_sizes.size() != layer_counts.size()) {
        *err = "num_layers mismatch";
        return false;
    }
    size_t start = METADATA_LEN;
    ix->compressed.clear();
    for (u64 sz : layer_sizes) {
        if (start + sz > len) {
            *err = "layer exceeds file";
            return false;
        }
        CompressedLayer L;
        if (!L.load(ix->bytes.data() + start, (size_t)sz)) {
            *err = "bad layer blob";
            return false;
        }
        ix->compressed.push_back(L);
        start += sz;
    }
    ix->use_fixed = false;
    return true;
}

// io.rs:11-70 (write_index); serde_json Map is a BTreeMap by default -> keys in alphabetical order.
void write_index_bytes(const Index& ix, std::vector<u8>& out) {
    out.assign(METADATA_LEN, (u8)' ');
    std::vector<u64> layer_counts, layer_sizes;
    size_t nl = ix.num_layers();
    std::vector<u32> tmp;
    size_t num_neighbors = 0;
    if (nl > 0 && ix.layer_len(nl - 1) > 0) {
        ix.get_neighbors(nl - 1, 0, tmp);
        num_neighbors = tmp.size();  // io.rs:20-24: degree of node 0 in the last layer
    }
    for (size_t l = 0; l < nl; ++l) {
        size_t n = ix.layer_len(l);
        layer_counts.push_back(n);
        std::vector<std::vector<u32>> lists(n);
        for (size_t i = 0; i < n; ++i) ix.get_neighbors(l, i, lists[i]);
        size_t before = out.size();
        write_layer_blob(lists, out);
        layer_sizes.push_back(out.size() - before);
    }
    auto arr = [](const std::vector<u64>& v) {
        std::string s = "[";
        for (size_t i = 0; i < v.size(); ++i) {
            if (i) s += ",";
            s += std::to_string(v[i]);
        }
        return s + "]";
    };
    std::string meta = "granne";
    meta += "{\"compressed\":true,\"granne_version\":\"0.5.2\",\"layer_counts\":" + arr(layer_counts) +
            ",\"layer_sizes\":" + arr(layer_sizes) +
            ",\"num_elements\":" + std::to_string(layer_counts.empty() ? 0 : layer_counts.back()) +
            ",\"num_layers\":" + std::to_string(nl) + ",\"num_neighbors\":" + std::to_string(num_neighbors) +
            ",\"version\":2}";
    if (meta.size() > METADATA_LEN) {
        std::fprintf(stderr, "oracle: metadata too long\n");
        std::abort();
    }
    std::memcpy(out.data(), meta.data(), meta.size());
}

// ---------------------------------------------------------------------------------------------------------------
// search (src/index/mod.rs:962-1037, src/max_size_heap.rs)
// ---------------------------------------------------------------------------------------------------------------
struct SearchStats {
    u64 n_dist = 0;      // dist_to_element calls (index/mod.rs:1012,1027)
    u64 n_expand = 0;    // get_neighbors calls (:1025)
    u64 n_nbr_read = 0;  // total neighbour ids returned by those calls
};

using DI = std::pair<float, u64>;  // (NotNan<f32>, usize) — lexicographic order

// FxHashSet<usize> stand-in: open addressing with the Fx multiplicative hash (fxhash 0.2); set semantics only.
struct VisitedSet {
    std::vector<u64> slots;
    size_t mask = 0, count = 0;
    explicit VisitedSet(size_t cap) {
        size_t n = 16;
        while (n < cap * 2) n <<= 1;
        slots.assign(n, ~0ull);
        mask = n - 1;
    }
    void grow() {
        std::vector<u64> old;
        old.swap(slots);
        slots.assign(old.size() * 2, ~0ull);
        mask = slots.size() - 1;
        count = 0;
        for (u64 v : old)
            if (v != ~0ull) insert(v);
    }
    bool insert(u64 v) {  // true if newly inserted
        if ((count + 1) * 2 > slots.size()) grow();
        size_t h = (size_t)((v * 0x517cc1b727220a95ull) >> 20) & mask;
        while (slots[h] != ~0ull) {
            if (slots[h] == v) return false;
            h = (h + 1) & mask;
        }
        slots[h] = v;
        ++count;
        return true;
    }
};

// src/index/mod.rs:999-1037.  GetNeighbors: void(size_t idx, std::vector<u32>& out)
template <class GetNeighbors>
std::vector<std::pair<u64, float>> search_for_neighbors(GetNeighbors&& get_neighbors, u64 entrypoint,
                                                        const Elements& elements, const Query& goal,
                                                        size_t max_search, SearchStats* st) {
    std::priority_queue<DI> res;                                        // MaxSizeHeap (max_size_heap.rs:5-45)
    std::priority_queue<DI, std::vector<DI>, std::greater<DI>> pq;      // BinaryHeap<Reverse<_>>
    VisitedSet visited(max_search * 20);                                // :1009-1010
    auto res_full = [&] { return res.size() >= max_search; };

    float distance = elements.dist_to_element(entrypoint, goal);       // :1012
    if (st) st->n_dist++;
    pq.push(DI(distance, entrypoint));
    visited.insert(entrypoint);

    std::vector<u32> nbrs;
    while (!pq.empty()) {
        DI top = pq.top();
        pq.pop();
        float d = top.first;
        u64 idx = top.second;
        if (res_full() && d > res.top().first) break;                  // :1019-1021
        // MaxSizeHeap::push (max_size_heap.rs:18-32)
        if (!res_full()) {
            res.push(top);
        } else if (top < res.top()) {
            res.pop();
            res.push(top);
        }
        get_neighbors((size_t)idx, nbrs);                               // :1025
        if (st) {
            st->n_expand++;
            st->n_nbr_read += nbrs.size();
        }
        for (u32 nb : nbrs) {
            if (visited.insert(nb)) {
                float dn = elements.dist_to_element(nb, goal);         // :1027
                if (st) st->n_dist++;
                if (!res_full() || dn < res.top().first) pq.push(DI(dn, nb));  // :1029-1031
            }
        }
    }
    std::vector<DI> sorted;                                             // into_sorted_vec :1036
    sorted.reserve(res.size());
    while (!res.empty()) {
        sorted.push_back(res.top());
        res.pop();
    }
    std::reverse(sorted.begin(), sorted.end());
    std::vector<std::pair<u64, float>> out;
    out.reserve(sorted.size());
    for (auto& e : sorted) out.emplace_back(e.second, e.first);
    return out;
}

// src/index/mod.rs:963-997 (search_internal + find_entrypoint) over layers [0, num_layers) of `ix`
std::vector<std::pair<u64, float>> index_search(const Index& ix, size_t num_layers, const Elements& elements,
                                                const Query& q, size_t max_search, size_t num_neighbors,
                                                SearchStats* st) {
    std::vector<std::pair<u64, float>> out;
    if (num_layers == 0) return out;
    u64 entrypoint = 0;
    for (size_t l = 0; l + 1 < num_layers; ++l) {
        auto res = search_for_neighbors([&](size_t i, std::vector<u32>& o) { ix.get_neighbors(l, i, o); },
                                        entrypoint, elements, q, 1, st);
        entrypoint = res[0].first;
    }
    out = search_for_neighbors([&](size_t i, std::vector<u32>& o) { ix.get_neighbors(num_layers - 1, i, o); },
                               entrypoint, elements, q, max_search, st);
    if (out.size() > num_neighbors) out.resize(num_neighbors);
    return out;
}

// ---------------------------------------------------------------------------------------------------------------
// reorder (src/index/reorder.rs:59-292, src/slice_vector/mod.rs:437-458, src/elements/embeddings/mod.rs:191-217,
// src/elements/embeddings/reorder.rs:31-58)
// ---------------------------------------------------------------------------------------------------------------
constexpr size_t TRAIL_LAYERS = 8;  // reorder.rs:177
using Trail = std::array<u32, TRAIL_LAYERS>;

// reorder.rs:180-207 (find_entrypoint_trail): the closest element (max_search = 1) in each of the first
// min(8, max_layer) layers.  The reference seeds layer i with `eps[i]`, which is still 0 at that point, so every layer
// is searched from node 0 (not from the previous layer's result); this restatement keeps that behaviour.
Trail find_entrypoint_trail(const Index& ix, const Elements& el, size_t max_layer, const Query& q) {
    Trail eps{};
    const size_t take = std::min<size_t>(std::min(TRAIL_LAYERS, max_layer), ix.num_layers());
    for (size_t i = 0; i < take; ++i) {
        const u64 ep = (i == 0) ? 0 : eps[i];
        auto res = search_for_neighbors([&](size_t n, std::vector<u32>& o) { ix.get_neighbors(i, n, o); }, ep, el, q,
                                        1, nullptr);
        eps[i] = (u32)res[0].first;
    }
    return eps;
}

// reorder.rs:126-174 (compute_order).  `order_inv` is only filled for ids >= layer_len(0) (reorder.rs:161-165); ids of
// the first layer map to 0, as in the reference.  (trail, idx) tuples are unique, so the unstable sort is deterministic.
std::vector<u64> compute_order(const Index& ix, const Elements& el, int threads) {
    const size_t nl = ix.num_layers();
    std::vector<u64> order;
    if (nl == 0) return order;
    for (size_t i = 0; i < ix.layer_len(0); ++i) order.push_back(i);
    std::vector<u64> order_inv(nl >= 2 ? ix.layer_len(nl - 2) : 0, 0);
    for (size_t layer = 1; layer < nl; ++layer) {
        const size_t begin = ix.layer_len(layer - 1), end = ix.layer_len(layer);
        std::vector<std::pair<Trail, u64>> eps(end - begin);
        auto run = [&](size_t b, size_t e) {
            Query q;
            for (size_t idx = b; idx < e; ++idx) {
                el.get(idx, &q);
                Trail t = find_entrypoint_trail(ix, el, layer, q);
                for (auto& v : t) v = (u32)order_inv[v];
                eps[idx - begin] = {t, idx};
            }
        };
        if (threads <= 1 || end - begin < 64) {
            run(begin, end);
        } else {
            std::vector<std::thread> ts;
            const size_t per = (end - begin + threads - 1) / threads;
            for (int t = 0; t < threads; ++t) {
                const size_t b = std::min(end, begin + per * t), e = std::min(end, begin + per * (t + 1));
                if (b < e) ts.emplace_back(run, b, e);
            }
            for (auto& t : ts) t.join();
        }
        std::sort(eps.begin(), eps.end());
        for (auto& e : eps) order.push_back(e.second);
        if (layer < nl - 1)
            for (size_t i = begin; i < end; ++i) order_inv[order[i]] = i;
    }
    return order;
}

// reorder.rs:89-124 (reorder_by_keys, the ordering part): a layer-preserving sort by (key, idx); keys are rows of
// `kw` u64 compared lexicographically (covers integer keys and the [usize; 8] keys of compute_keys_for_reordering).
std::vector<u64> order_by_keys(const Index& ix, const u64* keys, size_t kw) {
    std::vector<u64> order;
    for (size_t layer = 0; layer < ix.num_layers(); ++layer) {
        const size_t begin = layer ? ix.layer_len(layer - 1) : 0, end = ix.layer_len(layer);
        std::vector<u64> ids;
        for (size_t i = begin; i < end; ++i) ids.push_back(i);
        std::sort(ids.begin(), ids.end(), [&](u64 a, u64 b) {
            for (size_t j = 0; j < kw; ++j)
                if (keys[a * kw + j] != keys[b * kw + j]) return keys[a * kw + j] < keys[b * kw + j];
            return a < b;
        });
        order.insert(order.end(), ids.begin(), ids.end());
    }
    return order;
}

// reorder.rs:209-292 (reorder_layers / reorder_layer / get_reverse_mapping): node i of the new layer gets the
// neighbours of old node mapping[i], renamed through the reverse mapping; MultiSetVector::push sorts each list
// (set_vector.rs:41-47).  The result is returned as fixed-width rows (sorted), ready for write_index_bytes.
void reorder_layers(const Index& ix, const std::vector<u64>& mapping, Index* out) {
    std::vector<u64> rev(mapping.size(), 0);
    for (size_t i = 0; i < mapping.size(); ++i) rev[mapping[i]] = i;
    std::vector<std::vector<std::vector<u32>>> lists(ix.num_layers());
    size_t w = 1;
    std::vector<u32> tmp;
    for (size_t l = 0; l < ix.num_layers(); ++l) {
        lists[l].resize(ix.layer_len(l));
        for (size_t i = 0; i < ix.layer_len(l); ++i) {
            ix.get_neighbors(l, (size_t)mapping[i], tmp);
            for (u32& n : tmp) n = (u32)rev[n];
            std::sort(tmp.begin(), tmp.end());
            w = std::max(w, tmp.size());
            lists[l][i] = tmp;
        }
    }
    out->use_fixed = true;
    out->width = w;
    out->fixed.clear();
    for (size_t l = 0; l < ix.num_layers(); ++l) {
        std::vector<u32> rows(lists[l].size() * w, UNUSED);
        for (size_t i = 0; i < lists[l].size(); ++i) std::copy(lists[l][i].begin(), lists[l][i].end(), rows.begin() + i * w);
        out->fixed.push_back(std::move(rows));
    }
}

// Permutable::permute — FixedWidthSliceVector (slice_vector/mod.rs:437-458) and SumEmbeddings
// (embeddings/mod.rs:191-217): new element i = old element permutation[i].
void permute_elements(Elements* el, const std::vector<u64>& perm) {
    const size_t n = el->n, dim = el->dim;
    if (el->kind == KIND_F32) {
        std::vector<float> r(el->f32.size());
        for (size_t i = 0; i < n; ++i) std::memcpy(&r[i * dim], &el->f32[(size_t)perm[i] * dim], dim * sizeof(float));
        el->f32.swap(r);
    } else if (el->kind == KIND_I8) {
        std::vector<int8_t> r(el->i8.size());
        for (size_t i = 0; i < n; ++i) std::memcpy(&r[i * dim], &el->i8[(size_t)perm[i] * dim], dim);
        el->i8.swap(r);
    } else {
        std::vector<u64> off(1, 0);
        std::vector<u32> terms;
        for (size_t i = 0; i < n; ++i) {
            for (u64 t = el->offsets[perm[i]]; t < el->offsets[perm[i] + 1]; ++t) terms.push_back(el->terms[t]);
            off.push_back(terms.size());
        }
        el->offsets.swap(off);
        el->terms.swap(terms);
    }
}

// embeddings/reorder.rs:31-58 (compute_keys_for_reordering): per element, its embedding ids ordered by decreasing
// norm (stable sort by norm, then reversed), first 8, zero padded.  The norm is a plain left-to-right f32 sum of
// squares (`iter().map(|x| x * x).sum::<f32>().sqrt()`), not the 32-lane dot product.
void embedding_reorder_keys(const Elements& el, u64* keys) {
    std::vector<float> norms(el.num_embeddings);
    for (size_t w = 0; w < el.num_embeddings; ++w) {
        float acc = 0.0f;
        for (size_t j = 0; j < el.dim; ++j) {
            const float x = el.f32[w * el.dim + j];
            acc = acc + x * x;
        }
        norms[w] = std::sqrt(acc);
    }
    for (size_t q = 0; q < el.n; ++q) {
        std::vector<u32> ids(el.terms.begin() + el.offsets[q], el.terms.begin() + el.offsets[q + 1]);
        std::stable_sort(ids.begin(), ids.end(), [&](u32 a, u32 b) { return norms[a] < norms[b]; });
        std::reverse(ids.begin(), ids.end());
        for (size_t j = 0; j < TRAIL_LAYERS; ++j) keys[q * TRAIL_LAYERS + j] = j < ids.size() ? ids[j] : 0;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// builder (src/index/mod.rs:198-231, 366-402, 634-960) — fixture generator.
// threads == 1 restates the `singlethreaded` feature order (:771-772,789-790); threads > 1 mirrors the rayon
// par_iter build (:773-774) with per-node locks (nondeterministic, like the reference).
// Deviation: add_and_limit_neighbors uses sort_unstable_by_key on distance only (:945); ties are ordered here by a
// stable sort, the reference's pdqsort tie order is implementation-defined.
// ---------------------------------------------------------------------------------------------------------------
struct BuildConfig {  // index/mod.rs:198-231
    float layer_multiplier = 15.0f;
    long expected_num_elements = -1;
    size_t num_neighbors = 30;
    size_t max_search = 200;
    bool reinsert_elements = true;
};

// index/mod.rs:634-643
size_t compute_num_elements_in_layer(size_t total, float layer_multiplier, size_t layer_idx) {
    double m = (double)layer_multiplier;
    double expo = std::floor(std::log((double)total) / std::log(m)) - (double)layer_idx;
    // f64::log(self, base) = ln(self)/ln(base)
    double v = std::ceil((double)total / std::pow(m, expo));
    size_t r = v < 0 ? 0 : (v > 1.8e19 ? (size_t)-1 : (size_t)v);
    return std::min(r, total);
}

struct SpinLocks {
    std::unique_ptr<std::atomic<u8>[]> l;
    bool enabled = false;
    void init(size_t n, bool en) {
        enabled = en;
        if (en) {
            l.reset(new std::atomic<u8>[n]);
            for (size_t i = 0; i < n; ++i) l[i].store(0, std::memory_order_relaxed);
        }
    }
    void lock(size_t i) {
        if (!enabled) return;
        u8 exp = 0;
        while (!l[i].compare_exchange_weak(exp, 1, std::memory_order_acquire)) {
            exp = 0;
        }
    }
    void unlock(size_t i) {
        if (enabled) l[i].store(0, std::memory_order_release);
    }
};

// What the batched model (Builder::index_batches) did: the conditions under which its image is order-independent, and
// evidence that a case really exercises batches, overflowing connects and contended rows.
struct BuildCounters {
    std::atomic<u64> batches{0};
    std::atomic<u64> max_batch{0};
    std::atomic<u64> connect_present{0};     // connect_nodes found j already in the row
    std::atomic<u64> connect_overflow{0};    // connect_nodes found the row full and went to add_and_limit_neighbors
    std::atomic<u64> nontrivial_selects{0};  // select_neighbors with more candidates than its limit (link or prune)
    std::atomic<u64> max_batch_in_links{0};  // most reverse links one node received within one batch
};

struct Builder {
    const Elements* elements;
    BuildConfig config;
    Index ix;  // fixed-width layers, width = config.num_neighbors (index/mod.rs:394)
    size_t max_batch = 0;               // > 0: the product's batch schedule (index_batches) instead of the reference's
    BuildCounters* counters = nullptr;  // set together with max_batch

    using Cand = std::pair<u64, float>;

    // index/mod.rs:849-883
    std::vector<Cand> select_neighbors(std::vector<Cand> candidates, size_t max_neighbors) const {
        if (candidates.size() <= max_neighbors) return candidates;
        if (counters) counters->nontrivial_selects.fetch_add(1, std::memory_order_relaxed);
        std::vector<Cand> neighbors;
        Query e;
        for (auto& c : candidates) {
            if (neighbors.size() >= max_neighbors) break;
            elements->get(c.first, &e);
            bool ok = true;
            for (auto& n : neighbors) {
                if (!(c.second <= elements->dist_to_element(n.first, e))) {
                    ok = false;
                    break;
                }
            }
            if (ok) neighbors.push_back(c);
        }
        return neighbors;
    }

    // index/mod.rs:923-959 (node = row pointer of width `w`)
    void add_and_limit_neighbors(u32* node, size_t w, size_t node_id, const Cand* extra, size_t n_extra,
                                 size_t num_neighbors) const {
        std::vector<Cand> cands;
        Query e;
        elements->get(node_id, &e);
        for (size_t i = 0; i < w && node[i] != UNUSED; ++i)
            cands.emplace_back(node[i], elements->dist_to_element(node[i], e));  // elements.dists :938
        for (size_t i = 0; i < n_extra; ++i) cands.push_back(extra[i]);
        std::stable_sort(cands.begin(), cands.end(), [](const Cand& a, const Cand& b) { return a.second < b.second; });
        auto nb = select_neighbors(cands, num_neighbors);
        for (size_t k = 0; k < w; ++k) node[k] = k < nb.size() ? (u32)nb[k].first : UNUSED;
    }

    // index/mod.rs:899-921
    void connect_nodes(u32* node, size_t w, size_t i, size_t j, float d, SpinLocks& locks) const {
        if (i == j) return;
        locks.lock(i);
        size_t free_pos = w;
        for (size_t k = 0; k < w; ++k)
            if (node[k] == UNUSED || node[k] == (u32)j) {
                free_pos = k;
                break;
            }
        if (free_pos < w) {
            if (counters && node[free_pos] == (u32)j) counters->connect_present.fetch_add(1, std::memory_order_relaxed);
            node[free_pos] = (u32)j;
        } else {
            if (counters) counters->connect_overflow.fetch_add(1, std::memory_order_relaxed);
            Cand ex(j, d);
            add_and_limit_neighbors(node, w, i, &ex, 1, w);
        }
        locks.unlock(i);
    }

    // index_element (index/mod.rs:805-846) in two halves: the search half only reads the layer, the link half writes it.
    // The sequential / threaded build runs them back to back; build_batched runs the search halves of a whole batch
    // against one snapshot of the layer and then the link halves in batch order.
    static constexpr float EPS100 = 100.0f * 1.1920929e-07f;  // NotNan::new(100.0 * f32::EPSILON) (:813,829)

    bool is_zero(size_t idx) const { return elements->dist(idx, idx) > EPS100; }  // :812-815

    // :816-822: candidates = search_for_neighbors(layer, prev_layers.search(e,1,1), e, max_search) without idx itself
    std::vector<Cand> search_element(const BuildConfig& cfg, size_t num_prev_layers, const std::vector<u32>& layer,
                                     size_t idx, SpinLocks& locks) const {
        const size_t w = ix.width;
        Query element;
        elements->get(idx, &element);
        u64 entrypoint = 0;
        {
            auto r = index_search(ix, num_prev_layers, *elements, element, 1, 1, nullptr);  // prev_layers.search(e,1,1)
            if (!r.empty()) entrypoint = r[0].first;
        }
        auto getn = [&](size_t i, std::vector<u32>& o) {
            o.clear();
            locks.lock(i);
            const u32* row = &layer[i * w];
            for (size_t k = 0; k < w && row[k] != UNUSED; ++k) o.push_back(row[k]);
            locks.unlock(i);
        };
        auto found = search_for_neighbors(getn, entrypoint, *elements, element, cfg.max_search, nullptr);
        std::vector<Cand> candidates;
        for (auto& c : found)
            if (c.first != idx) candidates.push_back(c);
        return candidates;
    }

    // :824-845: select, the dead-duplicate rule, the own row (initialize_node or connect_nodes), the reverse links.
    // Returns the selected neighbours (empty when the element stays unconnected).
    std::vector<Cand> link_element(const BuildConfig& cfg, std::vector<u32>& layer, size_t idx,
                                   const std::vector<Cand>& candidates, SpinLocks& locks) const {
        const size_t w = ix.width;
        auto neighbors = select_neighbors(candidates, cfg.num_neighbors);
        if (neighbors.size() > cfg.num_neighbors / 2 && neighbors[cfg.num_neighbors / 2].second < EPS100) return {};
        locks.lock(idx);
        bool empty = layer[idx * w] == UNUSED;
        if (empty) {  // initialize_node :886-895
            for (size_t k = 0; k < neighbors.size() && k < w; ++k) layer[idx * w + k] = (u32)neighbors[k].first;
        }
        locks.unlock(idx);
        if (!empty)
            for (auto& n : neighbors) connect_nodes(&layer[idx * w], w, idx, n.first, n.second, locks);
        for (auto& n : neighbors) connect_nodes(&layer[n.first * w], w, n.first, idx, n.second, locks);
        return neighbors;
    }

    void index_element(const BuildConfig& cfg, size_t num_prev_layers, std::vector<u32>& layer, size_t idx,
                       SpinLocks& locks) const {
        if (is_zero(idx)) return;  // do not index zero elements
        link_element(cfg, layer, idx, search_element(cfg, num_prev_layers, layer, idx, locks), locks);
    }

    // NOT a reference behaviour: a restatement of the PRODUCT's batch schedule (builder_index_elements in
    // granne_b200/csrc/granne_b200.cu) with its link phase serialized, so that the GPU build can be checked exactly.
    // Per batch: bsz = min(max_batch, max(1, present / 16), remaining), present = the layer's length when reinserting,
    // else the nodes linked before the batch; ids ascend from `first` (insertion) or descend from the last node
    // (reinsertion).  Every member searches the layer as it was before the batch (in parallel: nothing is written
    // during that phase), then the members are linked one after another in batch order, like the product's link kernel
    // when its work counter hands out members to a single warp.
    void index_batches(const BuildConfig& cfg, size_t num_prev_layers, std::vector<u32>& layer, size_t first,
                       bool reinsert, int threads) const {
        const size_t nrows = layer.size() / ix.width;
        const size_t total = nrows - first;
        SpinLocks unlocked;  // the search phase only reads, the link phase is sequential
        std::vector<size_t> ids;
        std::vector<std::vector<Cand>> cands;
        std::unordered_map<size_t, u64> in_links;
        for (size_t pos = 0; pos < total;) {
            const size_t present = reinsert ? nrows : first + pos;
            const size_t bsz = std::min(std::min(max_batch, std::max<size_t>(1, present / 16)), total - pos);
            ids.resize(bsz);
            for (size_t k = 0; k < bsz; ++k) ids[k] = reinsert ? nrows - 1 - pos - k : first + pos + k;
            cands.assign(bsz, {});
            auto search = [&](size_t b, size_t e) {
                for (size_t k = b; k < e; ++k)
                    if (!is_zero(ids[k])) cands[k] = search_element(cfg, num_prev_layers, layer, ids[k], unlocked);
            };
            const size_t nt = std::min<size_t>(std::max(threads, 1), bsz / 16 + 1);
            if (nt <= 1) {
                search(0, bsz);
            } else {
                std::vector<std::thread> ts;
                const size_t per = (bsz + nt - 1) / nt;
                for (size_t t = 0; t < nt; ++t) ts.emplace_back(search, std::min(bsz, per * t), std::min(bsz, per * (t + 1)));
                for (auto& t : ts) t.join();
            }
            in_links.clear();
            for (size_t k = 0; k < bsz; ++k) {
                if (is_zero(ids[k])) continue;  // do not index zero elements
                for (auto& n : link_element(cfg, layer, ids[k], cands[k], unlocked)) {
                    const u64 c = ++in_links[n.first];
                    if (c > counters->max_batch_in_links) counters->max_batch_in_links = c;
                }
            }
            counters->batches += 1;
            if (bsz > counters->max_batch) counters->max_batch = bsz;
            pos += bsz;
        }
    }

    // index/mod.rs:716-802
    void index_elements(const BuildConfig& cfg, size_t num_elements, size_t num_prev_layers, std::vector<u32>& layer,
                        bool reinsert, int threads) const {
        const size_t w = ix.width;
        size_t already = layer.size() / w;
        if (reinsert)
            already = 0;
        else
            layer.resize(num_elements * w, UNUSED);
        size_t nrows = layer.size() / w;
        SpinLocks locks;
        locks.init(nrows, threads > 1 && max_batch == 0);
        if (max_batch > 0) {
            index_batches(cfg, num_prev_layers, layer, reinsert ? 0 : already, reinsert, threads);
        } else if (threads <= 1) {
            if (reinsert)
                for (size_t i = nrows; i-- > 0;) index_element(cfg, num_prev_layers, layer, i, locks);
            else
                for (size_t i = already; i < nrows; ++i) index_element(cfg, num_prev_layers, layer, i, locks);
        } else {
            std::atomic<size_t> next(0);
            size_t total = reinsert ? nrows : nrows - already;
            auto work = [&] {
                for (;;) {
                    size_t k = next.fetch_add(64);
                    if (k >= total) break;
                    size_t kend = std::min(total, k + 64);
                    for (; k < kend; ++k) {
                        size_t i = reinsert ? nrows - 1 - k : already + k;
                        index_element(cfg, num_prev_layers, layer, i, locks);
                    }
                }
            };
            std::vector<std::thread> ts;
            for (int t = 0; t < threads; ++t) ts.emplace_back(work);
            for (auto& t : ts) t.join();
        }
        // limit number of neighbors (:794-797)
        auto prune = [&](size_t b, size_t e) {
            for (size_t i = b; i < e; ++i) add_and_limit_neighbors(&layer[i * w], w, i, nullptr, 0, cfg.num_neighbors);
        };
        if (threads <= 1) {
            prune(0, nrows);
        } else {
            std::vector<std::thread> ts;
            size_t per = (nrows + threads - 1) / threads;
            for (int t = 0; t < threads; ++t) {
                size_t b = std::min(nrows, per * t), e = std::min(nrows, per * (t + 1));
                ts.emplace_back(prune, b, e);
            }
            for (auto& t : ts) t.join();
        }
    }

    // index/mod.rs:646-713
    void index_elements_in_last_layer(size_t max_num_elements, int threads) {
        size_t total = config.expected_num_elements >= 0 ? (size_t)config.expected_num_elements : elements->len();
        size_t ideal = compute_num_elements_in_layer(std::max(total, elements->len()), config.layer_multiplier,
                                                     ix.fixed.size() - 1);
        size_t last_len = ix.fixed.back().size() / ix.width;
        if (ideal <= last_len) return;
        size_t num_in_layer = std::min(max_num_elements, ideal);
        BuildConfig cfg = config;
        if (ideal < total) cfg.num_neighbors = std::max<size_t>(1, cfg.num_neighbors / 2);
        std::vector<u32> layer;
        layer.swap(ix.fixed.back());
        ix.fixed.pop_back();
        size_t num_prev = ix.fixed.size();
        index_elements(cfg, num_in_layer, num_prev, layer, false, threads);
        if (config.reinsert_elements) {
            cfg.max_search = std::max<size_t>(1, cfg.max_search / 2);
            index_elements(cfg, num_in_layer, num_prev, layer, true, threads);
        }
        ix.fixed.push_back(std::move(layer));
    }

    // index/mod.rs:374-402
    void build_partial(size_t num_elements, int threads) {
        if (num_elements == 0) return;
        ix.use_fixed = true;
        ix.width = config.num_neighbors;
        if (!ix.fixed.empty()) index_elements_in_last_layer(num_elements, threads);
        while (ix.len() < num_elements) {
            if (ix.fixed.empty())
                ix.fixed.emplace_back();
            else
                ix.fixed.push_back(ix.fixed.back());
            index_elements_in_last_layer(num_elements, threads);
        }
    }
};

thread_local std::string g_err;

}  // namespace

// =================================================================================================================
// C API (ctypes) — oracle/granne_oracle.py wraps this.
// =================================================================================================================
extern "C" {

const char* orc_last_error() { return g_err.c_str(); }

// ---- KAT helpers ----
uint64_t orc_num_elements_in_layer(uint64_t total, float mult, uint64_t layer) {
    return compute_num_elements_in_layer(total, mult, layer);
}
float orc_dot_f32(const float* x, const float* y, uint64_t n) { return dot_product_f32(x, y, n); }
void orc_normalize_f32(float* x, uint64_t n) { normalize_f32(x, n); }
void orc_sum_into_f32(float* x, const float* y, uint64_t n) { sum_into_f32(x, y, n); }
float orc_dist_f32(const float* x, const float* y, uint64_t n) { return angular_dist_f32(x, y, n); }
float orc_dist_i8(const int8_t* x, const int8_t* y, uint64_t n) { return angular_dist_i8(x, y, n); }
void orc_quantize_i8(const float* x, uint64_t n, int8_t* out) { quantize_i8(x, n, out); }
void orc_dot_i8(const int8_t* x, const int8_t* y, uint64_t n, int32_t* out3) {
    dot_product_and_squared_norms_i8(x, y, n, out3, out3 + 1, out3 + 2);
}
uint64_t orc_read_uint(const uint8_t* p, int nbytes) { return read_uint_le(p, nbytes); }
void orc_write_uint(uint8_t* p, uint64_t v, int nbytes) { write_uint_le(p, v, nbytes); }
// set_encode: returns encoded length (cap must be >= 1 + 5*max(4,n))
uint64_t orc_set_encode(const uint32_t* sorted, uint64_t n, uint8_t* out, uint64_t cap) {
    std::vector<u8> enc;
    set_encode(std::vector<u32>(sorted, sorted + n), enc);
    if (enc.size() > cap) return 0;
    std::memcpy(out, enc.data(), enc.size());
    return enc.size();
}
uint64_t orc_set_decode(const uint8_t* enc, uint64_t len, uint32_t* out, uint64_t cap) {
    std::vector<u32> v;
    set_decode(enc, len, v);
    if (v.size() > cap) return (uint64_t)-1;
    std::memcpy(out, v.data(), v.size() * 4);
    return v.size();
}
void orc_delta_encode(uint32_t* d, uint64_t n) {
    for (size_t i = n; i-- > 1;) d[i] -= d[i - 1];
}

// ---- elements ----
void* orc_elements_new(int kind, uint64_t dim) {
    auto* e = new Elements();
    e->kind = kind;
    e->dim = dim;
    if (kind == KIND_SUM) e->offsets.push_back(0);
    return e;
}
void orc_elements_free(void* p) { delete (Elements*)p; }
uint64_t orc_elements_len(void* p) { return ((Elements*)p)->n; }
uint64_t orc_elements_dim(void* p) { return ((Elements*)p)->dim; }

// push `n` raw f32 vectors: f32 -> normalised (Vector::from), i8 -> quantised.  `as_is`: store rows unmodified
// (== Vectors::from_vec of already-normalised data, dense_vector.rs:73-78).
void orc_elements_push_f32(void* p, const float* data, uint64_t n, int as_is) {
    auto* e = (Elements*)p;
    if (e->kind == KIND_F32) {
        size_t base = e->f32.size();
        e->f32.insert(e->f32.end(), data, data + n * e->dim);
        if (!as_is)
            for (size_t i = 0; i < n; ++i) normalize_f32(&e->f32[base + i * e->dim], e->dim);
        e->n += n;
    } else if (e->kind == KIND_I8) {
        size_t base = e->i8.size();
        e->i8.resize(base + n * e->dim);
        for (size_t i = 0; i < n; ++i) quantize_i8(data + i * e->dim, e->dim, &e->i8[base + i * e->dim]);
        e->n += n;
    }
}
void orc_elements_push_i8(void* p, const int8_t* data, uint64_t n) {
    auto* e = (Elements*)p;
    e->i8.insert(e->i8.end(), data, data + n * e->dim);
    e->n += n;
}
// SumEmbeddings: push_embedding (embeddings/mod.rs:101-103) and push element (:95-98)
void orc_sum_push_embeddings(void* p, const float* data, uint64_t n) {
    auto* e = (Elements*)p;
    e->f32.insert(e->f32.end(), data, data + n * e->dim);
    e->num_embeddings += n;
}
void orc_sum_push_element(void* p, const uint32_t* ids, uint64_t n) {
    auto* e = (Elements*)p;
    e->terms.insert(e->terms.end(), ids, ids + n);
    e->offsets.push_back(e->terms.size());
    e->n += 1;
}
// raw row access
uint64_t orc_sum_num_embeddings(void* p) { return ((Elements*)p)->num_embeddings; }
// SumEmbeddings::get_terms (embeddings/mod.rs:106-108)
uint64_t orc_sum_terms(void* p, uint64_t idx, uint32_t* out, uint64_t cap) {
    auto* e = (Elements*)p;
    const u64 b = e->offsets[idx], n = e->offsets[idx + 1] - b;
    for (u64 i = 0; i < n && i < cap; ++i) out[i] = e->terms[b + i];
    return n;
}
const void* orc_elements_data(void* p) {
    auto* e = (Elements*)p;
    return e->kind == KIND_I8 ? (const void*)e->i8.data() : (const void*)e->f32.data();
}
// ElementContainer::get as f32 (f32 kinds) or i8
void orc_elements_get(void* p, uint64_t idx, void* out) {
    auto* e = (Elements*)p;
    Query q;
    e->get(idx, &q);
    if (e->kind == KIND_I8)
        std::memcpy(out, q.q.data(), e->dim);
    else
        std::memcpy(out, q.f.data(), e->dim * 4);
}
float orc_elements_dist_to(void* p, uint64_t idx, const float* raw_query, int already_element) {
    auto* e = (Elements*)p;
    Query q;
    e->make_query(raw_query, already_element != 0, &q);
    return e->dist_to_element(idx, q);
}

// Serialise: FixedWidthSliceVector::write (slice_vector/mod.rs:460-466): u64 width + raw rows.
// which: 0 = the dense vectors (f32/i8) or the SumEmbeddings *elements* file; 1 = SumEmbeddings embeddings file.
uint64_t orc_elements_serialize(void* p, int which, uint8_t* out, uint64_t cap) {
    auto* e = (Elements*)p;
    std::vector<u8> b;
    auto put_u64 = [&](u64 v) {
        size_t o = b.size();
        b.resize(o + 8);
        write_uint_le(&b[o], v, 8);
    };
    if (e->kind == KIND_F32 || (e->kind == KIND_SUM && which == 1)) {
        put_u64(e->dim);
        size_t o = b.size();
        b.resize(o + e->f32.size() * 4);
        std::memcpy(&b[o], e->f32.data(), e->f32.size() * 4);
    } else if (e->kind == KIND_I8) {
        put_u64(e->dim);
        size_t o = b.size();
        b.resize(o + e->i8.size());
        std::memcpy(&b[o], e->i8.data(), e->i8.size());
    } else {
        // VariableWidthSliceVector<ThreeByteInt, FiveByteInt>::write (slice_vector/mod.rs:623-634)
        put_u64(e->n);
        for (u64 off : e->offsets) {
            size_t o = b.size();
            b.resize(o + 5);
            write_uint_le(&b[o], off, 5);
        }
        for (u32 t : e->terms) {
            size_t o = b.size();
            b.resize(o + 3);
            write_uint_le(&b[o], t, 3);
        }
    }
    if (out == nullptr) return b.size();
    if (b.size() > cap) return 0;
    std::memcpy(out, b.data(), b.size());
    return b.size();
}

// Load: Vectors::from_bytes (dense_vector.rs:50-52) / SumEmbeddings::from_bytes (embeddings/mod.rs:56-61)
void* orc_elements_from_bytes(int kind, const uint8_t* buf, uint64_t len, const uint8_t* emb, uint64_t emb_len) {
    auto* e = new Elements();
    e->kind = kind;
    if (kind == KIND_F32 || kind == KIND_I8) {
        if (len < 8) {
            g_err = "short elements buffer";
            delete e;
            return nullptr;
        }
        e->dim = read_uint_le(buf, 8);
        size_t esz = kind == KIND_F32 ? 4 : 1;
        if (e->dim == 0 || (len - 8) % (e->dim * esz) != 0) {
            g_err = "width > 0 && data.len() % width == 0 violated";
            delete e;
            return nullptr;
        }
        e->n = (len - 8) / (e->dim * esz);
        if (kind == KIND_F32) {
            e->f32.resize(e->n * e->dim);
            std::memcpy(e->f32.data(), buf + 8, len - 8);
        } else {
            e->i8.resize(e->n * e->dim);
            std::memcpy(e->i8.data(), buf + 8, len - 8);
        }
    } else {
        e->dim = read_uint_le(emb, 8);
        e->num_embeddings = (emb_len - 8) / (e->dim * 4);
        e->f32.resize(e->num_embeddings * e->dim);
        std::memcpy(e->f32.data(), emb + 8, e->f32.size() * 4);
        u64 ns = read_uint_le(buf, 8);
        e->n = ns;
        e->offsets.resize(ns + 1);
        for (u64 i = 0; i <= ns; ++i) e->offsets[i] = read_uint_le(buf + 8 + 5 * i, 5);
        size_t nterms = (len - 8 - 5 * (ns + 1)) / 3;
        e->terms.resize(nterms);
        const u8* d = buf + 8 + 5 * (ns + 1);
        for (size_t i = 0; i < nterms; ++i) e->terms[i] = (u32)read_uint_le(d + 3 * i, 3);
    }
    return e;
}

// ---- index ----
void orc_index_free(void* p) { delete (Index*)p; }

void* orc_index_from_bytes(const uint8_t* buf, uint64_t len) {
    auto* ix = new Index();
    std::string err;
    if (!load_index_bytes(ix, buf, len, &err)) {
        g_err = err;
        delete ix;
        return nullptr;
    }
    return ix;
}

// Builds with GranneBuilder semantics; returns an Index with fixed-width layers.
void* orc_build(void* elements, uint64_t num_neighbors, uint64_t max_search, float layer_multiplier, int reinsert,
                int64_t expected_num_elements, uint64_t num_elements, int threads) {
    Builder b;
    b.elements = (Elements*)elements;
    b.config.num_neighbors = num_neighbors;
    b.config.max_search = max_search;
    b.config.layer_multiplier = layer_multiplier;
    b.config.reinsert_elements = reinsert != 0;
    b.config.expected_num_elements = expected_num_elements;
    b.build_partial(num_elements ? num_elements : b.elements->len(), threads);
    auto* ix = new Index(std::move(b.ix));
    ix->use_fixed = true;
    return ix;
}

uint64_t orc_index_serialize(void* p, uint8_t* out, uint64_t cap) {
    std::vector<u8> b;
    write_index_bytes(*(Index*)p, b);
    if (out == nullptr) return b.size();
    if (b.size() > cap) return 0;
    std::memcpy(out, b.data(), b.size());
    return b.size();
}

// Decode compressed layers into fixed-width rows (the "strong" CPU variant; GranneBuilder::from_bytes :439-457).
void* orc_index_to_fixed(void* p) {
    auto* src = (Index*)p;
    auto* ix = new Index();
    ix->use_fixed = true;
    // decode every list once per pass, node ranges spread over the host threads (a 100M-node layer takes seconds)
    const unsigned hw = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    auto ranges = [&](size_t n, const std::function<void(size_t, size_t, unsigned)>& fn) {
        const unsigned t = (unsigned)std::max<size_t>(1, std::min<size_t>(hw, n / 4096));
        if (t == 1) {
            fn(0, n, 0);
            return;
        }
        std::vector<std::thread> ts;
        const size_t per = (n + t - 1) / t;
        for (unsigned w = 0; w < t; ++w)
            if (w * per < n) ts.emplace_back(fn, w * per, std::min(n, (w + 1) * per), w);
        for (auto& th : ts) th.join();
    };
    std::vector<size_t> wmax(hw, 1);
    for (size_t l = 0; l < src->num_layers(); ++l)
        ranges(src->layer_len(l), [&](size_t b, size_t e, unsigned w) {
            std::vector<u32> tmp;
            for (size_t i = b; i < e; ++i) {
                src->get_neighbors(l, i, tmp);
                wmax[w] = std::max(wmax[w], tmp.size());
            }
        });
    const size_t w = *std::max_element(wmax.begin(), wmax.end());
    ix->width = w;
    for (size_t l = 0; l < src->num_layers(); ++l) {
        std::vector<u32> rows(src->layer_len(l) * w, UNUSED);
        ranges(src->layer_len(l), [&](size_t b, size_t e, unsigned) {
            std::vector<u32> tmp;
            for (size_t i = b; i < e; ++i) {
                src->get_neighbors(l, i, tmp);
                std::copy(tmp.begin(), tmp.end(), rows.begin() + i * w);
            }
        });
        ix->fixed.push_back(std::move(rows));
    }
    return ix;
}

uint64_t orc_index_len(void* p) { return ((Index*)p)->len(); }
uint64_t orc_index_num_layers(void* p) { return ((Index*)p)->num_layers(); }
uint64_t orc_index_layer_len(void* p, uint64_t l) { return ((Index*)p)->layer_len(l); }
uint64_t orc_index_get_neighbors(void* p, uint64_t idx, uint64_t layer, uint32_t* out, uint64_t cap) {
    std::vector<u32> v;
    ((Index*)p)->get_neighbors(layer, idx, v);
    for (size_t i = 0; i < v.size() && i < cap; ++i) out[i] = v[i];
    return v.size();
}

// Batch search. queries: nq x dim raw f32 (normalised/quantised here unless already_element). i8 kind with
// already_element: queries_i8 holds nq x dim i8 elements.  Outputs padded with 0xFFFFFFFF / +inf.
// stats (optional): nq x 3 u64 {n_dist, n_expand, n_nbr_read}.  threads: static chunks over queries
// (mirrors into_par_iter().for_each(search), src/index/rw/mod.rs:253-255).
int orc_search_batch(void* index, void* elements, const float* queries, const int8_t* queries_i8, uint64_t nq,
                     int already_element, uint64_t max_search, uint64_t num_neighbors, uint32_t* out_ids,
                     float* out_dists, uint32_t* out_counts, uint64_t* stats, int threads) {
    auto* ix = (Index*)index;
    auto* el = (Elements*)elements;
    if (max_search == 0) {
        g_err = "max_search == 0 panics in the reference (index/mod.rs:1019)";
        return 1;
    }
    size_t dim = el->dim;
    auto run = [&](size_t b, size_t e) {
        Query q;
        for (size_t i = b; i < e; ++i) {
            if (el->kind == KIND_I8 && already_element && queries_i8)
                q.q.assign(queries_i8 + i * dim, queries_i8 + (i + 1) * dim);
            else
                el->make_query(queries + i * dim, already_element != 0, &q);
            SearchStats st;
            auto r = index_search(*ix, ix->num_layers(), *el, q, max_search, num_neighbors, &st);
            for (size_t k = 0; k < num_neighbors; ++k) {
                out_ids[i * num_neighbors + k] = k < r.size() ? (u32)r[k].first : UNUSED;
                out_dists[i * num_neighbors + k] = k < r.size() ? r[k].second : INFINITY;
            }
            if (out_counts) out_counts[i] = (u32)r.size();
            if (stats) {
                stats[i * 3 + 0] = st.n_dist;
                stats[i * 3 + 1] = st.n_expand;
                stats[i * 3 + 2] = st.n_nbr_read;
            }
        }
    };
    if (threads <= 1 || nq < 2) {
        run(0, nq);
    } else {
        std::vector<std::thread> ts;
        size_t per = (nq + threads - 1) / threads;
        for (int t = 0; t < threads; ++t) {
            size_t b = std::min<size_t>(nq, per * t), e = std::min<size_t>(nq, per * (t + 1));
            if (b < e) ts.emplace_back(run, b, e);
        }
        for (auto& t : ts) t.join();
    }
    return 0;
}

// ---- reorder ----
void orc_entrypoint_trail(void* index, void* elements, uint64_t idx, uint64_t max_layer, uint32_t* out8) {
    auto* el = (Elements*)elements;
    Query q;
    el->get(idx, &q);
    Trail t = find_entrypoint_trail(*(Index*)index, *el, max_layer, q);
    for (size_t i = 0; i < TRAIL_LAYERS; ++i) out8[i] = t[i];
}
void orc_compute_order(void* index, void* elements, uint64_t* order_out, int threads) {
    auto o = compute_order(*(Index*)index, *(Elements*)elements, threads);
    std::copy(o.begin(), o.end(), order_out);
}
void orc_order_by_keys(void* index, const uint64_t* keys, uint64_t kw, uint64_t* order_out) {
    auto o = order_by_keys(*(Index*)index, keys, kw);
    std::copy(o.begin(), o.end(), order_out);
}
// Returns a new index (compressed, as the reference's reordered Granne holds it) = reorder_layers(index, order).
void* orc_index_apply_order(void* index, const uint64_t* order, uint64_t n) {
    Index fixed;
    reorder_layers(*(Index*)index, std::vector<u64>(order, order + n), &fixed);
    std::vector<u8> bytes;
    write_index_bytes(fixed, bytes);
    return orc_index_from_bytes(bytes.data(), bytes.size());
}
void orc_elements_permute(void* elements, const uint64_t* order, uint64_t n) {
    permute_elements((Elements*)elements, std::vector<u64>(order, order + n));
}
void orc_sum_reorder_keys(void* elements, uint64_t* keys_out) { embedding_reorder_keys(*(Elements*)elements, keys_out); }

// ---- format KAT hooks ----
// Offsets: push every offset, then read them back through the reader (offsets.rs:245-270).  Returns the number of
// offsets the reader reports, or -1 where the reference panics (offsets.rs:158-160,223).
int64_t orc_offsets_roundtrip(const uint64_t* offsets, uint64_t n, uint64_t* out, uint64_t* last_out) {
    OffsetsWriter w;
    for (uint64_t i = 0; i < n; ++i) {
        w.push(offsets[i]);
        if (!w.ok) return -1;
        if (last_out) last_out[i] = w.last_offset;  // Offsets::last (offsets.rs:261-265)
    }
    CompressedLayer r;
    r.chunks = w.chunks.data();
    r.num_chunks = w.chunks.size() / CHUNK_BYTES;
    // Offsets::len (offsets.rs:267-270)
    size_t len = 0;
    if (r.num_chunks) {
        const u8* last = r.chunks + (r.num_chunks - 1) * CHUNK_BYTES;
        size_t l = 0;
        while (l < OFFSETS_PER_CHUNK && CompressedLayer::chunk_delta(last, l) != DELTA_UNUSED) ++l;
        len = OFFSETS_PER_CHUNK * (r.num_chunks - 1) + l;
    }
    for (size_t i = 0; i < len && i < n; ++i) out[i] = r.offset_get(i);
    return (int64_t)len;
}
// MultiSetVector blob from lists (write_as_multi_set_vector, set_vector.rs:169-221, with the predicate already applied
// by the caller); lists are given flattened with their lengths.
uint64_t orc_multiset_blob(const uint32_t* flat, const uint64_t* lens, uint64_t n, uint8_t* out, uint64_t cap) {
    std::vector<std::vector<u32>> lists(n);
    size_t pos = 0;
    for (uint64_t i = 0; i < n; ++i) {
        lists[i].assign(flat + pos, flat + pos + lens[i]);
        pos += lens[i];
    }
    std::vector<u8> blob;
    write_layer_blob(lists, blob);
    if (out == nullptr) return blob.size();
    if (blob.size() > cap) return 0;
    std::memcpy(out, blob.data(), blob.size());
    return blob.size();
}
// MultiSetVector::from_bytes(...).len() / .get(idx) (set_vector.rs:57-69, offsets.rs:127-139)
int64_t orc_multiset_len(const uint8_t* blob, uint64_t len) {
    CompressedLayer L;
    if (!L.load(blob, len)) return -1;
    return (int64_t)L.n;
}
uint64_t orc_multiset_get(const uint8_t* blob, uint64_t len, uint64_t idx, uint32_t* out, uint64_t cap) {
    CompressedLayer L;
    if (!L.load(blob, len) || idx >= L.n) return ~0ull;
    std::vector<u32> v;
    L.get(idx, v);
    for (size_t i = 0; i < v.size() && i < cap; ++i) out[i] = v[i];
    return v.size();
}

// GranneBuilder::select_neighbors (index/mod.rs:849-883) over `elements`; candidates ascending by distance.
uint64_t orc_select_neighbors(void* elements, const uint64_t* cand_ids, const float* cand_dists, uint64_t n,
                              uint64_t max_neighbors, uint64_t* out_ids, float* out_dists) {
    Builder b;
    b.elements = (Elements*)elements;
    std::vector<Builder::Cand> c(n);
    for (uint64_t i = 0; i < n; ++i) c[i] = {cand_ids[i], cand_dists[i]};
    auto r = b.select_neighbors(c, max_neighbors);
    for (size_t i = 0; i < r.size(); ++i) {
        out_ids[i] = r[i].first;
        out_dists[i] = r[i].second;
    }
    return r.size();
}

// Stateful builder (GranneBuilder::new / build_partial / get_index, index/mod.rs:303-315,374-402,483-488): successive
// build_partial calls continue from the layers built so far, like the reference's incremental_build tests.
void* orc_builder_new(void* elements, uint64_t num_neighbors, uint64_t max_search, float layer_multiplier, int reinsert,
                      int64_t expected_num_elements) {
    auto* b = new Builder();
    b->elements = (Elements*)elements;
    b->config.num_neighbors = num_neighbors;
    b->config.max_search = max_search;
    b->config.layer_multiplier = layer_multiplier;
    b->config.reinsert_elements = reinsert != 0;
    b->config.expected_num_elements = expected_num_elements;
    b->ix.use_fixed = true;
    b->ix.width = num_neighbors;
    return b;
}
void orc_builder_free(void* p) {
    auto* b = (Builder*)p;
    delete b->counters;
    delete b;
}
// max_batch > 0: later build_partial calls follow the product's batch schedule (Builder::index_batches), not the
// reference's order; 0 switches back.  The counters accumulate over the builder's life.
void orc_builder_set_max_batch(void* p, uint64_t max_batch) {
    auto* b = (Builder*)p;
    b->max_batch = max_batch;
    if (!b->counters) b->counters = new BuildCounters();
}
// out[6] = {batches, largest batch, connects that found j present, connects that overflowed, non-trivial selects,
// most reverse links into one node within one batch}
void orc_builder_counters(void* p, uint64_t* out) {
    const BuildCounters* c = ((Builder*)p)->counters;
    if (!c) {
        std::fill(out, out + 6, 0);
        return;
    }
    out[0] = c->batches, out[1] = c->max_batch, out[2] = c->connect_present, out[3] = c->connect_overflow;
    out[4] = c->nontrivial_selects, out[5] = c->max_batch_in_links;
}
// the distances add_and_limit_neighbors sorts a row by (:938): dist(ids[k], element idx)
void orc_elements_dists(void* p, uint64_t idx, const uint32_t* ids, uint64_t n, float* out) {
    auto* e = (Elements*)p;
    Query q;
    e->get(idx, &q);
    for (uint64_t k = 0; k < n; ++k) out[k] = e->dist_to_element(ids[k], q);
}
// build_partial(num_elements) exactly (0 indexes nothing); returns 1 where the reference panics
// ("Cannot index fewer elements than already in index", :379-382).
int orc_builder_build_partial(void* p, uint64_t num_elements, int threads) {
    auto* b = (Builder*)p;
    if (num_elements < b->ix.len()) {
        g_err = "Cannot index fewer elements than already in index.";
        return 1;
    }
    b->build_partial(std::min<size_t>(num_elements, b->elements->len()), threads);
    return 0;
}
void* orc_builder_get_index(void* p) {  // a copy of the layers built so far
    auto* b = (Builder*)p;
    auto* ix = new Index(b->ix);
    ix->use_fixed = true;
    if (ix->width == 0) ix->width = b->config.num_neighbors;
    return ix;
}

// GranneBuilder::from_bytes (index/mod.rs:428-457): a builder that continues from an already built index; every
// neighbour list is resized to the new config's num_neighbors (longer lists are truncated, :447).
void* orc_builder_from_index(void* index, void* elements, uint64_t num_neighbors, uint64_t max_search,
                             float layer_multiplier, int reinsert, int64_t expected_num_elements) {
    auto* b = (Builder*)orc_builder_new(elements, num_neighbors, max_search, layer_multiplier, reinsert,
                                        expected_num_elements);
    auto* src = (Index*)index;
    std::vector<u32> tmp;
    for (size_t l = 0; l < src->num_layers(); ++l) {
        std::vector<u32> rows(src->layer_len(l) * num_neighbors, UNUSED);
        for (size_t i = 0; i < src->layer_len(l); ++i) {
            src->get_neighbors(l, i, tmp);
            tmp.resize(num_neighbors, UNUSED);
            std::copy(tmp.begin(), tmp.end(), rows.begin() + i * num_neighbors);
        }
        b->ix.fixed.push_back(std::move(rows));
    }
    return b;
}

}  // extern "C"
