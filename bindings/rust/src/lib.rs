//! Rust shim over the C ABI of granne_b200 (`include/granne_b200.h`): `GpuGranne` and `GpuGranneBuilder` keep the
//! signatures of `granne::Granne` (`src/index/mod.rs:38-160`), the `granne::Index` trait (`:54-104`) and
//! `granne::GranneBuilder` (`:295-531`) on the search path, so call sites only change the type name.
//!
//! This crate cannot be compiled in the repository's build image (it has no Rust toolchain); the same calls are
//! exercised from C++ (`include/granne_b200.hpp`, `tests/helpers/cxx_client.cpp`) and Python (`granne_b200/api.py`).
//! Where the reference panics (malformed file, NaN distance, `max_search == 0`) these methods panic with the
//! library's message, like the reference.

use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

#[repr(C)]
pub struct RawIndex {
    _private: [u8; 0],
}
#[repr(C)]
pub struct RawBuilder {
    _private: [u8; 0],
}
#[repr(C)]
pub struct RawMulti {
    _private: [u8; 0],
}

/// `granne_b200_build_config` — `granne::BuildConfig` (`src/index/mod.rs:198-231`).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct RawBuildConfig {
    pub layer_multiplier: f32,
    pub expected_num_elements: i64, // < 0: None
    pub num_neighbors: u32,
    pub max_search: u32,
    pub reinsert_elements: c_int,
    pub show_progress: c_int,
}

extern "C" {
    fn granne_b200_last_error() -> *const c_char;
    fn granne_b200_open(
        index: *const c_void, index_len: usize, element_kind: c_int, elements: *const c_void, elements_len: usize,
        embeddings: *const c_void, embeddings_len: usize, device: c_int, out: *mut *mut RawIndex,
    ) -> c_int;
    fn granne_b200_close(h: *mut RawIndex);
    fn granne_b200_len(h: *const RawIndex) -> u64;
    fn granne_b200_num_layers(h: *const RawIndex) -> u64;
    fn granne_b200_layer_len(h: *const RawIndex, layer: u64) -> u64;
    fn granne_b200_get_neighbors(
        h: *const RawIndex, idx: u64, layer: u64, out: *mut u32, cap: usize, n_out: *mut usize,
    ) -> c_int;
    fn granne_b200_dim(h: *const RawIndex) -> u64;
    fn granne_b200_get_element(h: *const RawIndex, idx: u64, out: *mut c_void) -> c_int;
    fn granne_b200_get_elements(h: *mut RawIndex, ids: *const u32, n: usize, out: *mut c_void) -> c_int;
    fn granne_b200_get_elements_device(h: *mut RawIndex, d_ids: *const u32, n: usize, d_out: *mut c_void,
                                       cuda_stream: *mut c_void) -> c_int;
    fn granne_b200_search_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32, out_stats: *mut u64,
    ) -> c_int;
    fn granne_b200_write_index(h: *const RawIndex, out: *mut c_void, cap: usize, out_len: *mut usize) -> c_int;
    fn granne_b200_compute_order(h: *mut RawIndex, order_out: *mut u64, cap: u64) -> c_int;

    fn granne_b200_build_config_default(cfg: *mut RawBuildConfig);
    fn granne_b200_builder_new(
        cfg: *const RawBuildConfig, element_kind: c_int, elements: *const c_void, elements_len: usize,
        embeddings: *const c_void, embeddings_len: usize, device: c_int, out: *mut *mut RawBuilder,
    ) -> c_int;
    fn granne_b200_builder_from_index(
        cfg: *const RawBuildConfig, index: *const c_void, index_len: usize, element_kind: c_int,
        elements: *const c_void, elements_len: usize, embeddings: *const c_void, embeddings_len: usize, device: c_int,
        out: *mut *mut RawBuilder,
    ) -> c_int;
    fn granne_b200_builder_from_index_device_elements(
        cfg: *const RawBuildConfig, index: *const c_void, index_len: usize, element_kind: c_int,
        d_element_rows: *const c_void, num_elements: u64, dim: u32, device: c_int, out: *mut *mut RawBuilder,
    ) -> c_int;
    fn granne_b200_builder_free(b: *mut RawBuilder);
    fn granne_b200_builder_append(b: *mut RawBuilder, elements: *const c_void, elements_len: usize) -> c_int;
    fn granne_b200_builder_build(b: *mut RawBuilder, num_elements: u64) -> c_int;
    fn granne_b200_builder_len(b: *const RawBuilder) -> u64;
    fn granne_b200_builder_num_elements(b: *const RawBuilder) -> u64;
    fn granne_b200_builder_num_layers(b: *const RawBuilder) -> u64;
    fn granne_b200_builder_layer_len(b: *const RawBuilder, layer: u64) -> u64;
    fn granne_b200_builder_write_index(b: *mut RawBuilder, out: *mut c_void, cap: usize, out_len: *mut usize) -> c_int;
    fn granne_b200_builder_get_index(b: *mut RawBuilder, out: *mut *mut RawIndex) -> c_int;

    fn granne_b200_compute_embeddings(
        element_kind: c_int, elements: *const c_void, elements_len: usize, embeddings: *const c_void,
        embeddings_len: usize, device: c_int, out: *mut c_void, cap: usize, out_len: *mut usize,
    ) -> c_int;

    fn granne_b200_multi_open(
        mode: c_int, devices: *const c_int, num_devices: usize, element_kind: c_int, index: *const *const c_void,
        index_len: *const usize, elements: *const *const c_void, elements_len: *const usize, num_shards: usize,
        embeddings: *const c_void, embeddings_len: usize, out: *mut *mut RawMulti,
    ) -> c_int;
    fn granne_b200_multi_close(m: *mut RawMulti);
    fn granne_b200_multi_len(m: *const RawMulti) -> u64;
    fn granne_b200_multi_shard_base(m: *const RawMulti, s: usize) -> u64;
    fn granne_b200_multi_part_len(m: *const RawMulti, s: usize) -> u64;
    fn granne_b200_multi_search_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        out_ids: *mut u64, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_exact_search_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, num_neighbors: u32,
        out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_multi_exact_search_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, num_neighbors: u32,
        out_ids: *mut u64, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_exact_range_count(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, radius: f32, counts: *mut u64,
    ) -> c_int;
    fn granne_b200_exact_range_search(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, radius: f32, offsets: *const u64,
        ids: *mut u32, dists: *mut f32,
    ) -> c_int;
    fn granne_b200_multi_exact_range_count(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, radius: f32, counts: *mut u64,
    ) -> c_int;
    fn granne_b200_multi_exact_range_search(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, radius: f32, offsets: *const u64,
        ids: *mut u64, dists: *mut f32,
    ) -> c_int;
    fn granne_b200_exact_search_within_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, offsets: *const u64,
        ids: *const u32, num_neighbors: u32, out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_multi_exact_search_within_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, offsets: *const u64,
        ids: *const u64, num_neighbors: u32, out_ids: *mut u64, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_search_filtered_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        filters: *const u32, num_filters: u32, filter_words: u64, query_filter: *const u32, out_ids: *mut u32,
        out_dists: *mut f32, out_counts: *mut u32, out_stats: *mut u64,
    ) -> c_int;
    fn granne_b200_multi_search_filtered_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        filters: *const u32, num_filters: u32, filter_words: u64, query_filter: *const u32, out_ids: *mut u64,
        out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_exact_search_filtered_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, filters: *const u32,
        num_filters: u32, filter_words: u64, query_filter: *const u32, num_neighbors: u32, out_ids: *mut u32,
        out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_multi_exact_search_filtered_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, filters: *const u32,
        num_filters: u32, filter_words: u64, query_filter: *const u32, num_neighbors: u32, out_ids: *mut u64,
        out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_set_rerank_elements(h: *mut RawIndex, elements: *const c_void, elements_len: usize) -> c_int;
    fn granne_b200_search_rerank_batch(
        h: *mut RawIndex, queries: *const f32, nq: usize, query_format: c_int, max_search: u32, num_candidates: u32,
        num_neighbors: u32, out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32, out_stats: *mut u64,
    ) -> c_int;
    fn granne_b200_multi_set_rerank_elements(
        m: *mut RawMulti, elements: *const *const c_void, elements_len: *const usize,
    ) -> c_int;
    fn granne_b200_set_rerank_embeddings(
        h: *mut RawIndex, elements: *const c_void, elements_len: usize, embeddings: *const c_void,
        embeddings_len: usize,
    ) -> c_int;
    fn granne_b200_multi_set_rerank_embeddings(
        m: *mut RawMulti, elements: *const *const c_void, elements_len: *const usize, embeddings: *const c_void,
        embeddings_len: usize,
    ) -> c_int;
    fn granne_b200_multi_search_rerank_batch(
        m: *mut RawMulti, queries: *const f32, nq: usize, query_format: c_int, max_search: u32, num_candidates: u32,
        num_neighbors: u32, out_ids: *mut u64, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_search_diverse_batch(
        h: *mut RawIndex, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32, out_stats: *mut u64,
    ) -> c_int;
    fn granne_b200_search_diverse_batch_device(
        h: *mut RawIndex, d_queries: *const c_void, nq: usize, query_format: c_int, max_search: u32,
        num_neighbors: u32, d_out_ids: *mut u32, d_out_dists: *mut f32, d_out_counts: *mut u32, d_out_stats: *mut u64,
        cuda_stream: *mut c_void,
    ) -> c_int;
    fn granne_b200_select_neighbors_batch(
        h: *mut RawIndex, cand_ids: *const u32, cand_dists: *const f32, cand_counts: *const u32, nq: usize,
        stride: u32, num_neighbors: u32, out_ids: *mut u32, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_multi_search_diverse_batch(
        m: *mut RawMulti, queries: *const c_void, nq: usize, query_format: c_int, max_search: u32, num_neighbors: u32,
        out_ids: *mut u64, out_dists: *mut f32, out_counts: *mut u32,
    ) -> c_int;
    fn granne_b200_select_neighbors_batch_device(
        h: *mut RawIndex, d_cand_ids: *const u32, d_cand_dists: *const f32, d_cand_counts: *const u32, nq: usize,
        stride: u32, num_neighbors: u32, d_out_ids: *mut u32, d_out_dists: *mut f32, d_out_counts: *mut u32,
        cuda_stream: *mut c_void,
    ) -> c_int;
}

pub const ANGULAR: c_int = 0; // angular::Vectors
pub const ANGULAR_INT: c_int = 1; // angular_int::Vectors
pub const EMBEDDINGS: c_int = 2; // embeddings::SumEmbeddings
const QUERY_RAW_F32: c_int = 0; // the library applies Vector::from
const QUERY_ELEMENT: c_int = 1; // the caller passes an Elements::Element
pub const QUERY_ID: c_int = 2; // u32 element ids (u64 global ids on a multi handle): the query is get_element(id)
pub const QUERY_ID_EXCLUDING: c_int = 3; // QUERY_ID without the element itself (k + 1 searched, self dropped)

fn last_error() -> String {
    unsafe { CStr::from_ptr(granne_b200_last_error()).to_string_lossy().into_owned() }
}

fn check(rc: c_int) {
    if rc != 0 {
        panic!("granne_b200: {}", last_error()); // the reference panics in the same situations
    }
}

fn ptr_or_null(bytes: Option<&[u8]>) -> (*const c_void, usize) {
    match bytes {
        Some(b) => (b.as_ptr() as *const c_void, b.len()),
        None => (std::ptr::null(), 0),
    }
}

/// `granne::embeddings::parsing::compute_embeddings_and_save_to_disk` (`src/elements/embeddings/parsing.rs:102-152`)
/// in memory: the elements file image of the sum of embeddings of every element of a SumEmbeddings container
/// (`elements`, `embeddings`: its two file images), as `ANGULAR_INT` vectors (the quantised raw sum, what the reference
/// writes) or `ANGULAR` vectors (the normalised sum, `SumEmbeddings::get`).  Write the returned image to a file to get
/// the reference's output file.  Panics where the reference does (malformed images, a NaN in a sum).
pub fn compute_embeddings(element_kind: c_int, elements: &[u8], embeddings: &[u8], device: i32) -> Vec<u8> {
    let (el, el_len) = ptr_or_null(Some(elements));
    let (emb, emb_len) = ptr_or_null(Some(embeddings));
    let mut need = 0usize;
    check(unsafe {
        granne_b200_compute_embeddings(element_kind, el, el_len, emb, emb_len, device, std::ptr::null_mut(), 0, &mut need)
    });
    let mut out = vec![0u8; need];
    check(unsafe {
        granne_b200_compute_embeddings(
            element_kind, el, el_len, emb, emb_len, device, out.as_mut_ptr() as *mut c_void, out.len(), &mut need,
        )
    });
    out.truncate(need);
    out
}

/// Drop-in for `Granne<'_, Elements>` on the search path.
pub struct GpuGranne {
    h: *mut RawIndex,
    dim: usize,
}
unsafe impl Send for GpuGranne {}
unsafe impl Sync for GpuGranne {} // Granne::search takes &self (src/index/mod.rs:140)

impl GpuGranne {
    /// `Granne::from_bytes(index, Elements::from_bytes(elements))` (`:108-113`); `element_kind` selects the
    /// container type, `embeddings` is the SumEmbeddings table.
    pub fn from_bytes(index: &[u8], element_kind: c_int, elements: &[u8], embeddings: Option<&[u8]>, device: i32) -> Self {
        let mut h = std::ptr::null_mut();
        let (emb, emb_len) = ptr_or_null(embeddings);
        check(unsafe {
            granne_b200_open(
                index.as_ptr() as *const c_void, index.len(), element_kind, elements.as_ptr() as *const c_void,
                elements.len(), emb, emb_len, device, &mut h,
            )
        });
        let dim = unsafe { granne_b200_dim(h) } as usize;
        Self { h, dim }
    }

    /// `Index::len` (`:54-104`)
    pub fn len(&self) -> usize {
        unsafe { granne_b200_len(self.h) as usize }
    }
    pub fn num_layers(&self) -> usize {
        unsafe { granne_b200_num_layers(self.h) as usize }
    }
    pub fn layer_len(&self, layer: usize) -> usize {
        unsafe { granne_b200_layer_len(self.h, layer as u64) as usize }
    }
    pub fn get_neighbors(&self, index: usize, layer: usize) -> Vec<usize> {
        let mut buf = [0u32; 256];
        let mut n = 0usize;
        check(unsafe { granne_b200_get_neighbors(self.h, index as u64, layer as u64, buf.as_mut_ptr(), buf.len(), &mut n) });
        buf[..n].iter().map(|&x| x as usize).collect()
    }
    /// `Index::write_index` (`src/index/io.rs:11-70`)
    pub fn write_index<B: std::io::Write>(&self, buffer: &mut B) -> std::io::Result<()> {
        let mut need = 0usize;
        check(unsafe { granne_b200_write_index(self.h, std::ptr::null_mut(), 0, &mut need) });
        let mut image = vec![0u8; need];
        check(unsafe { granne_b200_write_index(self.h, image.as_mut_ptr() as *mut c_void, image.len(), &mut need) });
        buffer.write_all(&image[..need])
    }

    /// `Granne::get_element` (`:153-155`) for the f32 element types (normalised vector).
    pub fn get_element(&self, index: usize) -> Vec<f32> {
        let mut out = vec![0f32; self.dim];
        check(unsafe { granne_b200_get_element(self.h, index as u64, out.as_mut_ptr() as *mut c_void) });
        out
    }

    /// `Granne::search(&self, &element, max_search, num_neighbors) -> Vec<(usize, f32)>` (`:140-150`); `element`
    /// holds the components of an `angular::Vector` (already normalised).
    pub fn search(&self, element: &[f32], max_search: usize, num_neighbors: usize) -> Vec<(usize, f32)> {
        self.search_batch(element, 1, QUERY_ELEMENT, max_search, num_neighbors).pop().unwrap()
    }
    /// `search(&Vector::from(raw), ..)`: the raw vector is normalised (or quantised) by the library.
    pub fn search_raw(&self, raw: &[f32], max_search: usize, num_neighbors: usize) -> Vec<(usize, f32)> {
        self.search_batch(raw, 1, QUERY_RAW_F32, max_search, num_neighbors).pop().unwrap()
    }
    /// `nq` independent searches in one launch; `queries` holds `nq * dim` values.
    pub fn search_batch(
        &self, queries: &[f32], nq: usize, query_format: c_int, max_search: usize, num_neighbors: usize,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        let mut ids = vec![0u32; nq * num_neighbors];
        let mut dists = vec![0f32; nq * num_neighbors];
        let mut counts = vec![0u32; nq];
        check(unsafe {
            granne_b200_search_batch(
                self.h, queries.as_ptr() as *const c_void, nq, query_format, max_search as u32, num_neighbors as u32,
                ids.as_mut_ptr(), dists.as_mut_ptr(), counts.as_mut_ptr(), std::ptr::null_mut(),
            )
        });
        (0..nq)
            .map(|q| {
                (0..counts[q] as usize)
                    .map(|j| (ids[q * num_neighbors + j] as usize, dists[q * num_neighbors + j]))
                    .collect()
            })
            .collect()
    }
    /// Exact k nearest neighbours (not a reference function): the first `min(k, len())` elements by
    /// `(dist_to_element, id)`, the reference's distance bit for bit; `k <= 1024`.  The ground truth of recall.
    pub fn exact_search_batch(
        &self, queries: &[f32], nq: usize, query_format: c_int, num_neighbors: usize,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        let mut ids = vec![0u32; nq * num_neighbors];
        let mut dists = vec![0f32; nq * num_neighbors];
        let mut counts = vec![0u32; nq];
        check(unsafe {
            granne_b200_exact_search_batch(
                self.h, queries.as_ptr() as *const c_void, nq, query_format, num_neighbors as u32, ids.as_mut_ptr(),
                dists.as_mut_ptr(), counts.as_mut_ptr(),
            )
        });
        (0..nq)
            .map(|q| {
                (0..counts[q] as usize)
                    .map(|j| (ids[q * num_neighbors + j] as usize, dists[q * num_neighbors + j]))
                    .collect()
            })
            .collect()
    }

    /// Exact range search (not a reference function): every element of `[0, len())` whose distance to the query is
    /// `<= radius`, sorted by `(dist_to_element, id)`, the reference's distance bit for bit; count, then fill.
    pub fn exact_range_search(
        &self, queries: &[f32], nq: usize, query_format: c_int, radius: f32,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        let q = queries.as_ptr() as *const c_void;
        let mut counts = vec![0u64; nq];
        check(unsafe { granne_b200_exact_range_count(self.h, q, nq, query_format, radius, counts.as_mut_ptr()) });
        let mut offsets = vec![0u64; nq + 1];
        for i in 0..nq {
            offsets[i + 1] = offsets[i] + counts[i];
        }
        let mut ids = vec![0u32; offsets[nq] as usize];
        let mut dists = vec![0f32; offsets[nq] as usize];
        check(unsafe {
            granne_b200_exact_range_search(self.h, q, nq, query_format, radius, offsets.as_ptr(), ids.as_mut_ptr(),
                                           dists.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (offsets[i] as usize..offsets[i + 1] as usize).map(|j| (ids[j] as usize, dists[j])).collect())
            .collect()
    }

    /// Exact k nearest neighbours of each query within its own candidate list (not a reference function):
    /// `lists[q]` holds query q's ids (< `len()`; duplicates count once); the first min(k, |set(lists[q])|) by
    /// (distance, id), the reference's distance bit for bit.
    pub fn exact_search_within(
        &self, queries: &[f32], nq: usize, query_format: c_int, lists: &[Vec<u32>], num_neighbors: usize,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        assert_eq!(lists.len(), nq);
        let mut offsets = vec![0u64];
        let mut cand = Vec::new();
        for l in lists {
            cand.extend_from_slice(l);
            offsets.push(cand.len() as u64);
        }
        let mut ids = vec![0u32; nq * num_neighbors];
        let mut dists = vec![0f32; nq * num_neighbors];
        let mut counts = vec![0u32; nq];
        check(unsafe {
            granne_b200_exact_search_within_batch(
                self.h, queries.as_ptr() as *const c_void, nq, query_format, offsets.as_ptr(), cand.as_ptr(),
                num_neighbors as u32, ids.as_mut_ptr(), dists.as_mut_ptr(), counts.as_mut_ptr(),
            )
        });
        (0..nq)
            .map(|q| {
                (0..counts[q] as usize)
                    .map(|j| (ids[q * num_neighbors + j] as usize, dists[q * num_neighbors + j]))
                    .collect()
            })
            .collect()
    }

    /// Filtered search (not a reference function): `search`'s traversal, unchanged, keeping the first k elements by
    /// (distance, id) among those it scores in the bottom layer that the query's filter admits.  `filters` holds
    /// `filters.len() / filter_words` bitmaps (id i: bit i % 32 of word i / 32, `filter_words >= ceil(len() / 32)`);
    /// `query_filter` picks each query's bitmap (None: bitmap 0).  k <= GRANNE_B200_EXACT_MAX_K.
    pub fn search_filtered(
        &self, queries: &[f32], nq: usize, query_format: c_int, max_search: usize, num_neighbors: usize,
        filters: &[u32], filter_words: usize, query_filter: Option<&[u32]>,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        assert!(filter_words > 0 && filters.len() % filter_words == 0);
        if let Some(f) = query_filter {
            assert_eq!(f.len(), nq);
        }
        let mut ids = vec![0u32; nq * num_neighbors];
        let mut dists = vec![0f32; nq * num_neighbors];
        let mut counts = vec![0u32; nq];
        check(unsafe {
            granne_b200_search_filtered_batch(
                self.h, queries.as_ptr() as *const c_void, nq, query_format, max_search as u32, num_neighbors as u32,
                filters.as_ptr(), (filters.len() / filter_words) as u32, filter_words as u64,
                query_filter.map_or(std::ptr::null(), |f| f.as_ptr()), ids.as_mut_ptr(), dists.as_mut_ptr(),
                counts.as_mut_ptr(), std::ptr::null_mut(),
            )
        });
        (0..nq)
            .map(|q| {
                (0..counts[q] as usize)
                    .map(|j| (ids[q * num_neighbors + j] as usize, dists[q * num_neighbors + j]))
                    .collect()
            })
            .collect()
    }

    /// Exact filtered k-NN (not a reference function): the first min(k, |A|) of the ids < len() the query's filter
    /// admits, by (distance, id), with `exact_search`'s distances.  Filters as in `search_filtered`; no max_search.
    pub fn exact_search_filtered(
        &self, queries: &[f32], nq: usize, query_format: c_int, num_neighbors: usize, filters: &[u32],
        filter_words: usize, query_filter: Option<&[u32]>,
    ) -> Vec<Vec<(usize, f32)>> {
        assert_eq!(queries.len(), nq * self.dim);
        assert!(filter_words > 0 && filters.len() % filter_words == 0);
        if let Some(f) = query_filter {
            assert_eq!(f.len(), nq);
        }
        let mut ids = vec![0u32; nq * num_neighbors];
        let mut dists = vec![0f32; nq * num_neighbors];
        let mut counts = vec![0u32; nq];
        check(unsafe {
            granne_b200_exact_search_filtered_batch(
                self.h, queries.as_ptr() as *const c_void, nq, query_format, filters.as_ptr(),
                (filters.len() / filter_words) as u32, filter_words as u64,
                query_filter.map_or(std::ptr::null(), |f| f.as_ptr()), num_neighbors as u32, ids.as_mut_ptr(),
                dists.as_mut_ptr(), counts.as_mut_ptr(),
            )
        });
        (0..nq)
            .map(|q| {
                (0..counts[q] as usize)
                    .map(|j| (ids[q * num_neighbors + j] as usize, dists[q * num_neighbors + j]))
                    .collect()
            })
            .collect()
    }

    /// The ordering half of `Granne::reorder` (`src/index/reorder.rs:126-174`); apply it with
    /// `granne_b200_apply_order` (or granne's own `reorder_layers` + `Permutable::permute`).
    pub fn compute_order(&mut self) -> Vec<usize> {
        let mut order = vec![0u64; self.len()];
        check(unsafe { granne_b200_compute_order(self.h, order.as_mut_ptr(), order.len() as u64) });
        order.into_iter().map(|x| x as usize).collect()
    }
}

impl Drop for GpuGranne {
    fn drop(&mut self) {
        unsafe { granne_b200_close(self.h) }
    }
}

/// `granne::BuildConfig` with the reference's fluent setters (`src/index/mod.rs:233-291`).
#[derive(Clone, Copy)]
pub struct GpuBuildConfig(pub RawBuildConfig);

impl Default for GpuBuildConfig {
    fn default() -> Self {
        let mut raw = RawBuildConfig {
            layer_multiplier: 0.0, expected_num_elements: -1, num_neighbors: 0, max_search: 0, reinsert_elements: 0,
            show_progress: 0,
        };
        unsafe { granne_b200_build_config_default(&mut raw) };
        GpuBuildConfig(raw)
    }
}

impl GpuBuildConfig {
    pub fn layer_multiplier(mut self, v: f32) -> Self { self.0.layer_multiplier = v; self }
    pub fn expected_num_elements(mut self, v: usize) -> Self { self.0.expected_num_elements = v as i64; self }
    pub fn num_neighbors(mut self, v: usize) -> Self { self.0.num_neighbors = v as u32; self }
    pub fn max_search(mut self, v: usize) -> Self { self.0.max_search = v as u32; self }
    pub fn reinsert_elements(mut self, v: bool) -> Self { self.0.reinsert_elements = v as c_int; self }
    pub fn show_progress(mut self, v: bool) -> Self { self.0.show_progress = v as c_int; self }
}

/// Drop-in for `GranneBuilder<Elements>` (`src/index/mod.rs:295-531`).
pub struct GpuGranneBuilder {
    b: *mut RawBuilder,
}
unsafe impl Send for GpuGranneBuilder {}

impl GpuGranneBuilder {
    /// `GranneBuilder::new(config, elements)` (`:303-315`); `elements` is the container's file image
    /// (`io::Writeable::write`).
    pub fn new(config: GpuBuildConfig, element_kind: c_int, elements: &[u8], embeddings: Option<&[u8]>, device: i32) -> Self {
        let mut b = std::ptr::null_mut();
        let (emb, emb_len) = ptr_or_null(embeddings);
        check(unsafe {
            granne_b200_builder_new(
                &config.0, element_kind, elements.as_ptr() as *const c_void, elements.len(), emb, emb_len, device, &mut b,
            )
        });
        Self { b }
    }
    /// `GranneBuilder::from_bytes(config, index, elements)` (`:428-461`): continues from an index file image; every
    /// neighbour list is truncated or padded to the config's `num_neighbors`, like the reference.
    pub fn from_bytes(
        config: GpuBuildConfig, index: &[u8], element_kind: c_int, elements: &[u8], embeddings: Option<&[u8]>,
        device: i32,
    ) -> Self {
        let mut b = std::ptr::null_mut();
        let (emb, emb_len) = ptr_or_null(embeddings);
        check(unsafe {
            granne_b200_builder_from_index(
                &config.0, index.as_ptr() as *const c_void, index.len(), element_kind,
                elements.as_ptr() as *const c_void, elements.len(), emb, emb_len, device, &mut b,
            )
        });
        Self { b }
    }
    /// `from_bytes` over a device-resident container: `d_element_rows` is `num_elements x dim` elements in the
    /// memory of `device` (see `granne_b200_builder_new_device_elements`).
    pub unsafe fn from_bytes_device_elements(
        config: GpuBuildConfig, index: &[u8], element_kind: c_int, d_element_rows: *const c_void, num_elements: usize,
        dim: usize, device: i32,
    ) -> Self {
        let mut b = std::ptr::null_mut();
        check(granne_b200_builder_from_index_device_elements(
            &config.0, index.as_ptr() as *const c_void, index.len(), element_kind, d_element_rows,
            num_elements as u64, dim as u32, device, &mut b,
        ));
        Self { b }
    }
    /// `Builder::build` (`:366-368`)
    pub fn build(&mut self) {
        check(unsafe { granne_b200_builder_build(self.b, 0) });
    }
    /// `Builder::build_partial` (`:374-402`)
    pub fn build_partial(&mut self, num_elements: usize) {
        if num_elements > 0 {
            check(unsafe { granne_b200_builder_build(self.b, num_elements as u64) });
        }
    }
    /// `GranneBuilder::push` for every row of an elements file image (`:512-531`)
    pub fn push_all(&mut self, elements: &[u8]) {
        check(unsafe { granne_b200_builder_append(self.b, elements.as_ptr() as *const c_void, elements.len()) });
    }
    pub fn len(&self) -> usize {
        unsafe { granne_b200_builder_len(self.b) as usize }
    }
    pub fn num_elements(&self) -> usize {
        unsafe { granne_b200_builder_num_elements(self.b) as usize }
    }
    pub fn num_layers(&self) -> usize {
        unsafe { granne_b200_builder_num_layers(self.b) as usize }
    }
    pub fn layer_len(&self, layer: usize) -> usize {
        unsafe { granne_b200_builder_layer_len(self.b, layer as u64) as usize }
    }
    /// `Index::write_index` (`:358-361`)
    pub fn write_index<B: std::io::Write>(&mut self, buffer: &mut B) -> std::io::Result<()> {
        let mut need = 0usize;
        check(unsafe { granne_b200_builder_write_index(self.b, std::ptr::null_mut(), 0, &mut need) });
        let mut image = vec![0u8; need];
        check(unsafe { granne_b200_builder_write_index(self.b, image.as_mut_ptr() as *mut c_void, image.len(), &mut need) });
        buffer.write_all(&image[..need])
    }
    /// `GranneBuilder::get_index` (`:483-488`): a searchable snapshot
    pub fn get_index(&mut self) -> GpuGranne {
        let mut h = std::ptr::null_mut();
        check(unsafe { granne_b200_builder_get_index(self.b, &mut h) });
        let dim = unsafe { granne_b200_dim(h) } as usize;
        GpuGranne { h, dim }
    }
}

impl Drop for GpuGranneBuilder {
    fn drop(&mut self) {
        unsafe { granne_b200_builder_free(self.b) }
    }
}

pub const MODE_REPLICATED: c_int = 0; // one index on every device, query batches sliced
pub const MODE_RANGE_PARTITIONED: c_int = 1; // one independent index per shard, merged by (distance, global id)

/// Several GPUs of this process behind one handle (`granne_b200_multi_*`): `Granne::from_bytes` + `search` with the
/// index replicated on every device or range-partitioned into independent shards (granne's own sharding of the
/// element set, `src/elements/embeddings/parsing.rs:63-100`; merge order of `into_sorted_vec`, `src/index/mod.rs:1036`).
pub struct GpuMultiGranne {
    m: *mut RawMulti,
    dim: usize,
}
unsafe impl Send for GpuMultiGranne {}
unsafe impl Sync for GpuMultiGranne {}

impl GpuMultiGranne {
    /// `shards`: one `(index bytes, elements bytes)` pair (replicated) or one per shard (range-partitioned);
    /// angular f32 elements (`dim` floats per row).
    pub fn open(mode: c_int, shards: &[(&[u8], &[u8])], devices: &[i32], dim: usize) -> Self {
        let ip: Vec<*const c_void> = shards.iter().map(|s| s.0.as_ptr() as *const c_void).collect();
        let il: Vec<usize> = shards.iter().map(|s| s.0.len()).collect();
        let ep: Vec<*const c_void> = shards.iter().map(|s| s.1.as_ptr() as *const c_void).collect();
        let el: Vec<usize> = shards.iter().map(|s| s.1.len()).collect();
        let dv: Vec<c_int> = devices.iter().map(|&d| d as c_int).collect();
        let mut m = std::ptr::null_mut();
        check(unsafe {
            granne_b200_multi_open(mode, dv.as_ptr(), dv.len(), ANGULAR, ip.as_ptr(), il.as_ptr(), ep.as_ptr(),
                                   el.as_ptr(), shards.len(), std::ptr::null(), 0, &mut m)
        });
        GpuMultiGranne { m, dim }
    }
    pub fn len(&self) -> usize {
        unsafe { granne_b200_multi_len(self.m) as usize }
    }
    pub fn shard_base(&self, s: usize) -> usize {
        unsafe { granne_b200_multi_shard_base(self.m, s) as usize }
    }
    /// `Granne::search` for a batch of normalised vectors; ids are global.
    pub fn search_batch(&self, elements: &[f32], max_search: usize, num_neighbors: usize) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        let (mut ids, mut d, mut c) = (vec![0u64; nq * num_neighbors], vec![0f32; nq * num_neighbors], vec![0u32; nq]);
        check(unsafe {
            granne_b200_multi_search_batch(self.m, elements.as_ptr() as *const c_void, nq, QUERY_ELEMENT,
                                           max_search as u32, num_neighbors as u32, ids.as_mut_ptr(), d.as_mut_ptr(),
                                           c.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (0..c[i] as usize).map(|j| (ids[i * num_neighbors + j] as usize, d[i * num_neighbors + j])).collect())
            .collect()
    }
    /// Exact k nearest neighbours over every shard for a batch of normalised vectors; ids are global.
    pub fn exact_search_batch(&self, elements: &[f32], num_neighbors: usize) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        let (mut ids, mut d, mut c) = (vec![0u64; nq * num_neighbors], vec![0f32; nq * num_neighbors], vec![0u32; nq]);
        check(unsafe {
            granne_b200_multi_exact_search_batch(self.m, elements.as_ptr() as *const c_void, nq, QUERY_ELEMENT,
                                                 num_neighbors as u32, ids.as_mut_ptr(), d.as_mut_ptr(),
                                                 c.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (0..c[i] as usize).map(|j| (ids[i * num_neighbors + j] as usize, d[i * num_neighbors + j])).collect())
            .collect()
    }

    /// `exact_range_search` over every shard for a batch of normalised vectors; ids are global.
    pub fn exact_range_search(&self, elements: &[f32], radius: f32) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        let q = elements.as_ptr() as *const c_void;
        let mut counts = vec![0u64; nq];
        check(unsafe { granne_b200_multi_exact_range_count(self.m, q, nq, QUERY_ELEMENT, radius, counts.as_mut_ptr()) });
        let mut offsets = vec![0u64; nq + 1];
        for i in 0..nq {
            offsets[i + 1] = offsets[i] + counts[i];
        }
        let (mut ids, mut d) = (vec![0u64; offsets[nq] as usize], vec![0f32; offsets[nq] as usize]);
        check(unsafe {
            granne_b200_multi_exact_range_search(self.m, q, nq, QUERY_ELEMENT, radius, offsets.as_ptr(),
                                                 ids.as_mut_ptr(), d.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (offsets[i] as usize..offsets[i + 1] as usize).map(|j| (ids[j] as usize, d[j])).collect())
            .collect()
    }

    /// `exact_search_within` over every part: GLOBAL ids in the lists and in the results.
    pub fn exact_search_within(
        &self, elements: &[f32], lists: &[Vec<u64>], num_neighbors: usize,
    ) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        assert_eq!(lists.len(), nq);
        let mut offsets = vec![0u64];
        let mut cand = Vec::new();
        for l in lists {
            cand.extend_from_slice(l);
            offsets.push(cand.len() as u64);
        }
        let (mut ids, mut d, mut c) = (vec![0u64; nq * num_neighbors], vec![0f32; nq * num_neighbors], vec![0u32; nq]);
        check(unsafe {
            granne_b200_multi_exact_search_within_batch(self.m, elements.as_ptr() as *const c_void, nq, QUERY_ELEMENT,
                                                        offsets.as_ptr(), cand.as_ptr(), num_neighbors as u32,
                                                        ids.as_mut_ptr(), d.as_mut_ptr(), c.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (0..c[i] as usize).map(|j| (ids[i * num_neighbors + j] as usize, d[i * num_neighbors + j])).collect())
            .collect()
    }

    /// `search_filtered` over every part: the bitmaps are over GLOBAL ids, and so are the results.
    pub fn search_filtered(
        &self, elements: &[f32], max_search: usize, num_neighbors: usize, filters: &[u32], filter_words: usize,
        query_filter: Option<&[u32]>,
    ) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        assert!(filter_words > 0 && filters.len() % filter_words == 0);
        if let Some(f) = query_filter {
            assert_eq!(f.len(), nq);
        }
        let (mut ids, mut d, mut c) = (vec![0u64; nq * num_neighbors], vec![0f32; nq * num_neighbors], vec![0u32; nq]);
        check(unsafe {
            granne_b200_multi_search_filtered_batch(self.m, elements.as_ptr() as *const c_void, nq, QUERY_ELEMENT,
                                                    max_search as u32, num_neighbors as u32, filters.as_ptr(),
                                                    (filters.len() / filter_words) as u32, filter_words as u64,
                                                    query_filter.map_or(std::ptr::null(), |f| f.as_ptr()),
                                                    ids.as_mut_ptr(), d.as_mut_ptr(), c.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (0..c[i] as usize).map(|j| (ids[i * num_neighbors + j] as usize, d[i * num_neighbors + j])).collect())
            .collect()
    }

    /// `exact_search_filtered` over every part: the bitmaps are over GLOBAL ids, and so are the results.
    pub fn exact_search_filtered(
        &self, elements: &[f32], num_neighbors: usize, filters: &[u32], filter_words: usize,
        query_filter: Option<&[u32]>,
    ) -> Vec<Vec<(usize, f32)>> {
        let nq = elements.len() / self.dim;
        assert!(filter_words > 0 && filters.len() % filter_words == 0);
        if let Some(f) = query_filter {
            assert_eq!(f.len(), nq);
        }
        let (mut ids, mut d, mut c) = (vec![0u64; nq * num_neighbors], vec![0f32; nq * num_neighbors], vec![0u32; nq]);
        check(unsafe {
            granne_b200_multi_exact_search_filtered_batch(self.m, elements.as_ptr() as *const c_void, nq, QUERY_ELEMENT,
                                                          filters.as_ptr(), (filters.len() / filter_words) as u32,
                                                          filter_words as u64,
                                                          query_filter.map_or(std::ptr::null(), |f| f.as_ptr()),
                                                          num_neighbors as u32, ids.as_mut_ptr(), d.as_mut_ptr(),
                                                          c.as_mut_ptr())
        });
        (0..nq)
            .map(|i| (0..c[i] as usize).map(|j| (ids[i * num_neighbors + j] as usize, d[i * num_neighbors + j])).collect())
            .collect()
    }
}

impl Drop for GpuMultiGranne {
    fn drop(&mut self) {
        unsafe { granne_b200_multi_close(self.m) }
    }
}
