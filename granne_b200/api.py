"""ctypes binding over include/granne_b200.h."""
import collections
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.environ.get("GRANNE_B200_LIB") or os.path.join(_HERE, "libgranne_b200.so")  # env: tuning variants

ANGULAR, ANGULAR_INT, EMBEDDINGS = 0, 1, 2
QUERY_RAW_F32, QUERY_ELEMENT, QUERY_ID, QUERY_ID_EXCLUDING = 0, 1, 2, 3
_ELEMENT_TYPES = {"angular": ANGULAR, "angular_int": ANGULAR_INT, "embeddings": EMBEDDINGS}
STATS_PER_QUERY = 4
EXACT_MAX_K = 1024  # GRANNE_B200_EXACT_MAX_K
RERANK_MAX_CANDIDATES = 1024  # GRANNE_B200_RERANK_MAX_CANDIDATES
DIVERSE_MAX_CANDIDATES = 1024  # GRANNE_B200_DIVERSE_MAX_CANDIDATES
DEFAULT_MAX_SEARCH = 200   # py/src/lib.rs:14
DEFAULT_NUM_ELEMENTS = 10  # py/src/lib.rs:15


class GranneError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("granne_b200 error %d: %s" % (code, message))
        self.code = code


def library_path():
    return _LIB


_lib = None


def load_library():
    """Loads libgranne_b200.so; raises if it has not been built (python -m granne_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB):
        raise ImportError("granne_b200: %s is missing — build it with `python -m granne_b200.build` "
                          "(there is no CPU fallback)" % _LIB)
    L = C.CDLL(_LIB)
    vp, sz, u64, u32, i32 = C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint32, C.c_int
    sig = {
        "granne_b200_abi_version": (i32, []),
        "granne_b200_last_error": (C.c_char_p, []),
        "granne_b200_open": (i32, [vp, sz, i32, vp, sz, vp, sz, i32, C.POINTER(vp)]),
        "granne_b200_open_files": (i32, [C.c_char_p, i32, C.c_char_p, C.c_char_p, i32, C.POINTER(vp)]),
        "granne_b200_open_device_elements": (i32, [vp, sz, i32, vp, u64, u32, i32, C.POINTER(vp)]),
        "granne_b200_builder_new_device_elements": (i32, [vp, i32, vp, u64, u32, i32, C.POINTER(vp)]),
        "granne_b200_elements_from_raw_device": (i32, [i32, vp, u64, u32, i32, vp, vp]),
        "granne_b200_compute_embeddings": (i32, [i32, vp, sz, vp, sz, i32, vp, sz, C.POINTER(sz)]),
        "granne_b200_compute_embeddings_device": (i32, [i32, vp, sz, vp, sz, i32, vp, C.POINTER(u64), C.POINTER(u32),
                                                        vp]),
        "granne_b200_close": (None, [vp]),
        "granne_b200_len": (u64, [vp]),
        "granne_b200_num_layers": (u64, [vp]),
        "granne_b200_layer_len": (u64, [vp, u64]),
        "granne_b200_get_neighbors": (i32, [vp, u64, u64, vp, sz, C.POINTER(sz)]),
        "granne_b200_num_elements": (u64, [vp]),
        "granne_b200_dim": (u64, [vp]),
        "granne_b200_element_kind": (i32, [vp]),
        "granne_b200_get_element": (i32, [vp, u64, vp]),
        "granne_b200_get_elements": (i32, [vp, vp, sz, vp]),
        "granne_b200_get_elements_device": (i32, [vp, vp, sz, vp, vp]),
        "granne_b200_search_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp, vp]),
        "granne_b200_search_batch_device": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp, vp, vp]),
        "granne_b200_search_batch_device_gather": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp, vp]),
        "granne_b200_stream_status": (i32, [vp]),
        "granne_b200_stream_status_of": (i32, [vp, vp]),
        "granne_b200_multi_part_len": (u64, [vp, sz]),
        "granne_b200_release_stream": (i32, [vp, vp]),
        "granne_b200_merge_topk_device": (i32, [i32, vp, vp, vp, sz, sz, u32, vp, vp, vp]),
        "granne_b200_inspect_index": (i32, [vp, sz, vp, vp, vp, vp, sz]),
        "granne_b200_decode_layer": (i32, [vp, sz, u64, vp, sz]),
        "granne_b200_compute_distances": (i32, [i32, vp, vp, u64, u32, i32, vp]),
        "granne_b200_write_index": (i32, [vp, vp, sz, C.POINTER(sz)]),
        "granne_b200_reencode_index": (i32, [vp, sz, vp, sz, C.POINTER(sz)]),
        "granne_b200_compute_order": (i32, [vp, vp, u64]),
        "granne_b200_order_from_trails": (i32, [vp, u32, vp, u64, vp]),
        "granne_b200_order_by_keys": (i32, [vp, sz, vp, u64, u32, vp]),
        "granne_b200_embedding_reorder_keys": (i32, [vp, sz, vp, sz, vp]),
        "granne_b200_apply_order": (i32, [vp, sz, i32, vp, sz, vp, u64, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]),
        "granne_b200_build_config_default": (None, [vp]),
        "granne_b200_builder_new": (i32, [vp, i32, vp, sz, vp, sz, i32, C.POINTER(vp)]),
        "granne_b200_builder_from_index": (i32, [vp, vp, sz, i32, vp, sz, vp, sz, i32, C.POINTER(vp)]),
        "granne_b200_builder_from_index_device_elements": (i32, [vp, vp, sz, i32, vp, u64, u32, i32, C.POINTER(vp)]),
        "granne_b200_builder_append": (i32, [vp, vp, sz]),
        "granne_b200_builder_build": (i32, [vp, u64]),
        "granne_b200_builder_len": (u64, [vp]),
        "granne_b200_builder_num_layers": (u64, [vp]),
        "granne_b200_builder_layer_len": (u64, [vp, u64]),
        "granne_b200_builder_num_elements": (u64, [vp]),
        "granne_b200_builder_get_neighbors": (i32, [vp, u64, u64, vp, sz, C.POINTER(sz)]),
        "granne_b200_builder_write_index": (i32, [vp, vp, sz, C.POINTER(sz)]),
        "granne_b200_builder_get_index": (i32, [vp, C.POINTER(vp)]),
        "granne_b200_builder_free": (None, [vp]),
        "granne_b200_elements_from_raw": (i32, [i32, vp, u64, u32, i32, vp, sz, C.POINTER(sz)]),
        "granne_b200_launch_count": (u64, [vp]),
        "granne_b200_multi_open": (i32, [i32, vp, sz, i32, vp, vp, vp, vp, sz, vp, sz, C.POINTER(vp)]),
        "granne_b200_multi_close": (None, [vp]),
        "granne_b200_multi_len": (u64, [vp]),
        "granne_b200_multi_num_parts": (sz, [vp]),
        "granne_b200_multi_shard_base": (u64, [vp, sz]),
        "granne_b200_multi_search_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp]),
        "granne_b200_exact_search_batch": (i32, [vp, vp, sz, i32, u32, vp, vp, vp]),
        "granne_b200_exact_search_batch_device": (i32, [vp, vp, sz, i32, u32, vp, vp, vp, vp]),
        "granne_b200_multi_exact_search_batch": (i32, [vp, vp, sz, i32, u32, vp, vp, vp]),
        "granne_b200_exact_search_within_batch": (i32, [vp, vp, sz, i32, vp, vp, u32, vp, vp, vp]),
        "granne_b200_exact_search_within_batch_device": (i32, [vp, vp, sz, i32, vp, vp, u32, vp, vp, vp, vp]),
        "granne_b200_multi_exact_search_within_batch": (i32, [vp, vp, sz, i32, vp, vp, u32, vp, vp, vp]),
        "granne_b200_exact_range_count": (i32, [vp, vp, sz, i32, C.c_float, vp]),
        "granne_b200_exact_range_count_device": (i32, [vp, vp, sz, i32, C.c_float, vp, vp]),
        "granne_b200_exact_range_search": (i32, [vp, vp, sz, i32, C.c_float, vp, vp, vp]),
        "granne_b200_exact_range_search_device": (i32, [vp, vp, sz, i32, C.c_float, vp, vp, vp, vp]),
        "granne_b200_multi_exact_range_count": (i32, [vp, vp, sz, i32, C.c_float, vp]),
        "granne_b200_multi_exact_range_search": (i32, [vp, vp, sz, i32, C.c_float, vp, vp, vp]),
        "granne_b200_search_filtered_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, u32, u64, vp, vp, vp, vp, vp]),
        "granne_b200_search_filtered_batch_device": (i32, [vp, vp, sz, i32, u32, u32, vp, u32, u64, vp, vp, vp, vp, vp,
                                                           vp]),
        "granne_b200_multi_search_filtered_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, u32, u64, vp, vp, vp, vp]),
        "granne_b200_exact_search_filtered_batch": (i32, [vp, vp, sz, i32, vp, u32, u64, vp, u32, vp, vp, vp]),
        "granne_b200_exact_search_filtered_batch_device": (i32, [vp, vp, sz, i32, vp, u32, u64, vp, u32, vp, vp, vp,
                                                                 vp]),
        "granne_b200_multi_exact_search_filtered_batch": (i32, [vp, vp, sz, i32, vp, u32, u64, vp, u32, vp, vp, vp]),
        "granne_b200_set_rerank_elements": (i32, [vp, vp, sz]),
        "granne_b200_set_rerank_elements_device": (i32, [vp, vp, u64, u32]),
        "granne_b200_search_rerank_batch": (i32, [vp, vp, sz, i32, u32, u32, u32, vp, vp, vp, vp]),
        "granne_b200_search_rerank_batch_device": (i32, [vp, vp, sz, i32, u32, u32, u32, vp, vp, vp, vp, vp]),
        "granne_b200_multi_set_rerank_elements": (i32, [vp, vp, vp]),
        "granne_b200_set_rerank_embeddings": (i32, [vp, vp, sz, vp, sz]),
        "granne_b200_multi_set_rerank_embeddings": (i32, [vp, vp, vp, vp, sz]),
        "granne_b200_multi_search_rerank_batch": (i32, [vp, vp, sz, i32, u32, u32, u32, vp, vp, vp]),
        "granne_b200_search_diverse_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp, vp]),
        "granne_b200_search_diverse_batch_device": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp, vp, vp]),
        "granne_b200_multi_search_diverse_batch": (i32, [vp, vp, sz, i32, u32, u32, vp, vp, vp]),
        "granne_b200_select_neighbors_batch": (i32, [vp, vp, vp, vp, sz, u32, u32, vp, vp, vp]),
        "granne_b200_select_neighbors_batch_device": (i32, [vp, vp, vp, vp, sz, u32, u32, vp, vp, vp, vp]),
        "granne_b200_device_bytes": (u64, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise GranneError(rc, load_library().granne_b200_last_error().decode("utf-8", "replace"))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _kind(element_type):
    if isinstance(element_type, str):
        try:
            return _ELEMENT_TYPES[element_type.lower()]
        except KeyError:
            raise ValueError("Invalid element type")  # py/src/lib.rs:208
    return int(element_type)


def _host_queries(queries, already_element, dim=None):
    """(contiguous queries, query format) of a host call: int8 rows are elements, everything else becomes float32.
    dim: the index's width, where the handle tells it."""
    q = np.asarray(queries)
    fmt = QUERY_ELEMENT if already_element or q.dtype == np.int8 else QUERY_RAW_F32
    q = np.ascontiguousarray(q, dtype=None if q.dtype == np.int8 else np.float32)
    if q.ndim != 2 or (dim is not None and q.shape[1] != dim):
        raise ValueError("queries must have shape (nq, %s)" % ("dim" if dim is None else dim))
    return q, fmt


def _id_queries(ids, exclude_self, id_dtype):
    """(contiguous ids, query format) of a host call by element id: a 1-D array of non-negative integers that fit
    id_dtype (uint32 for one index, uint64 global ids for a MultiGranne)."""
    a = np.asarray(ids)
    if a.ndim != 1:
        raise ValueError("ids must be a 1-D integer array")
    if a.size and a.dtype.kind not in "iu":
        raise ValueError("ids must be integers, not %s" % a.dtype)
    if a.size and a.dtype.kind == "i" and a.min() < 0:
        raise ValueError("ids must be non-negative")
    if a.size and int(a.max()) > np.iinfo(id_dtype).max:
        raise ValueError("ids must fit %s" % np.dtype(id_dtype).name)
    return np.ascontiguousarray(a, dtype=id_dtype), QUERY_ID_EXCLUDING if exclude_self else QUERY_ID


def _raw_f32_queries(queries, dim=None):
    """The queries of a two-stage call: raw float32 only."""
    if np.asarray(queries).dtype == np.int8:
        raise ValueError("the two-stage search takes raw float32 queries")
    return _host_queries(queries, False, dim)[0]


def _host_outputs(nq, k, id_dtype, with_stats=False):
    """(ids, dists, counts, stats) for the results of nq queries; stats is None unless with_stats."""
    shape = (nq, k)
    return (np.empty(shape, dtype=id_dtype), np.empty(shape, dtype=np.float32), np.empty(nq, dtype=np.uint32),
            np.zeros((nq, STATS_PER_QUERY), dtype=np.uint64) if with_stats else None)


class CsrLists(collections.namedtuple("CsrLists", ["offsets", "ids"])):
    """The candidate lists of nq queries in CSR form: query q's list is ids[offsets[q]:offsets[q + 1]] (offsets: nq + 1
    values, offsets[0] == 0, non-decreasing).  A plain tuple of arrays is a sequence of per-query lists, never this."""


def _candidate_lists(candidates, nq, id_dtype):
    """(offsets u64 [nq + 1], ids) of the candidate lists of nq queries: a sequence of nq 1-D integer arrays, or a
    CsrLists.  Ids must be non-negative and fit id_dtype, and a CsrLists' ids must hold offsets[-1] of them; the
    library checks the offsets' shape and the ids against the index."""
    if isinstance(candidates, CsrLists):
        offsets, ids = np.asarray(candidates.offsets), np.asarray(candidates.ids)
        if offsets.ndim != 1 or offsets.shape[0] != nq + 1:
            raise ValueError("offsets must have shape (nq + 1,)")
        if ids.ndim != 1:
            raise ValueError("ids must be 1-D")
        if offsets.dtype.kind in "iu" and int(offsets[-1]) > ids.shape[0]:
            # the library reads offsets[-1] ids from the buffer: more than it holds is out of bounds
            raise ValueError("offsets[-1] = %d exceeds the %d ids given" % (int(offsets[-1]), ids.shape[0]))
    else:
        lists = [np.asarray(c) for c in candidates]
        lists = [c.astype(id_dtype) if c.size == 0 else c for c in lists]  # an empty Python list is float64
        if len(lists) != nq:
            raise ValueError("one candidate list per query: got %d lists for %d queries" % (len(lists), nq))
        if any(c.ndim != 1 for c in lists):
            raise ValueError("each candidate list must be 1-D")
        offsets = np.zeros(nq + 1, dtype=np.uint64)
        np.cumsum([c.shape[0] for c in lists], out=offsets[1:])
        ids = np.concatenate(lists) if lists else np.zeros(0, dtype=id_dtype)
    for a, what in ((offsets, "offsets"), (ids, "ids")):
        if a.size and a.dtype.kind not in "iu":
            raise ValueError("%s must be integers" % what)
        if a.size and a.dtype.kind == "i" and a.min() < 0:
            raise ValueError("%s must be non-negative" % what)
    if ids.size and int(ids.max()) > np.iinfo(id_dtype).max:
        raise ValueError("ids must fit %s" % np.dtype(id_dtype).name)
    return (np.ascontiguousarray(offsets, dtype=np.uint64), np.ascontiguousarray(ids, dtype=id_dtype))


def _filter_words(filters, n):
    """The packed bitmaps (uint32 [F, W], C-contiguous) of a filtered search over ids [0, n): a bool mask of shape (n,)
    or (F, n), packed LSB first (id i is bit i % 32 of word i // 32), or uint32 words of shape (F, W) with
    W >= ceil(n / 32), passed as they are."""
    f = np.asarray(filters)
    if f.dtype == np.bool_:
        if f.ndim == 1:
            f = f[None, :]
        if f.ndim != 2 or f.shape[1] != n:
            raise ValueError("a bool filter mask must have shape (%d,) or (F, %d)" % (n, n))
        w = (n + 31) // 32
        b = np.zeros((f.shape[0], 4 * w), dtype=np.uint8)
        b[:, :(n + 7) // 8] = np.packbits(f, axis=1, bitorder="little")
        words = b.view("<u4").astype(np.uint32, copy=False)
    elif f.dtype == np.uint32:
        if f.ndim != 2:
            raise ValueError("filter words must have shape (F, W)")
        if f.shape[1] < (n + 31) // 32:
            raise ValueError("filter words: W = %d is less than ceil(%d / 32) = %d" % (f.shape[1], n, (n + 31) // 32))
        words = f
    else:
        raise ValueError("filters must be a bool mask or uint32 words, not %s" % f.dtype)
    if words.shape[0] == 0:
        raise ValueError("filters must hold at least one filter")
    return np.ascontiguousarray(words)


def _query_filter(query_filter, nq):
    """query_filter as uint32 [nq] (the library checks each entry against the number of filters), or None."""
    if query_filter is None:
        return None
    qf = np.asarray(query_filter)
    if qf.ndim != 1 or qf.shape[0] != nq:
        raise ValueError("query_filter must have shape (nq,) = (%d,)" % nq)
    if qf.size and qf.dtype.kind not in "iu":
        raise ValueError("query_filter must be integers")
    if qf.size and (qf.min() < 0 or int(qf.max()) > 0xFFFFFFFF):
        raise ValueError("query_filter entries must be non-negative and fit uint32")
    return np.ascontiguousarray(qf, dtype=np.uint32)


def _check_device_filters(filters, query_filter, q):
    """The filters (int32 [F, W]) and query_filter (int32 [nq] or None) of a device call for the queries q: contiguous
    CUDA tensors on the queries' device, since the kernels index them directly."""
    import torch

    for t, shape, what in ((filters, None, "filters"), (query_filter, (q.shape[0],), "query_filter")):
        if t is None and what == "query_filter":
            continue
        if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != q.device or t.dtype != torch.int32
                or not t.is_contiguous() or (shape is None and t.dim() != 2)
                or (shape is not None and tuple(t.shape) != shape)):
            raise ValueError("%s must be a contiguous int32 CUDA tensor of shape %s on the queries' device"
                             % (what, "(F, W)" if shape is None else "(nq,)"))


def _radius(radius):
    """The radius of a range call as the library takes it: a real number, rounded to float32 (NaN is the library's to
    reject)."""
    if isinstance(radius, (bool, np.bool_)) or not isinstance(radius, (int, float, np.integer, np.floating)):
        raise ValueError("radius must be a real number, not %r" % (radius,))
    return float(np.float32(radius))


def _csr_offsets(counts):
    """The offsets (uint64 [nq + 1]) of a range search's output: the exclusive prefix sum of its counts."""
    offsets = np.zeros(counts.shape[0] + 1, dtype=np.uint64)
    np.cumsum(counts, out=offsets[1:])
    return offsets


def _device_outputs(q, k, out):
    """The (ids, dists, counts) tensors of a device call for the queries q: `out` checked, or fresh ones."""
    import torch

    nq = q.shape[0]
    if out is None:
        return (torch.empty((nq, k), dtype=torch.int32, device=q.device),
                torch.empty((nq, k), dtype=torch.float32, device=q.device),
                torch.empty((nq,), dtype=torch.int32, device=q.device))
    for t, dt, shape in zip(out, (torch.int32, torch.float32, torch.int32), ((nq, k), (nq, k), (nq,))):
        if (not t.is_cuda or t.device != q.device or t.dtype != dt or tuple(t.shape) != shape
                or not t.is_contiguous()):
            raise ValueError("out tensors must be contiguous (ids int32 [nq,k], dists float32 [nq,k], counts "
                             "int32 [nq]) on the queries' device")
    return out


def _raw_stream(stream, device):
    """The raw cudaStream_t of `stream`, a torch.cuda.Stream or a raw pointer; None: torch's current stream on
    `device`."""
    if stream is None:
        import torch

        stream = torch.cuda.current_stream(device)
    return getattr(stream, "cuda_stream", stream)


class Granne:
    """granne.Granne (py/src/lib.rs:149-344) on the GPU.

    Granne(index_path, element_type, elements_path, embeddings_path=None, words_path=None, device=0)
    element_type: "angular" | "angular_int" | "embeddings".  With `words_path` an "embeddings" index also takes string
    queries and reports elements as words (WordEmbeddingsGranne, py/src/variants/index.rs:41-139); the lookup and the
    ordered row sum happen on the host, the search itself on the GPU.
    """

    def __init__(self, index_path, element_type, elements_path, embeddings_path=None, words_path=None, device=0):
        L = load_library()
        h = C.c_void_p()
        kind = _kind(element_type)
        if kind == EMBEDDINGS and embeddings_path is None:
            raise ValueError("embeddings_path required for this element type!")
        _check(L.granne_b200_open_files(os.fsencode(index_path), kind, os.fsencode(elements_path),
                                        os.fsencode(embeddings_path) if embeddings_path else None, device,
                                        C.byref(h)))
        self._h = h
        self.device = device
        self._elements_src = ("path", elements_path)
        self._embeddings_src = ("path", embeddings_path) if embeddings_path else None
        self._words_path = words_path

    @classmethod
    def from_bytes(cls, index_bytes, element_type, elements_bytes, embeddings_bytes=None, device=0):
        """Granne::from_bytes (src/index/mod.rs:108-113) + Vectors::from_bytes / SumEmbeddings::from_bytes."""
        L = load_library()
        self = cls.__new__(cls)
        h = C.c_void_p()
        ib = np.frombuffer(index_bytes, dtype=np.uint8)
        eb = np.frombuffer(elements_bytes, dtype=np.uint8)
        mb = np.frombuffer(embeddings_bytes, dtype=np.uint8) if embeddings_bytes is not None else None
        _check(L.granne_b200_open(_ptr(ib), ib.size, _kind(element_type), _ptr(eb), eb.size,
                                  _ptr(mb) if mb is not None else None, mb.size if mb is not None else 0, device,
                                  C.byref(h)))
        self._h = h
        self.device = device
        self._elements_src = ("bytes", elements_bytes)
        self._embeddings_src = ("bytes", embeddings_bytes) if embeddings_bytes is not None else None
        return self

    @classmethod
    def from_device_elements(cls, index_bytes, element_type, elements, device=None):
        """Granne::from_bytes with a device-resident element container: `elements` is a contiguous CUDA torch tensor
        [n, dim] of ELEMENTS (normalised float32 for "angular", int8 for "angular_int") on the target device — e.g.
        the output of elements_from_raw_device.  Nothing bounces through the host (100M x 128 f32 = 51 GB)."""
        L = load_library()
        kind = _kind(element_type)
        _check_device_rows(kind, elements)
        device = elements.device.index if device is None else device
        if elements.device.index != device:
            raise ValueError("elements tensor lives on cuda:%d, not cuda:%d" % (elements.device.index, device))
        self = cls.__new__(cls)
        h = C.c_void_p()
        ib = np.frombuffer(index_bytes, dtype=np.uint8)
        _check(L.granne_b200_open_device_elements(_ptr(ib), ib.size, kind, C.c_void_p(elements.data_ptr()),
                                                  elements.shape[0], elements.shape[1], device, C.byref(h)))
        self._h = h
        self.device = device
        self._elements_src = None
        self._embeddings_src = None
        return self

    @staticmethod
    def _source_bytes(src):
        if src is None:
            raise GranneError(-1, "this handle does not own a host image of that data")
        kind, value = src
        if kind == "path":
            with open(value, "rb") as f:
                return f.read()
        return bytes(value)

    def index_bytes(self):
        """Index::write_index (src/index/io.rs:11-70) into memory, from the staged graph."""
        return _write_index(load_library().granne_b200_write_index, self._h,
                            [self.layer_len(l) for l in range(self.num_layers())]).tobytes()

    def elements_bytes(self):
        """The elements file image (u64 dim + rows, src/slice_vector/mod.rs:460-466; offsets + 3-byte ids for
        "embeddings")."""
        return self._source_bytes(getattr(self, "_elements_src", None))

    def save_index(self, path):
        """Granne.save_index(path) (py/src/lib.rs:325-329)."""
        with open(path, "wb") as f:
            f.write(self.index_bytes())

    def save_elements(self, path):
        """Granne.save_elements(path) (py/src/lib.rs:339-343)."""
        with open(path, "wb") as f:
            f.write(self.elements_bytes())

    # ---- reorder (src/index/reorder.rs) ----
    def compute_order(self):
        """Granne::compute_order (reorder.rs:126-174) on the GPU: order[i] == j moves element j to position i."""
        order = np.zeros(len(self), dtype=np.uint64)
        _check(load_library().granne_b200_compute_order(self._h, _ptr(order), order.size))
        return order

    def _reopen_reordered(self, order):
        kind = self.element_kind
        index_bytes = self.index_bytes()
        elements_bytes = self._source_bytes(getattr(self, "_elements_src", None))
        new_index, new_elements = apply_order(index_bytes, kind, elements_bytes, order)
        emb = getattr(self, "_embeddings_src", None)
        emb_bytes = self._source_bytes(emb) if emb is not None else None
        fresh = Granne.from_bytes(new_index, kind, new_elements, emb_bytes, device=self.device)
        fresh._words_path = getattr(self, "_words_path", None)
        self.close()
        self._words = None
        self.__dict__.update(fresh.__dict__)
        fresh._h = None
        return [int(x) for x in order]

    def reorder(self, show_progress=False):
        """Granne.reorder(show_progress) (py/src/lib.rs:311-315, reorder.rs:59-82): reorders index and elements in
        place for locality; returns the permutation (new -> old).  "embeddings" indexes are reordered by
        compute_keys_for_reordering like the reference's Python class (py/src/variants/index.rs:70-75)."""
        if self.element_kind == EMBEDDINGS:
            keys = compute_keys_for_reordering(self._source_bytes(self._elements_src),
                                               self._source_bytes(self._embeddings_src))
            return self.reorder_by_keys(keys)
        return self._reopen_reordered(self.compute_order())

    def reorder_by_keys(self, keys, show_progress=False):
        """Granne::reorder_by_keys (reorder.rs:89-124): layer-preserving sort by `keys` (uint64 [n] or [n, kw])."""
        return self._reopen_reordered(order_by_keys(self.index_bytes(), keys))

    def close(self):
        if getattr(self, "_h", None):
            load_library().granne_b200_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- Index trait ----
    def __len__(self):
        return int(load_library().granne_b200_len(self._h))

    def num_layers(self):
        return int(load_library().granne_b200_num_layers(self._h))

    def layer_len(self, layer):
        return int(load_library().granne_b200_layer_len(self._h, layer))

    def get_neighbors(self, idx, layer=None):
        if layer is None:
            layer = self.num_layers() - 1  # py/src/lib.rs:268-276
        out = np.empty(256, dtype=np.uint32)
        n = C.c_size_t()
        _check(load_library().granne_b200_get_neighbors(self._h, idx, layer, _ptr(out), out.size, C.byref(n)))
        return out[:n.value].tolist()

    # ---- ElementContainer ----
    @property
    def dim(self):
        return int(load_library().granne_b200_dim(self._h))

    @property
    def element_kind(self):
        return int(load_library().granne_b200_element_kind(self._h))

    def num_elements(self):
        return int(load_library().granne_b200_num_elements(self._h))

    def get_element(self, idx):
        out = np.empty(self.dim, dtype=np.int8 if self.element_kind == ANGULAR_INT else np.float32)
        _check(load_library().granne_b200_get_element(self._h, idx, _ptr(out)))
        return out

    def get_elements(self, ids):
        """get_element for a 1-D integer array of ids in one launch: (n, dim) float32 (int8 for angular_int), row i
        bit for bit get_element(ids[i]).  Every id must be < num_elements()."""
        q, _ = _id_queries(ids, False, np.uint32)
        out = np.empty((q.shape[0], self.dim), dtype=np.int8 if self.element_kind == ANGULAR_INT else np.float32)
        _check(load_library().granne_b200_get_elements(self._h, _ptr(q), q.shape[0], _ptr(out)))
        return out

    def get_elements_device(self, ids, out=None, stream=None):
        """Device-resident get_elements: `ids` a contiguous 1-D int32 CUDA tensor (the u32 ids' bits) on this index's
        device; returns (n, dim) float32 (int8 for angular_int) CUDA rows, asynchronous on `stream`.  A bad id's row
        is zeros and stream_status() raises."""
        import torch

        q, _ = self._device_queries(ids, False, by_id=True)
        dt = torch.int8 if self.element_kind == ANGULAR_INT else torch.float32
        if out is None:
            out = torch.empty((q.shape[0], self.dim), dtype=dt, device=q.device)
        elif (not isinstance(out, torch.Tensor) or out.device != q.device or out.dtype != dt
              or tuple(out.shape) != (q.shape[0], self.dim) or not out.is_contiguous()):
            raise ValueError("out must be a contiguous %s CUDA tensor of shape (n, dim) on the ids' device" % dt)
        _check(load_library().granne_b200_get_elements_device(self._h, C.c_void_p(q.data_ptr()), q.shape[0],
                                                              C.c_void_p(out.data_ptr()),
                                                              C.c_void_p(_raw_stream(stream, q.device))))
        return out

    def knn_graph(self, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS, exclude_self=True,
                  exact=False, chunk=65536, out="host"):
        """The k-nearest-neighbour graph of the index: for every element i < len(self), search_batch(by_id) of i (or
        exact_search_batch with exact=True), without i itself when exclude_self.  The ids stream through the device
        calls in chunks made on the device, so no id array of length len(self) exists on the host.  The calls run on a
        stream of their own, and only their errors are reported (stream_status(stream)): other threads' device calls
        on this handle keep theirs.  Returns (ids, dists, counts) of shape [len, k]: uint32 / float32 / uint32 numpy
        arrays (out="host") or int32 / float32 / int32 CUDA tensors (out="device")."""
        import torch

        if out not in ("host", "device"):
            raise ValueError('out must be "host" or "device"')
        if int(chunk) < 1:
            raise ValueError("chunk must be >= 1")
        n, k, dev = len(self), int(num_elements), torch.device("cuda", self.device)
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        try:
            with torch.cuda.stream(s):
                ids = torch.empty((n, k), dtype=torch.int32, device=dev)
                dists = torch.empty((n, k), dtype=torch.float32, device=dev)
                counts = torch.empty((n,), dtype=torch.int32, device=dev)
                for c0 in range(0, n, int(chunk)):
                    c1 = min(n, c0 + int(chunk))
                    q = torch.arange(c0, c1, dtype=torch.int64, device=dev).to(torch.int32)  # the u32 ids' bits
                    part = (ids[c0:c1], dists[c0:c1], counts[c0:c1])
                    if exact:
                        self.exact_search_batch_device(q, k, by_id=True, exclude_self=exclude_self, out=part, stream=s)
                    else:
                        self.search_batch_device(q, max_search, k, by_id=True, exclude_self=exclude_self, out=part,
                                                 stream=s)
            self.stream_status(s)  # synchronises s and raises what any chunk reported
        finally:
            self.release_stream(s)
        if out == "device":
            return ids, dists, counts
        return ids.cpu().numpy().view(np.uint32), dists.cpu().numpy(), counts.cpu().numpy().view(np.uint32)

    # ---- search ----
    def search_batch(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                     already_element=False, with_stats=False, by_id=False, exclude_self=False):
        """nq independent Granne::search calls (src/index/mod.rs:140-150) in one launch; host buffers in and out.

        queries: (nq, dim) float32 raw vectors (normalised / quantised by the library like the reference's Python
        binding), or with already_element=True rows that already are elements (normalised f32; int8 for
        angular_int).  With by_id=True, a 1-D integer array of element ids < num_elements(): the query of row q is
        get_element(ids[q]), with results bit-identical to passing those rows as elements; exclude_self=True (which
        implies by_id) searches k + 1 and drops each query's own id.  The other query calls take the same keywords.
        Returns (ids uint32 [nq,k] padded 0xFFFFFFFF, dists float32 [nq,k] padded +inf, counts)."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, stats = _host_outputs(nq, k, np.uint32, with_stats)
        _check(load_library().granne_b200_search_batch(self._h, _ptr(q), nq, fmt, int(max_search), k, _ptr(ids),
                                                       _ptr(dists), _ptr(counts),
                                                       _ptr(stats) if with_stats else None))
        if with_stats:
            return ids, dists, counts, stats
        return ids, dists, counts

    def _host_queries(self, queries, already_element, by_id=False, exclude_self=False):
        """_host_queries for this index: its width, and its rules on int8 rows; element ids with by_id or
        exclude_self."""
        if by_id or exclude_self:
            return _id_queries(queries, exclude_self, np.uint32)
        q = np.asarray(queries)
        if q.dtype == np.int8:
            if self.element_kind != ANGULAR_INT:
                raise ValueError("int8 queries need an angular_int index")
        elif already_element and self.element_kind == ANGULAR_INT:
            raise ValueError("angular_int elements are int8")
        return _host_queries(q, already_element, self.dim)

    def exact_search_batch(self, queries, num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, by_id=False,
                           exclude_self=False):
        """Exact k nearest neighbours: the first min(k, len(self)) of all elements i < len(self) by (distance, id),
        with the reference's distance bit for bit (granne_b200_exact_search_batch) — the ground truth of recall.
        Not a reference function.  Queries as in search_batch; k <= EXACT_MAX_K.  Returns (ids, dists, counts) in
        search_batch's layout."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint32)
        _check(load_library().granne_b200_exact_search_batch(self._h, _ptr(q), nq, fmt, k, _ptr(ids), _ptr(dists),
                                                             _ptr(counts)))
        return ids, dists, counts

    def exact_search_batch_device(self, queries, num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, out=None,
                                  stream=None, by_id=False, exclude_self=False):
        """Device-resident exact_search_batch: CUDA tensors in and out, asynchronous on `stream` (a torch.cuda.Stream
        or a raw cudaStream_t; default: the current torch stream); a NaN distance is reported by stream_status()."""
        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts = _device_outputs(q, k, out)
        _check(load_library().granne_b200_exact_search_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, k, C.c_void_p(ids.data_ptr()), C.c_void_p(dists.data_ptr()),
            C.c_void_p(counts.data_ptr()), C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    def exact_search_within(self, queries, candidates, num_elements=DEFAULT_NUM_ELEMENTS, already_element=False,
                            by_id=False, exclude_self=False):
        """Exact k nearest neighbours of each query within its own candidate list: the first min(k, |set(list)|) ids
        of the list by (distance, id), with the reference's distance bit for bit (granne_b200_exact_search_within_batch).
        Not a reference function.  `candidates`: one 1-D integer array of ids per query, or a CsrLists(offsets, ids)
        (offsets [nq + 1], offsets[0] == 0, non-decreasing).  Duplicates count once; every id must be
        < len(self).  Queries as in exact_search_batch; k <= EXACT_MAX_K.  Returns (ids, dists, counts) in
        search_batch's layout."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        offsets, cand = _candidate_lists(candidates, nq, np.uint32)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint32)
        _check(load_library().granne_b200_exact_search_within_batch(
            self._h, _ptr(q), nq, fmt, _ptr(offsets), _ptr(cand), k, _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_search_within_device(self, queries, offsets, ids, num_elements=DEFAULT_NUM_ELEMENTS,
                                   already_element=False, out=None, stream=None, by_id=False, exclude_self=False):
        """Device-resident exact_search_within: CUDA tensors in (queries; offsets int64 [nq + 1]; ids int32 view of
        u32 ids) and out, asynchronous on `stream` (a torch.cuda.Stream or a raw cudaStream_t; default: the current
        torch stream).  The kernels check the lists: a bad list gives its query count 0 and padding, and
        stream_status() raises; so does a NaN distance.  `ids` must hold offsets[-1] ids: the kernels read that many,
        and checking it here would wait for the device."""
        import torch

        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        for t, dt, what in ((offsets, torch.int64, "offsets"), (ids, torch.int32, "ids")):
            if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != q.device or t.dtype != dt
                    or t.dim() != 1 or not t.is_contiguous()):
                raise ValueError("%s must be a contiguous 1-D %s CUDA tensor on the queries' device" % (what, dt))
        if offsets.shape[0] != nq + 1:
            raise ValueError("offsets must have shape (nq + 1,)")
        out_ids, dists, counts = _device_outputs(q, k, out)
        _check(load_library().granne_b200_exact_search_within_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, C.c_void_p(offsets.data_ptr()), C.c_void_p(ids.data_ptr()),
            k, C.c_void_p(out_ids.data_ptr()), C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(_raw_stream(stream, q.device))))
        return out_ids, dists, counts

    # ---- two-stage search (granne_b200_search_rerank_batch*) ----
    # ---- exact range search ----
    def exact_range_count(self, queries, radius, already_element=False, by_id=False, exclude_self=False):
        """|R(q)| of every query: the number of elements i < len(self) whose distance is <= radius (rounded to float32;
        IEEE <=, so +inf counts every element), with exact_search_batch's distances bit for bit
        (granne_b200_exact_range_count).  Not a reference function.  Queries as in search_batch; exclude_self leaves
        the query's own id out.  Returns uint64 [nq]."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        counts = np.empty(q.shape[0], dtype=np.uint64)
        _check(load_library().granne_b200_exact_range_count(self._h, _ptr(q), q.shape[0], fmt, _radius(radius),
                                                            _ptr(counts)))
        return counts

    def exact_range_search(self, queries, radius, already_element=False, by_id=False, exclude_self=False):
        """Every element within radius of each query, sorted by (distance, id), with no cap on their number: the
        count, its prefix sum, then the fill (granne_b200_exact_range_search), i.e. two exact scans.  Returns
        (offsets uint64 [nq + 1], ids uint32, dists float32): query q's entries are ids[offsets[q]:offsets[q + 1]]."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        r = _radius(radius)
        offsets = _csr_offsets(self.exact_range_count(q, r, already_element=fmt == QUERY_ELEMENT, by_id=by_id,
                                                      exclude_self=exclude_self))
        ids = np.empty(int(offsets[-1]), dtype=np.uint32)
        dists = np.empty(int(offsets[-1]), dtype=np.float32)
        _check(load_library().granne_b200_exact_range_search(self._h, _ptr(q), q.shape[0], fmt, r, _ptr(offsets),
                                                             _ptr(ids), _ptr(dists)))
        return offsets, ids, dists

    def exact_range_count_device(self, queries, radius, already_element=False, out=None, stream=None, by_id=False,
                                 exclude_self=False):
        """Device-resident exact_range_count: CUDA tensors in, int64 [nq] counts out (the u64 counts' bits),
        asynchronous on `stream` (a torch.cuda.Stream or a raw cudaStream_t; default: the current torch stream).  A
        bad id counts 0 and, like a NaN distance, is raised by stream_status()."""
        import torch

        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq = q.shape[0]
        if out is None:
            out = torch.empty((nq,), dtype=torch.int64, device=q.device)
        elif (not isinstance(out, torch.Tensor) or out.device != q.device or out.dtype != torch.int64
              or tuple(out.shape) != (nq,) or not out.is_contiguous()):
            raise ValueError("out must be a contiguous int64 [nq] CUDA tensor on the queries' device")
        _check(load_library().granne_b200_exact_range_count_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, _radius(radius), C.c_void_p(out.data_ptr()),
            C.c_void_p(_raw_stream(stream, q.device))))
        return out

    def exact_range_search_device(self, queries, radius, offsets, out=None, stream=None, already_element=False,
                                  by_id=False, exclude_self=False):
        """Device-resident fill of exact_range_search: `offsets` an int64 [nq + 1] CUDA tensor (normally the prefix
        sum of exact_range_count_device's counts), `out` (ids int32, dists float32) of offsets[-1] entries.  With
        out=None the outputs are sized from offsets[-1], which waits for the device; a caller that keeps its work
        asynchronous passes `out`.  A segment whose length differs from its query's count is padded and raised by
        stream_status().  Returns (ids, dists)."""
        import torch

        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq = q.shape[0]
        if (not isinstance(offsets, torch.Tensor) or offsets.device != q.device or offsets.dtype != torch.int64
                or tuple(offsets.shape) != (nq + 1,) or not offsets.is_contiguous()):
            raise ValueError("offsets must be a contiguous int64 [nq + 1] CUDA tensor on the queries' device")
        if out is None:
            total = int(offsets[-1])
            out = (torch.empty((total,), dtype=torch.int32, device=q.device),
                   torch.empty((total,), dtype=torch.float32, device=q.device))
        for t, dt in zip(out, (torch.int32, torch.float32)):
            if (not isinstance(t, torch.Tensor) or t.device != q.device or t.dtype != dt or t.dim() != 1
                    or not t.is_contiguous()):
                raise ValueError("out must be contiguous 1-D CUDA tensors (ids int32, dists float32) on the queries' "
                                 "device")
        _check(load_library().granne_b200_exact_range_search_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, _radius(radius), C.c_void_p(offsets.data_ptr()),
            C.c_void_p(out[0].data_ptr()), C.c_void_p(out[1].data_ptr()), C.c_void_p(_raw_stream(stream, q.device))))
        return out

    def range_graph(self, radius, exclude_self=True, chunk=65536, out="host"):
        """The exact range graph of the index (near duplicates at a small radius): for every element i < len(self),
        every element within radius of i, sorted by (distance, id), without i itself when exclude_self.  The ids
        stream through the device calls in chunks made on the device, on a stream of its own whose errors alone are
        reported (as knn_graph).  It computes len(self)^2 distances twice (count, then fill): O(n^2) work.  Returns
        CSR (offsets [len + 1], ids, dists): uint64 / uint32 / float32 numpy arrays (out="host") or int64 / int32 /
        float32 CUDA tensors (out="device")."""
        import torch

        if out not in ("host", "device"):
            raise ValueError('out must be "host" or "device"')
        if int(chunk) < 1:
            raise ValueError("chunk must be >= 1")
        r, n, step, dev = _radius(radius), len(self), int(chunk), torch.device("cuda", self.device)
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.current_stream(dev))

        def ids_of(c0, c1):
            return torch.arange(c0, c1, dtype=torch.int64, device=dev).to(torch.int32)  # the u32 ids' bits

        try:
            with torch.cuda.stream(s):
                counts = torch.empty((n,), dtype=torch.int64, device=dev)
                for c0 in range(0, n, step):
                    c1 = min(n, c0 + step)
                    self.exact_range_count_device(ids_of(c0, c1), r, by_id=True, exclude_self=exclude_self,
                                                  out=counts[c0:c1], stream=s)
                offsets = torch.zeros((n + 1,), dtype=torch.int64, device=dev)
                torch.cumsum(counts, 0, out=offsets[1:])
                host_off = offsets.cpu()  # sizes the output: waits for the counts
                total = int(host_off[-1])
                ids = torch.empty((total,), dtype=torch.int32, device=dev)
                dists = torch.empty((total,), dtype=torch.float32, device=dev)
                for c0 in range(0, n, step):
                    c1 = min(n, c0 + step)
                    b, e = int(host_off[c0]), int(host_off[c1])
                    self.exact_range_search_device(ids_of(c0, c1), r, offsets[c0:c1 + 1] - b, out=(ids[b:e], dists[b:e]),
                                                   by_id=True, exclude_self=exclude_self, stream=s)
            self.stream_status(s)  # synchronises s and raises what any chunk reported
        finally:
            self.release_stream(s)
        if out == "device":
            return offsets, ids, dists
        return offsets.cpu().numpy().view(np.uint64), ids.cpu().numpy().view(np.uint32), dists.cpu().numpy()

    def search_batch_filtered(self, queries, filters, query_filter=None, max_search=DEFAULT_MAX_SEARCH,
                              num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, with_stats=False, by_id=False,
                              exclude_self=False):
        """Filtered search (granne_b200_search_filtered_batch): search_batch's traversal, unchanged, returning the first
        k admitted elements among those it scores in the bottom layer, by (distance, id).  Not a reference function.
        `filters`: a bool mask of shape (len,) or (F, len), or packed uint32 words (F, W), W >= ceil(len / 32) (id i
        is bit i % 32 of word i // 32); query_filter: one filter index per query (None: filter 0 for all).  k <=
        EXACT_MAX_K and may exceed max_search; no exact fallback, so a selective filter may return fewer than k
        (exact_search_filtered returns the exact answer over the same filters).
        Returns search_batch's (ids, dists, counts[, stats]); stats columns 0..2 equal search_batch's."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        words = _filter_words(filters, len(self))
        qf = _query_filter(query_filter, nq)
        ids, dists, counts, stats = _host_outputs(nq, k, np.uint32, with_stats)
        _check(load_library().granne_b200_search_filtered_batch(
            self._h, _ptr(q), nq, fmt, int(max_search), k, _ptr(words), words.shape[0], words.shape[1],
            _ptr(qf) if qf is not None else None, _ptr(ids), _ptr(dists), _ptr(counts),
            _ptr(stats) if with_stats else None))
        if with_stats:
            return ids, dists, counts, stats
        return ids, dists, counts

    def search_batch_filtered_device(self, queries, filters, query_filter=None, max_search=DEFAULT_MAX_SEARCH,
                                     num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, out=None, stats=None,
                                     stream=None, by_id=False, exclude_self=False):
        """Device-resident search_batch_filtered: CUDA tensors in (queries; filters int32 [F, W] holding the uint32
        words; query_filter int32 [nq] or None) and out, asynchronous on `stream` like search_batch_device.  The kernel
        checks query_filter: an entry >= F gives its query count 0 and padding, and stream_status() raises."""
        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        _check_device_filters(filters, query_filter, q)
        ids, dists, counts = _device_outputs(q, k, out)
        _check_stats(stats, q)
        _check(load_library().granne_b200_search_filtered_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, int(max_search), k, C.c_void_p(filters.data_ptr()),
            filters.shape[0], filters.shape[1],
            C.c_void_p(query_filter.data_ptr()) if query_filter is not None else None, C.c_void_p(ids.data_ptr()),
            C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(stats.data_ptr()) if stats is not None else None, C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    def exact_search_filtered(self, queries, filters, query_filter=None, num_elements=DEFAULT_NUM_ELEMENTS,
                              already_element=False, by_id=False, exclude_self=False):
        """Exact filtered k nearest neighbours (granne_b200_exact_search_filtered_batch): for each query the first
        min(k, |A|) of the elements i < len(self) its filter admits, by (distance, id), with exact_search_batch's
        distances bit for bit.  Not a reference function.  `filters` and `query_filter` as in search_batch_filtered;
        queries as in exact_search_batch (exclude_self drops the query's own id when its filter admits it); k <=
        EXACT_MAX_K.  Only admitted rows are scanned: a chunk of 1024 queries costs the rows its filters' union admits,
        so queries that share a filter are best passed next to each other.  Returns (ids, dists, counts) in
        search_batch's layout."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        words = _filter_words(filters, len(self))
        qf = _query_filter(query_filter, nq)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint32)
        _check(load_library().granne_b200_exact_search_filtered_batch(
            self._h, _ptr(q), nq, fmt, _ptr(words), words.shape[0], words.shape[1],
            _ptr(qf) if qf is not None else None, k, _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_search_filtered_device(self, queries, filters, query_filter=None, num_elements=DEFAULT_NUM_ELEMENTS,
                                     already_element=False, out=None, stream=None, by_id=False, exclude_self=False):
        """Device-resident exact_search_filtered: CUDA tensors in (queries; filters int32 [F, W] holding the uint32
        words; query_filter int32 [nq] or None) and out, asynchronous on `stream` like exact_search_batch_device and
        without waiting for the device.  The kernels check query_filter: an entry >= F gives its query count 0 and
        padding, and stream_status() raises; so does a NaN distance to an admitted element."""
        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        _check_device_filters(filters, query_filter, q)
        ids, dists, counts = _device_outputs(q, k, out)
        _check(load_library().granne_b200_exact_search_filtered_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, C.c_void_p(filters.data_ptr()), filters.shape[0],
            filters.shape[1], C.c_void_p(query_filter.data_ptr()) if query_filter is not None else None, k,
            C.c_void_p(ids.data_ptr()), C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    def set_rerank_elements(self, elements):
        """Attaches the angular f32 rows (an angular elements file image, `bytes`) that re-rank the candidates of
        this angular_int index: at least len(self) rows of its width.  Once, before searching."""
        eb = np.frombuffer(elements, dtype=np.uint8)
        _check(load_library().granne_b200_set_rerank_elements(self._h, _ptr(eb), eb.size))

    def set_rerank_elements_device(self, elements):
        """set_rerank_elements from a contiguous CUDA float32 tensor [n, dim] of normalised rows on this index's
        device (e.g. elements_from_raw_device("angular", raw)); the rows are copied."""
        _check_device_rows(ANGULAR, elements)
        if elements.device.index != self.device:
            raise ValueError("elements tensor lives on cuda:%d, not cuda:%d" % (elements.device.index, self.device))
        _check(load_library().granne_b200_set_rerank_elements_device(self._h, C.c_void_p(elements.data_ptr()),
                                                                     elements.shape[0], elements.shape[1]))

    def set_rerank_embeddings(self, elements, embeddings, words_path=None):
        """Attaches the SumEmbeddings container (`bytes` images of its term lists and of its embedding table, as
        from_bytes takes them for an "embeddings" index) whose angular_int rows this index was built over
        (compute_embeddings): the candidates are re-ranked by their exact sum-of-embeddings distance.  At least
        len(self) elements, a table of the index's width (at most 4096).  Once, before searching; no other re-rank
        container may be attached.  With `words_path` (a words file of the table's rows), search_rerank also takes
        string queries."""
        eb = np.frombuffer(elements, dtype=np.uint8)
        mb = np.frombuffer(embeddings, dtype=np.uint8)
        _check(load_library().granne_b200_set_rerank_embeddings(self._h, _ptr(eb), eb.size, _ptr(mb), mb.size))
        if words_path is not None:
            from . import words as W

            self._rerank_words = (W.WordDict(words_path), W.read_dense_f32(embeddings))

    def search_batch_rerank(self, queries, num_candidates, max_search=DEFAULT_MAX_SEARCH,
                            num_elements=DEFAULT_NUM_ELEMENTS, with_stats=False):
        """Two-stage search: the first num_candidates results of search_batch on this angular_int index, re-ranked
        by their exact f32 angular distance to the query over the attached rows; the first num_elements by
        (distance, id).  Not a reference function.  queries: raw float32 (nq, dim).  Returns (ids, dists, counts)
        in search_batch's layout; with_stats adds stage 1's counters."""
        q = _raw_f32_queries(queries, self.dim)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, stats = _host_outputs(nq, k, np.uint32, with_stats)
        _check(load_library().granne_b200_search_rerank_batch(
            self._h, _ptr(q), nq, QUERY_RAW_F32, int(max_search), int(num_candidates), k, _ptr(ids), _ptr(dists),
            _ptr(counts), _ptr(stats) if with_stats else None))
        if with_stats:
            return ids, dists, counts, stats
        return ids, dists, counts

    def search_rerank(self, element, num_candidates, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS):
        """search_batch_rerank for one raw float32 query -> [(id, distance)], like search.  A str query, after
        set_rerank_embeddings(..., words_path=...), is the sum of its words' embeddings (create_embedding), as
        search builds it for an "embeddings" index (py/src/variants/index.rs:98-105)."""
        if isinstance(element, str):
            from . import words as W

            if getattr(self, "_rerank_words", None) is None:
                raise ValueError("string queries need set_rerank_embeddings(..., words_path=...)")
            words, table = self._rerank_words
            element = W.create_embedding(table, words.get_word_ids(element))
        ids, dists, counts = self.search_batch_rerank(np.asarray(element)[None, :], num_candidates, max_search,
                                                      num_elements)
        return [(int(ids[0, i]), float(dists[0, i])) for i in range(int(counts[0]))]

    def search_batch_rerank_device(self, queries, num_candidates, max_search=DEFAULT_MAX_SEARCH,
                                   num_elements=DEFAULT_NUM_ELEMENTS, out=None, stats=None, stream=None):
        """Device-resident search_batch_rerank: a CUDA float32 tensor in, CUDA tensors out (ids int32 view of u32
        bits, dists float32, counts int32), asynchronous on `stream` (a torch.cuda.Stream or a raw cudaStream_t;
        default: the current torch stream); a NaN distance is reported by stream_status()."""
        import torch

        q = self._check_device_queries(queries)
        if q.dtype != torch.float32:
            raise ValueError("the two-stage search takes raw float32 queries")
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts = _device_outputs(q, k, out)
        _check_stats(stats, q)
        _check(load_library().granne_b200_search_rerank_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, QUERY_RAW_F32, int(max_search), int(num_candidates), k,
            C.c_void_p(ids.data_ptr()), C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(stats.data_ptr()) if stats is not None else None, C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    # ---- diverse search (granne_b200_search_diverse_batch*, granne_b200_select_neighbors_batch*) ----
    def search_batch_diverse(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                             already_element=False, with_stats=False, by_id=False, exclude_self=False):
        """The neighbours granne would link each query to if it were inserted: search_batch(q, max_search,
        max_search) (without the element itself for exclude_self), then GranneBuilder::select_neighbors
        (src/index/mod.rs:849-883) keeps a candidate only if it is at least as close to the query as to every
        candidate kept before it, up to num_elements.  Not a reference function.  max_search <=
        DIVERSE_MAX_CANDIDATES; queries and keywords as in search_batch.  Returns (ids, dists, counts) in
        search_batch's layout, in candidate order with the search's distances; with_stats adds the search's
        counters."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, stats = _host_outputs(nq, k, np.uint32, with_stats)
        _check(load_library().granne_b200_search_diverse_batch(self._h, _ptr(q), nq, fmt, int(max_search), k,
                                                               _ptr(ids), _ptr(dists), _ptr(counts),
                                                               _ptr(stats) if with_stats else None))
        if with_stats:
            return ids, dists, counts, stats
        return ids, dists, counts

    def search_batch_diverse_device(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                                    already_element=False, out=None, stats=None, stream=None, by_id=False,
                                    exclude_self=False):
        """Device-resident search_batch_diverse: CUDA tensors in and out as in search_batch_device, asynchronous on
        `stream`; errors are raised by stream_status()."""
        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts = _device_outputs(q, k, out)
        _check_stats(stats, q)
        _check(load_library().granne_b200_search_diverse_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, int(max_search), k, C.c_void_p(ids.data_ptr()),
            C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(stats.data_ptr()) if stats is not None else None, C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    def select_neighbors(self, ids, dists, counts, num_elements=DEFAULT_NUM_ELEMENTS):
        """select_neighbors(list_q, num_elements) over caller lists, search_batch_diverse's selection: it composes with
        every query call's (ids, dists, counts) as they are (exact_search_batch(q, C) gives the exact diverse answer).
        ids uint32 [nq, C] (< len(self)), dists float32 [nq, C] ascending within each list's first counts[q] entries,
        counts [nq] <= C; C <= DIVERSE_MAX_CANDIDATES.  Returns (ids, dists, counts) in search_batch's layout."""
        ci = np.asarray(ids)
        if ci.ndim != 2:
            raise ValueError("ids must have shape (nq, C)")
        nq, stride = ci.shape
        ci = np.ascontiguousarray(ci, dtype=np.uint32)
        cd = np.ascontiguousarray(dists, dtype=np.float32)
        cc = np.ascontiguousarray(counts, dtype=np.uint32)
        if cd.shape != ci.shape or cc.shape != (nq,):
            raise ValueError("dists must have the shape of ids (nq, C), counts (nq,)")
        k = int(num_elements)
        out_ids, out_dists, out_counts, _ = _host_outputs(nq, k, np.uint32)
        _check(load_library().granne_b200_select_neighbors_batch(
            self._h, _ptr(ci), _ptr(cd), _ptr(cc), nq, stride, k, _ptr(out_ids), _ptr(out_dists), _ptr(out_counts)))
        return out_ids, out_dists, out_counts

    def select_neighbors_device(self, ids, dists, counts, num_elements=DEFAULT_NUM_ELEMENTS, out=None, stream=None):
        """Device-resident select_neighbors: the (ids int32 [nq, C], dists float32 [nq, C], counts int32 [nq]) CUDA
        tensors of any *_device call as they are, asynchronous on `stream`.  The kernel checks the lists: a bad list
        gets count 0 and padding, and stream_status() raises."""
        import torch

        for t, dt, what in ((ids, torch.int32, "ids"), (dists, torch.float32, "dists"), (counts, torch.int32, "counts")):
            if (not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device or t.dtype != dt
                    or not t.is_contiguous()):
                raise ValueError("%s must be a contiguous %s CUDA tensor on cuda:%d" % (what, dt, self.device))
        if ids.dim() != 2 or tuple(dists.shape) != tuple(ids.shape) or tuple(counts.shape) != (ids.shape[0],):
            raise ValueError("ids and dists must have shape (nq, C), counts (nq,)")
        nq, stride = ids.shape
        k = int(num_elements)
        out_ids, out_dists, out_counts = _device_outputs(ids, k, out)
        _check(load_library().granne_b200_select_neighbors_batch_device(
            self._h, C.c_void_p(ids.data_ptr()), C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()), nq,
            stride, k, C.c_void_p(out_ids.data_ptr()), C.c_void_p(out_dists.data_ptr()),
            C.c_void_p(out_counts.data_ptr()), C.c_void_p(_raw_stream(stream, ids.device))))
        return out_ids, out_dists, out_counts

    def _word_tables(self):
        """(WordDict, embeddings table, per-element id lists) for an "embeddings" index opened with words_path."""
        if getattr(self, "_words", None) is None:
            from . import words as W

            if self.element_kind != EMBEDDINGS or getattr(self, "_words_path", None) is None:
                raise ValueError("string queries need an \"embeddings\" index opened with words_path")
            self._words = (W.WordDict(self._words_path), W.read_dense_f32(self._source_bytes(self._embeddings_src)),
                           W.read_sum_terms(self._source_bytes(self._elements_src)))
        return self._words

    def get_internal_element(self, idx):
        """Granne.get_internal_element(idx) (py/src/lib.rs:255-257): the words of an "embeddings" element
        (py/src/variants/index.rs:133-138); the element itself for the vector types."""
        if self.element_kind != EMBEDDINGS:
            return self.get_element(idx)
        words, _, terms = self._word_tables()
        return words.get_words(terms[idx])

    def search(self, element, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS):
        """Granne.search(element, max_search=200, num_elements=10) -> [(id, distance)] (py/src/lib.rs:227-233); a str
        query is the sum of its words' embeddings (py/src/variants/index.rs:112-125)."""
        if isinstance(element, str):
            from . import words as W

            words, table, _ = self._word_tables()
            element = W.create_embedding(table, words.get_word_ids(element))
        ids, dists, counts = self.search_batch(np.asarray(element)[None, :], max_search, num_elements)
        return [(int(ids[0, i]), float(dists[0, i])) for i in range(int(counts[0]))]

    def search_batch_device(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                            already_element=False, out=None, stats=None, stream=None, by_id=False, exclude_self=False):
        """Device-resident variant: `queries` is a CUDA torch tensor on this index's device; returns CUDA tensors
        (ids int32 view of u32 bits, dists float32, counts int32).  Asynchronous on `stream` (a torch.cuda.Stream or a
        raw cudaStream_t; default: the current torch stream).  With by_id / exclude_self, `queries` is a contiguous
        1-D int32 tensor of element ids (the u32 bits); a query whose id is >= num_elements() gets count 0, padding
        and zero stats, and stream_status() raises."""
        q, fmt = self._device_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts = _device_outputs(q, k, out)
        _check_stats(stats, q)
        _check(load_library().granne_b200_search_batch_device(
            self._h, C.c_void_p(q.data_ptr()), nq, fmt, int(max_search), k, C.c_void_p(ids.data_ptr()),
            C.c_void_p(dists.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(stats.data_ptr()) if stats is not None else None, C.c_void_p(_raw_stream(stream, q.device))))
        return ids, dists, counts

    def search_batch_device_gather(self, queries, gather, max_search=DEFAULT_MAX_SEARCH,
                                   num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, counts=None, stats=None,
                                   stream=None):
        """Like search_batch_device, but the result rows are stored by the kernels straight into every peer's
        gathered buffer described by `gather` (a PeerGather).  stream: as for search_batch_device."""
        q, fmt = self._device_queries(queries, already_element)
        _check_stats(stats, q)
        _check(load_library().granne_b200_search_batch_device_gather(
            self._h, C.c_void_p(q.data_ptr()), q.shape[0], fmt, int(max_search), int(num_elements), C.byref(gather),
            C.c_void_p(counts.data_ptr()) if counts is not None else None,
            C.c_void_p(stats.data_ptr()) if stats is not None else None, C.c_void_p(_raw_stream(stream, q.device))))

    def _device_queries(self, queries, already_element, by_id=False, exclude_self=False):
        """(checked queries, query format) of a device call, as _host_queries gives them for a host call."""
        import torch

        if by_id or exclude_self:
            if (not isinstance(queries, torch.Tensor) or not queries.is_cuda or queries.device.index != self.device
                    or queries.dtype != torch.int32 or queries.dim() != 1 or not queries.is_contiguous()):
                raise ValueError("ids must be a contiguous 1-D int32 CUDA tensor (the u32 ids' bits) on cuda:%d"
                                 % self.device)
            return queries, QUERY_ID_EXCLUDING if exclude_self else QUERY_ID
        q = self._check_device_queries(queries)
        return q, QUERY_ELEMENT if already_element or q.dtype == torch.int8 else QUERY_RAW_F32

    def _check_device_queries(self, q):
        """Same checks as the host path (search_batch): a wrong dtype, width, device or a strided view would make the
        kernels read out of bounds (they index queries as qi * dim)."""
        import torch

        if not isinstance(q, torch.Tensor) or not q.is_cuda:
            raise ValueError("queries must be a CUDA torch tensor")
        if q.device.index != self.device:
            raise ValueError("queries live on cuda:%s, the index on cuda:%d" % (q.device.index, self.device))
        if q.dim() != 2 or q.shape[1] != self.dim:
            raise ValueError("queries must have shape (nq, %d)" % self.dim)
        if q.dtype == torch.int8:
            if self.element_kind != ANGULAR_INT:
                raise ValueError("int8 queries need an angular_int index")
        elif q.dtype != torch.float32:
            raise ValueError("queries must be float32 (or int8 elements for angular_int)")
        return q.contiguous()

    def stream_status(self, stream=None):
        """Raises the first error of the device calls issued since the previous check: of every stream of this handle
        (after synchronising the device), or, given `stream` (a torch.cuda.Stream or a raw cudaStream_t), of that
        stream's calls only, after synchronising it."""
        if stream is None:
            _check(load_library().granne_b200_stream_status(self._h))
        else:
            raw = getattr(stream, "cuda_stream", stream)
            _check(load_library().granne_b200_stream_status_of(self._h, C.c_void_p(raw)))

    def release_stream(self, stream):
        """Returns the workspace the library keeps for a caller stream (a raw cudaStream_t or a torch stream)."""
        raw = getattr(stream, "cuda_stream", stream)
        _check(load_library().granne_b200_release_stream(self._h, C.c_void_p(raw)))

    def launch_count(self):
        return int(load_library().granne_b200_launch_count(self._h))

    def device_bytes(self):
        return int(load_library().granne_b200_device_bytes(self._h))


MODE_REPLICATED, MODE_RANGE_PARTITIONED = 0, 1


class MultiGranne:
    """Several GPUs of THIS process behind one handle (granne_b200_multi_*): no torch, no NCCL.

    MultiGranne.replicated(index_bytes, element_type, elements_bytes, devices)       one index on every device,
                                                                                     query batches are sliced
    MultiGranne.partitioned([(index_bytes, elements_bytes), ...], element_type, devices)
                                                                                     one independent index per shard
    search_batch returns GLOBAL uint64 ids (0xFFFF_FFFF_FFFF_FFFF padded), float32 distances, counts."""

    def __init__(self, mode, shards, element_type, devices, embeddings_bytes=None):
        L = load_library()
        kind = _kind(element_type)
        n = len(shards)
        self._keep = [(np.frombuffer(i, dtype=np.uint8), np.frombuffer(e, dtype=np.uint8)) for i, e in shards]
        ip = (C.c_void_p * n)(*[a.ctypes.data for a, _ in self._keep])
        il = (C.c_size_t * n)(*[a.size for a, _ in self._keep])
        ep = (C.c_void_p * n)(*[b.ctypes.data for _, b in self._keep])
        el = (C.c_size_t * n)(*[b.size for _, b in self._keep])
        dv = (C.c_int * len(devices))(*[int(d) for d in devices])
        mb = np.frombuffer(embeddings_bytes, dtype=np.uint8) if embeddings_bytes is not None else None
        h = C.c_void_p()
        _check(L.granne_b200_multi_open(mode, dv, len(devices), kind, ip, il, ep, el, n,
                                        _ptr(mb) if mb is not None else None, mb.size if mb is not None else 0,
                                        C.byref(h)))
        self._h = h
        self._keep = None
        self.kind = kind
        self.mode = mode

    @classmethod
    def replicated(cls, index_bytes, element_type, elements_bytes, devices, embeddings_bytes=None):
        return cls(MODE_REPLICATED, [(index_bytes, elements_bytes)], element_type, devices, embeddings_bytes)

    @classmethod
    def partitioned(cls, shards, element_type, devices, embeddings_bytes=None):
        return cls(MODE_RANGE_PARTITIONED, shards, element_type, devices, embeddings_bytes)

    def __len__(self):
        return int(load_library().granne_b200_multi_len(self._h))

    def num_parts(self):
        return int(load_library().granne_b200_multi_num_parts(self._h))

    def shard_base(self, s):
        return int(load_library().granne_b200_multi_shard_base(self._h, s))

    def part_len(self, s):
        """Index::len of part s: its global ids are [shard_base(s), shard_base(s) + part_len(s))."""
        return int(load_library().granne_b200_multi_part_len(self._h, s))

    def global_ids(self):
        """The global ids of every indexed element, in order: [0, len) for a replicated handle, each shard's
        [shard_base, shard_base + part_len) for a partitioned one (equal to [0, len) when every shard's index covers
        its whole container)."""
        parts = [(0, len(self))] if self.mode == MODE_REPLICATED else \
            [(self.shard_base(s), self.part_len(s)) for s in range(self.num_parts())]
        return np.concatenate([np.arange(b, b + n, dtype=np.uint64) for b, n in parts] + [np.zeros(0, np.uint64)])

    def knn_graph(self, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS, exclude_self=True,
                  exact=False, chunk=65536):
        """Granne.knn_graph over all parts: for every global id of global_ids(), search_batch (exact_search_batch with
        exact=True) of that element by id, without itself when exclude_self.  The ids go through the host calls in
        chunks of `chunk`, each made as it is needed.  Returns (ids uint64 GLOBAL ids [len, k] padded with
        0xFFFF_FFFF_FFFF_FFFF, dists float32 [len, k], counts uint32 [len]); row r belongs to global_ids()[r]."""
        if int(chunk) < 1:
            raise ValueError("chunk must be >= 1")
        k = int(num_elements)
        parts = [(0, len(self))] if self.mode == MODE_REPLICATED else \
            [(self.shard_base(s), self.part_len(s)) for s in range(self.num_parts())]
        total = sum(n for _, n in parts)
        ids, dists, counts, _ = _host_outputs(total, k, np.uint64)
        row = 0
        for base, n in parts:
            for c0 in range(0, n, int(chunk)):
                q = np.arange(base + c0, base + min(n, c0 + int(chunk)), dtype=np.uint64)
                if exact:
                    r = self.exact_search_batch(q, k, by_id=True, exclude_self=exclude_self)
                else:
                    r = self.search_batch(q, max_search, k, by_id=True, exclude_self=exclude_self)
                ids[row:row + q.size], dists[row:row + q.size], counts[row:row + q.size] = r
                row += q.size
        return ids, dists, counts

    def _host_queries(self, queries, already_element, by_id, exclude_self):
        """(contiguous queries, query format) of a host call: rows, or GLOBAL uint64 element ids with by_id /
        exclude_self."""
        if by_id or exclude_self:
            return _id_queries(queries, exclude_self, np.uint64)
        return _host_queries(queries, already_element)

    def search_batch(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                     already_element=False, by_id=False, exclude_self=False):
        """Granne.search_batch over all parts: GLOBAL uint64 ids in the results, and as queries with by_id (each in
        some part's [shard_base, shard_base + Index::len) range) — exclude_self drops each query's own global id."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_search_batch(self._h, _ptr(q), nq, fmt, int(max_search), k, _ptr(ids),
                                                             _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def search_batch_diverse(self, queries, max_search=DEFAULT_MAX_SEARCH, num_elements=DEFAULT_NUM_ELEMENTS,
                             already_element=False, by_id=False, exclude_self=False):
        """Granne.search_batch_diverse over all parts (granne_b200_multi_search_diverse_batch): GLOBAL uint64 ids.
        Partitioned, the shards' max_search lists are merged by (distance, global id) and select_neighbors runs over
        the global container."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_search_diverse_batch(self._h, _ptr(q), nq, fmt, int(max_search), k,
                                                                     _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_search_batch(self, queries, num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, by_id=False,
                           exclude_self=False):
        """Exact k nearest neighbours over all shards (granne_b200_multi_exact_search_batch): GLOBAL uint64 ids."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_exact_search_batch(self._h, _ptr(q), nq, fmt, k, _ptr(ids),
                                                                   _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_search_within(self, queries, candidates, num_elements=DEFAULT_NUM_ELEMENTS, already_element=False,
                            by_id=False, exclude_self=False):
        """Granne.exact_search_within over all parts (granne_b200_multi_exact_search_within_batch): GLOBAL ids in the
        candidate lists (uint64) and in the results."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        offsets, cand = _candidate_lists(candidates, nq, np.uint64)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_exact_search_within_batch(
            self._h, _ptr(q), nq, fmt, _ptr(offsets), _ptr(cand), k, _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_range_count(self, queries, radius, already_element=False, by_id=False, exclude_self=False):
        """Granne.exact_range_count over all parts (granne_b200_multi_exact_range_count): a range-partitioned handle
        sums the shards' counts.  GLOBAL uint64 ids as queries with by_id."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        counts = np.empty(q.shape[0], dtype=np.uint64)
        _check(load_library().granne_b200_multi_exact_range_count(self._h, _ptr(q), q.shape[0], fmt, _radius(radius),
                                                                  _ptr(counts)))
        return counts

    def exact_range_search(self, queries, radius, already_element=False, by_id=False, exclude_self=False):
        """Granne.exact_range_search over all parts (granne_b200_multi_exact_range_search): (offsets uint64 [nq + 1],
        GLOBAL ids uint64, dists float32), each query's entries sorted by (distance, global id)."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        r = _radius(radius)
        offsets = _csr_offsets(self.exact_range_count(q, r, already_element=fmt == QUERY_ELEMENT, by_id=by_id,
                                                      exclude_self=exclude_self))
        ids = np.empty(int(offsets[-1]), dtype=np.uint64)
        dists = np.empty(int(offsets[-1]), dtype=np.float32)
        _check(load_library().granne_b200_multi_exact_range_search(self._h, _ptr(q), q.shape[0], fmt, r, _ptr(offsets),
                                                                   _ptr(ids), _ptr(dists)))
        return offsets, ids, dists

    def search_batch_filtered(self, queries, filters, query_filter=None, max_search=DEFAULT_MAX_SEARCH,
                              num_elements=DEFAULT_NUM_ELEMENTS, already_element=False, by_id=False,
                              exclude_self=False):
        """Granne.search_batch_filtered over all parts (granne_b200_multi_search_filtered_batch): the filters are over
        GLOBAL ids (a bool mask of shape (len,) or (F, len), or uint32 words), the results are GLOBAL uint64 ids."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        words = _filter_words(filters, len(self))
        qf = _query_filter(query_filter, nq)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_search_filtered_batch(
            self._h, _ptr(q), nq, fmt, int(max_search), k, _ptr(words), words.shape[0], words.shape[1],
            _ptr(qf) if qf is not None else None, _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def exact_search_filtered(self, queries, filters, query_filter=None, num_elements=DEFAULT_NUM_ELEMENTS,
                              already_element=False, by_id=False, exclude_self=False):
        """Granne.exact_search_filtered over all parts (granne_b200_multi_exact_search_filtered_batch): the filters
        are over GLOBAL ids, as in search_batch_filtered, and the results are GLOBAL uint64 ids."""
        q, fmt = self._host_queries(queries, already_element, by_id, exclude_self)
        nq, k = q.shape[0], int(num_elements)
        words = _filter_words(filters, len(self))
        qf = _query_filter(query_filter, nq)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_exact_search_filtered_batch(
            self._h, _ptr(q), nq, fmt, _ptr(words), words.shape[0], words.shape[1],
            _ptr(qf) if qf is not None else None, k, _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def set_rerank_elements(self, elements):
        """Granne.set_rerank_elements on every part: one angular elements image (`bytes`) for a replicated handle,
        a list with one image per shard for a partitioned one."""
        keep, ptrs, lens = self._part_images(elements)
        _check(load_library().granne_b200_multi_set_rerank_elements(self._h, ptrs, lens))

    def set_rerank_embeddings(self, elements_list, embeddings):
        """Granne.set_rerank_embeddings on every part: one term-list image (`bytes`) for a replicated handle, a list
        with one per shard for a partitioned one, and one embedding table image shared by all parts."""
        keep, ptrs, lens = self._part_images(elements_list)
        mb = np.frombuffer(embeddings, dtype=np.uint8)
        _check(load_library().granne_b200_multi_set_rerank_embeddings(self._h, ptrs, lens, _ptr(mb), mb.size))

    def _part_images(self, images):
        """One image (`bytes`) or a list of them as (arrays that keep them alive, void*[], size_t[]): one for a
        replicated handle, one per shard for a partitioned one."""
        images = [images] if isinstance(images, (bytes, bytearray, memoryview)) else list(images)
        keep = [np.frombuffer(e, dtype=np.uint8) for e in images]
        if len(keep) != (1 if self.mode == MODE_REPLICATED else self.num_parts()):
            raise ValueError("one image for a replicated handle, one per shard for a partitioned one")
        return (keep, (C.c_void_p * len(keep))(*[a.ctypes.data for a in keep]),
                (C.c_size_t * len(keep))(*[a.size for a in keep]))

    def search_batch_rerank(self, queries, num_candidates, max_search=DEFAULT_MAX_SEARCH,
                            num_elements=DEFAULT_NUM_ELEMENTS):
        """Two-stage search over all parts (granne_b200_multi_search_rerank_batch): GLOBAL uint64 ids."""
        q = _raw_f32_queries(queries)
        nq, k = q.shape[0], int(num_elements)
        ids, dists, counts, _ = _host_outputs(nq, k, np.uint64)
        _check(load_library().granne_b200_multi_search_rerank_batch(self._h, _ptr(q), nq, QUERY_RAW_F32,
                                                                    int(max_search), int(num_candidates), k,
                                                                    _ptr(ids), _ptr(dists), _ptr(counts)))
        return ids, dists, counts

    def close(self):
        if getattr(self, "_h", None):
            load_library().granne_b200_multi_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PeerGather(C.Structure):
    """granne_b200_peer_gather: peer-mapped result buffers for the fused multi-GPU gather."""
    _fields_ = [("n_peers", C.c_uint32), ("my_rank", C.c_uint32), ("row_offset", C.c_uint64), ("seq", C.c_uint32),
                ("reserved", C.c_uint32), ("ids", C.c_void_p * 8), ("dists", C.c_void_p * 8),
                ("flags", C.c_void_p * 8)]


class BuildConfig(C.Structure):
    """granne::BuildConfig (src/index/mod.rs:198-291) as the C ABI struct granne_b200_build_config."""
    _fields_ = [("layer_multiplier", C.c_float), ("expected_num_elements", C.c_int64),
                ("num_neighbors", C.c_uint32), ("max_search", C.c_uint32), ("reinsert_elements", C.c_int32),
                ("show_progress", C.c_int32)]


def _build_config(num_neighbors, max_search, layer_multiplier, reinsert_elements, expected_num_elements,
                  show_progress=False):
    cfg = BuildConfig()
    load_library().granne_b200_build_config_default(C.byref(cfg))
    cfg.num_neighbors = num_neighbors
    cfg.max_search = max_search
    cfg.layer_multiplier = layer_multiplier
    cfg.reinsert_elements = int(bool(reinsert_elements))
    cfg.expected_num_elements = -1 if expected_num_elements is None else int(expected_num_elements)
    cfg.show_progress = int(bool(show_progress))
    return cfg


def elements_from_raw(element_type, raw, device=0):
    """Builds an elements file image from raw f32 rows on the GPU exactly like `Vector::from(Vec<f32>)` per row
    (normalise for "angular", quantise for "angular_int")."""
    L = load_library()
    raw = np.ascontiguousarray(raw, dtype=np.float32)
    n, dim = raw.shape
    kind = _kind(element_type)
    need = C.c_size_t()
    _check(L.granne_b200_elements_from_raw(kind, None, n, dim, device, None, 0, C.byref(need)))
    out = np.empty(need.value, dtype=np.uint8)
    _check(L.granne_b200_elements_from_raw(kind, _ptr(raw), n, dim, device, _ptr(out), out.size, C.byref(need)))
    return out


def _write_index(fn, handle, layer_lens):
    """One encode instead of two: the first call gets a buffer sized for the common case (<= 32 neighbours per node:
    1 count byte + 4 bytes per id is the writer's worst case); only an index with wider rows needs the size query."""
    guess = 1024 + sum(8 + (1 + n // 60) * 128 + n * (1 + 4 * 32) for n in layer_lens)
    out = np.empty(guess, dtype=np.uint8)
    need = C.c_size_t()
    rc = fn(handle, _ptr(out), out.size, C.byref(need))
    if rc != 0 and need.value > out.size:
        out = np.empty(need.value, dtype=np.uint8)
        rc = fn(handle, _ptr(out), out.size, C.byref(need))
    _check(rc)
    return out[:need.value]


def _check_stats(stats, q):
    import torch

    if stats is not None and (not isinstance(stats, torch.Tensor) or not stats.is_cuda or stats.device != q.device
                              or stats.dtype != torch.int64 or tuple(stats.shape) != (q.shape[0], STATS_PER_QUERY)
                              or not stats.is_contiguous()):
        raise ValueError("stats must be a contiguous int64 [nq, %d] tensor on the queries' device" % STATS_PER_QUERY)


def _check_device_rows(kind, t):
    import torch

    want = torch.int8 if kind == ANGULAR_INT else torch.float32
    if kind not in (ANGULAR, ANGULAR_INT):
        raise ValueError("device-resident elements: angular or angular_int")
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dim() != 2 or t.dtype != want or not t.is_contiguous():
        raise ValueError("elements must be a contiguous CUDA tensor [n, dim] of %s" % want)


def elements_from_raw_device(element_type, raw, out=None, stream=None):
    """`Vector::from(Vec<f32>)` per row, device to device: raw = CUDA float32 [n, dim]; returns (or fills `out`) the
    elements as a CUDA tensor [n, dim] (float32 normalised for "angular", int8 for "angular_int").  Asynchronous on
    `stream` (a torch.cuda.Stream or a raw cudaStream_t; default: the current torch stream)."""
    import torch

    kind = _kind(element_type)
    if not raw.is_cuda or raw.dtype != torch.float32 or raw.dim() != 2 or not raw.is_contiguous():
        raise ValueError("raw must be a contiguous CUDA float32 tensor [n, dim]")
    n, dim = raw.shape
    if out is None:
        out = torch.empty((n, dim), dtype=torch.int8 if kind == ANGULAR_INT else torch.float32, device=raw.device)
    _check_device_rows(kind, out)
    if tuple(out.shape) != (n, dim) or out.device != raw.device:
        raise ValueError("out must match raw's shape and device")
    _check(load_library().granne_b200_elements_from_raw_device(kind, C.c_void_p(raw.data_ptr()), n, dim,
                                                               raw.device.index, C.c_void_p(out.data_ptr()),
                                                               C.c_void_p(_raw_stream(stream, raw.device))))
    return out


def _embeddings_kind(element_type):
    kind = _kind(element_type)
    if kind not in (ANGULAR, ANGULAR_INT):
        raise ValueError("compute_embeddings writes \"angular\" or \"angular_int\" vectors")
    return kind


def _compute_embeddings_into(kind, eb, mb, device, make_out):
    """The two calls of granne_b200_compute_embeddings: the first learns the image's size, make_out(size) gives the
    uint8 buffer (at least that long), the second fills it.  Returns the image's part of the buffer."""
    L = load_library()
    need = C.c_size_t()
    _check(L.granne_b200_compute_embeddings(kind, _ptr(eb), eb.size, _ptr(mb), mb.size, device, None, 0,
                                            C.byref(need)))
    out = make_out(need.value)
    _check(L.granne_b200_compute_embeddings(kind, _ptr(eb), eb.size, _ptr(mb), mb.size, device, _ptr(out), out.size,
                                            C.byref(need)))
    return out[:need.value]


def compute_embeddings(element_type, elements_bytes, embeddings_bytes, out=None, device=0):
    """compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152) in memory: the elements file
    image of the sum of embeddings of every element of a SumEmbeddings container, made into "angular_int" vectors (the
    quantised raw sum; what the reference writes) or "angular" vectors (the normalised sum: SumEmbeddings::get, so that
    searching the rows searches the container).  Returns the image as a uint8 array, or fills `out` (a writable
    uint8 buffer of at least the image's size, e.g. an np.memmap) and returns the image's part of it."""
    kind = _embeddings_kind(element_type)
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    mb = np.frombuffer(embeddings_bytes, dtype=np.uint8)

    def buffer(size):
        if out is None:
            return np.empty(size, dtype=np.uint8)
        if (not isinstance(out, np.ndarray) or out.dtype != np.uint8 or out.ndim != 1 or not out.flags.c_contiguous
                or not out.flags.writeable):
            raise ValueError("out must be a writable contiguous 1-d uint8 array")
        if out.size < size:
            raise ValueError("out holds %d bytes; the image needs %d" % (out.size, size))
        return out

    return _compute_embeddings_into(kind, eb, mb, device, buffer)


def compute_embeddings_device(element_type, elements_bytes, embeddings_bytes, out=None, device=None, stream=None):
    """The rows of compute_embeddings as a CUDA tensor [n, dim] (float32 for "angular", int8 for "angular_int"), or
    written into `out`; for Granne.from_device_elements / GranneBuilder.from_device_elements.  device: out's device,
    else the current one.  stream: a torch.cuda.Stream or a raw cudaStream_t (default: the current torch stream).
    Returns when the rows are written."""
    import torch

    L = load_library()
    kind = _embeddings_kind(element_type)
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    mb = np.frombuffer(embeddings_bytes, dtype=np.uint8)
    n, dim = C.c_uint64(), C.c_uint32()
    _check(L.granne_b200_compute_embeddings_device(kind, _ptr(eb), eb.size, _ptr(mb), mb.size, 0, None, C.byref(n),
                                                   C.byref(dim), None))
    if device is None:
        device = out.device.index if isinstance(out, torch.Tensor) and out.is_cuda else torch.cuda.current_device()
    if out is None:
        out = torch.empty((n.value, dim.value), dtype=torch.int8 if kind == ANGULAR_INT else torch.float32,
                          device=torch.device("cuda", device))
    _check_device_rows(kind, out)
    if tuple(out.shape) != (n.value, dim.value) or out.device != torch.device("cuda", device):
        raise ValueError("out must be a [%d, %d] tensor on cuda:%d" % (n.value, dim.value, device))
    _check(L.granne_b200_compute_embeddings_device(kind, _ptr(eb), eb.size, _ptr(mb), mb.size, device,
                                                   C.c_void_p(out.data_ptr()), C.byref(n), C.byref(dim),
                                                   C.c_void_p(_raw_stream(stream, out.device))))
    return out


def compute_embeddings_and_save_to_disk(elements_path, embeddings_path, output_path, show_progress=True,
                                        element_type="angular_int", device=0):
    """granne.compute_embeddings_and_save_to_disk (py/src/lib.rs:132-147; parsing.rs:102-152) on the GPU, same
    argument order.  The image is written through a memory map of the output file.  show_progress is accepted and
    ignored."""
    kind = _embeddings_kind(element_type)
    eb = np.memmap(elements_path, dtype=np.uint8, mode="r") if os.path.getsize(elements_path) else np.zeros(0, np.uint8)
    mb = (np.memmap(embeddings_path, dtype=np.uint8, mode="r") if os.path.getsize(embeddings_path)
          else np.zeros(0, np.uint8))
    image = _compute_embeddings_into(kind, eb, mb, device,
                                     lambda size: np.memmap(output_path, dtype=np.uint8, mode="w+", shape=(size,)))
    image.flush()


class GranneBuilder:
    """granne.GranneBuilder (py/src/lib.rs:346-579; src/index/mod.rs:295-531) on the GPU.

    GranneBuilder(element_type, elements_bytes, embeddings_bytes=None, num_neighbors=30, max_search=200,
                  layer_multiplier=15.0, reinsert_elements=True, expected_num_elements=None, device=0,
                  index_bytes=None)
    `elements_bytes` is an elements file image (see elements_from_raw / Granne.save_elements).  num_neighbors may be
    anything the file format can hold (1..255: a list's length is one byte); show_progress is accepted and ignored.
    With `index_bytes` (an index file image built over these elements, or over a prefix of them) the builder continues
    from that index (GranneBuilder::from_bytes, src/index/mod.rs:428-461): the next build() indexes only the elements
    beyond it.  Every loaded neighbour list is cut to its first `num_neighbors` ids (the lowest, as in the reference)."""

    def __init__(self, element_type, elements_bytes, embeddings_bytes=None, num_neighbors=30, max_search=200,
                 layer_multiplier=15.0, reinsert_elements=True, expected_num_elements=None, show_progress=False,
                 device=0, index_bytes=None):
        L = load_library()
        cfg = _build_config(num_neighbors, max_search, layer_multiplier, reinsert_elements, expected_num_elements,
                            show_progress)
        eb = np.frombuffer(elements_bytes, dtype=np.uint8)
        mb = np.frombuffer(embeddings_bytes, dtype=np.uint8) if embeddings_bytes is not None else None
        h = C.c_void_p()
        mb_args = (_ptr(mb) if mb is not None else None, mb.size if mb is not None else 0)
        if index_bytes is None:
            _check(L.granne_b200_builder_new(C.byref(cfg), _kind(element_type), _ptr(eb), eb.size, *mb_args, device,
                                             C.byref(h)))
        else:
            ib = np.frombuffer(index_bytes, dtype=np.uint8)
            _check(L.granne_b200_builder_from_index(C.byref(cfg), _ptr(ib), ib.size, _kind(element_type), _ptr(eb),
                                                    eb.size, *mb_args, device, C.byref(h)))
        self._h = h
        self.device = device
        self._element_type = element_type
        self._elements_bytes = elements_bytes
        self._embeddings_bytes = embeddings_bytes
        self._pending = []

    @classmethod
    def from_files(cls, element_type, elements_path, index_path=None, embeddings_path=None, **config):
        """The reference's keyword form GranneBuilder(element_type, elements_path=..., index_path=...,
        embeddings_path=...) (py/src/lib.rs:384-442): reads the files and builds from them; with `index_path` the
        builder continues from that index.  `config`: the keyword arguments of GranneBuilder (num_neighbors, ...,
        device).  An "embeddings" builder takes term lists, not a words file."""
        kind = _kind(element_type)
        if elements_path is None:
            raise ValueError("elements_path is required%s" % (" together with index_path" if index_path else ""))
        if kind == EMBEDDINGS and embeddings_path is None:
            raise ValueError("embeddings_path required for this element type!")

        def read(path):
            with open(path, "rb") as f:
                return f.read()

        return cls(element_type, read(elements_path), read(embeddings_path) if kind == EMBEDDINGS else None,
                   index_bytes=read(index_path) if index_path is not None else None, **config)

    @classmethod
    def from_device_elements(cls, element_type, elements, num_neighbors=30, max_search=200, layer_multiplier=15.0,
                             reinsert_elements=True, expected_num_elements=None, device=None, index_bytes=None):
        """GranneBuilder::new(config, elements) over a device-resident container (see Granne.from_device_elements);
        with `index_bytes`, GranneBuilder::from_bytes over it (see GranneBuilder)."""
        L = load_library()
        kind = _kind(element_type)
        _check_device_rows(kind, elements)
        device = elements.device.index if device is None else device
        cfg = _build_config(num_neighbors, max_search, layer_multiplier, reinsert_elements, expected_num_elements)
        self = cls.__new__(cls)
        h = C.c_void_p()
        rows = (kind, C.c_void_p(elements.data_ptr()), elements.shape[0], elements.shape[1], device, C.byref(h))
        if index_bytes is None:
            _check(L.granne_b200_builder_new_device_elements(C.byref(cfg), *rows))
        else:
            ib = np.frombuffer(index_bytes, dtype=np.uint8)
            _check(L.granne_b200_builder_from_index_device_elements(C.byref(cfg), _ptr(ib), ib.size, *rows))
        self._h = h
        self.device = device
        self._element_type = element_type
        self._elements_bytes = None
        self._embeddings_bytes = None
        self._pending = []
        return self

    def append(self, element):
        """GranneBuilder.append(element) (py/src/lib.rs:474-476; py/src/variants/builder.rs:6-21): the raw vector
        becomes an element (`Vector::from`) and is pushed; it is indexed by the next build().  Rows are buffered and
        handed to the library in one batch."""
        if _kind(self._element_type) == EMBEDDINGS:
            # SumEmbeddings::push (src/elements/embeddings/mod.rs:97-100): an element is a list of embedding ids
            # (the reference's WordEmbeddingsBuilder maps a string to ids first, py/src/variants/builder.rs:84-93)
            if isinstance(element, str):
                raise ValueError("pass embedding ids (WordDict.get_word_ids(text)) — this builder holds no word list")
            self._pending.append([int(t) for t in element])
            return
        self._pending.append(np.asarray(element, dtype=np.float32))

    def _flush(self):
        if not self._pending:
            return
        if _kind(self._element_type) == EMBEDDINGS:
            from . import words as W

            fresh, self._pending = self._pending, []
            image = np.frombuffer(W.write_sum_terms(fresh), dtype=np.uint8)
            _check(load_library().granne_b200_builder_append(self._h, _ptr(image), image.size))
            if self._elements_bytes is not None:
                self._elements_bytes = W.write_sum_terms(W.read_sum_terms(bytes(self._elements_bytes)) + fresh)
            return
        raw = np.stack(self._pending)
        self._pending = []
        image = elements_from_raw(self._element_type, raw, self.device)
        _check(load_library().granne_b200_builder_append(self._h, _ptr(image), image.size))
        if self._elements_bytes is not None:
            old = np.frombuffer(self._elements_bytes, dtype=np.uint8)
            self._elements_bytes = np.concatenate([old, image[8:]])  # same u64 width prefix, more rows

    def build(self, num_elements=0):
        """Builder::build() / build_partial(num_elements)."""
        self._flush()
        _check(load_library().granne_b200_builder_build(self._h, int(num_elements)))

    def __len__(self):
        return int(load_library().granne_b200_builder_len(self._h))

    def num_layers(self):
        return int(load_library().granne_b200_builder_num_layers(self._h))

    def layer_len(self, layer):
        return int(load_library().granne_b200_builder_layer_len(self._h, layer))

    def index_bytes(self):
        """Index::write_index into memory: a granne index file image (uint8 array)."""
        return _write_index(load_library().granne_b200_builder_write_index, self._h,
                            [self.layer_len(l) for l in range(self.num_layers())])

    def save_index(self, path):
        """GranneBuilder.save_index(path) (py/src/lib.rs)."""
        with open(path, "wb") as f:
            f.write(self.index_bytes().tobytes())

    def get_index(self):
        """GranneBuilder::get_index: a searchable Granne sharing the staged elements."""
        self._flush()
        h = C.c_void_p()
        _check(load_library().granne_b200_builder_get_index(self._h, C.byref(h)))
        g = Granne.__new__(Granne)
        g._h = h
        g.device = self.device
        g._elements_src = ("bytes", self._elements_bytes) if self._elements_bytes is not None else None
        g._embeddings_src = ("bytes", self._embeddings_bytes) if self._embeddings_bytes is not None else None
        return g

    def save_elements(self, path):
        """GranneBuilder.save_elements(path) (py/src/lib.rs:518-522)."""
        self._flush()
        if self._elements_bytes is None:
            raise GranneError(-1, "this builder was made from device-resident elements: no host image to save")
        with open(path, "wb") as f:
            f.write(bytes(self._elements_bytes))

    def get_neighbors(self, idx, layer=None):
        """GranneBuilder.get_neighbors(idx, layer=last) (py/src/lib.rs:544-552)."""
        if layer is None:
            layer = self.num_layers() - 1
        out = np.empty(256, dtype=np.uint32)
        n = C.c_size_t()
        _check(load_library().granne_b200_builder_get_neighbors(self._h, idx, layer, _ptr(out), out.size,
                                                                C.byref(n)))
        return out[:n.value].tolist()

    def num_elements(self):
        """GranneBuilder.num_elements() (py/src/lib.rs:559-561): elements held, indexed or not."""
        self._flush()
        return int(load_library().granne_b200_builder_num_elements(self._h))

    def close(self):
        if getattr(self, "_h", None):
            load_library().granne_b200_builder_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def inspect_index(index_bytes):
    """Host-only: [(layer_len, max_degree, row_width)] per layer of a granne index image."""
    L = load_library()
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    nl = C.c_uint64()
    lens = np.zeros(64, dtype=np.uint64)
    degs = np.zeros(64, dtype=np.uint32)
    widths = np.zeros(64, dtype=np.uint32)
    _check(L.granne_b200_inspect_index(_ptr(ib), ib.size, C.byref(nl), _ptr(lens), _ptr(degs), _ptr(widths), 64))
    return [(int(lens[i]), int(degs[i]), int(widths[i])) for i in range(nl.value)]


def reencode_index(index_bytes):
    """Host-only: decode an index image and write it again with the library's writer (Index::write_index)."""
    L = load_library()
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    need = C.c_size_t()
    _check(L.granne_b200_reencode_index(_ptr(ib), ib.size, None, 0, C.byref(need)))
    out = np.empty(need.value, dtype=np.uint8)
    _check(L.granne_b200_reencode_index(_ptr(ib), ib.size, _ptr(out), out.size, C.byref(need)))
    return out.tobytes()


def compute_distances(element_type, a, b, device=0):
    """n pairwise distances Vector::from(a_i).dist(&Vector::from(b_i)) on the GPU; a, b: (n, dim) raw float32."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    if a.ndim != 2 or a.shape != b.shape:
        raise ValueError("a and b must both have shape (n, dim)")
    out = np.empty(a.shape[0], dtype=np.float32)
    _check(load_library().granne_b200_compute_distances(_kind(element_type), _ptr(a), _ptr(b), a.shape[0], a.shape[1],
                                                        device, _ptr(out)))
    return out


def compute_distance(element_type, a, b, device=0):
    """granne.compute_distance(element_type, a, b) (py/src/lib.rs:71-89)."""
    if element_type not in ("angular", "angular_int"):
        raise ValueError("Unsupported element type")
    return float(compute_distances(element_type, np.asarray(a, dtype=np.float32)[None, :],
                                   np.asarray(b, dtype=np.float32)[None, :], device)[0])


def order_from_trails(layer_lens, trails):
    """Host-only: the sort half of compute_order for trails (uint32 [n, 8]) computed elsewhere."""
    lens = np.ascontiguousarray(layer_lens, dtype=np.uint64)
    t = np.ascontiguousarray(trails, dtype=np.uint32)
    order = np.zeros(t.shape[0], dtype=np.uint64)
    _check(load_library().granne_b200_order_from_trails(_ptr(lens), lens.size, _ptr(t), t.shape[0], _ptr(order)))
    return order


def order_by_keys(index_bytes, keys):
    """Host-only: the layer-preserving sort of Granne::reorder_by_keys (reorder.rs:96-108)."""
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    k = np.ascontiguousarray(keys, dtype=np.uint64)
    k = k.reshape(k.shape[0], -1)
    order = np.zeros(k.shape[0], dtype=np.uint64)
    _check(load_library().granne_b200_order_by_keys(_ptr(ib), ib.size, _ptr(k), k.shape[0], k.shape[1], _ptr(order)))
    return order


def compute_keys_for_reordering(elements_bytes, embeddings_bytes):
    """Host-only: embeddings::compute_keys_for_reordering (embeddings/reorder.rs:31-58) -> uint64 [n, 8]."""
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    mb = np.frombuffer(embeddings_bytes, dtype=np.uint8)
    n = int(np.frombuffer(eb[:8].tobytes(), dtype=np.uint64)[0]) if eb.size >= 8 else -1
    if n < 0 or 8 + (n + 1) * 5 > eb.size:  # u64 count | (count + 1) five-byte offsets | ids
        raise GranneError(-2, "embeddings elements file: offset table exceeds the file")
    keys = np.zeros((n, 8), dtype=np.uint64)
    _check(load_library().granne_b200_embedding_reorder_keys(_ptr(eb), eb.size, _ptr(mb), mb.size, _ptr(keys)))
    return keys


def apply_order(index_bytes, element_type, elements_bytes, order):
    """Host-only: reorder_layers + Permutable::permute -> (index file image, elements file image) as bytes."""
    L = load_library()
    kind = element_type if isinstance(element_type, int) else _kind(element_type)
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    o = np.ascontiguousarray(order, dtype=np.uint64)
    n_i, n_e = C.c_size_t(), C.c_size_t()
    _check(L.granne_b200_apply_order(_ptr(ib), ib.size, kind, _ptr(eb), eb.size, _ptr(o), o.size, None, 0,
                                     C.byref(n_i), None, 0, C.byref(n_e)))
    oi, oe = np.empty(n_i.value, dtype=np.uint8), np.empty(n_e.value, dtype=np.uint8)
    _check(L.granne_b200_apply_order(_ptr(ib), ib.size, kind, _ptr(eb), eb.size, _ptr(o), o.size, _ptr(oi), oi.size,
                                     C.byref(n_i), _ptr(oe), oe.size, C.byref(n_e)))
    return oi.tobytes(), oe.tobytes()


def decode_layer(index_bytes, layer):
    """Host-only: the fixed-width u32 rows (padded with 0xFFFFFFFF) the loader stages in HBM for `layer`."""
    shape = inspect_index(index_bytes)
    n, _, w = shape[layer]
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    rows = np.empty((n, w), dtype=np.uint32)
    _check(load_library().granne_b200_decode_layer(_ptr(ib), ib.size, layer, _ptr(rows), rows.size))
    return rows


def merge_topk_device(device, part_ids, part_dists, part_base, out_ids=None, out_dists=None, stream=None):
    """granne_b200_merge_topk_device over CUDA torch tensors: part_ids int32 [P, nq, k] (u32 bits), part_dists
    float32 [P, nq, k], part_base list of P global id offsets.  Returns (int64 [nq,k] global ids, float32 dists).
    Asynchronous on `stream` (a torch.cuda.Stream or a raw cudaStream_t; default: the current torch stream)."""
    import torch

    # the library takes raw pointers and indexes them as [P][nq][k]: anything else would be read out of bounds
    def tensor_ok(t, dtype, shape):
        return (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()
                and tuple(t.shape) == shape and t.device == torch.device("cuda", device))

    if not isinstance(part_ids, torch.Tensor) or part_ids.dim() != 3:
        raise ValueError("part_ids must be a CUDA int32 tensor [P, nq, k]")
    P, nq, k = part_ids.shape
    if not tensor_ok(part_ids, torch.int32, (P, nq, k)) or not tensor_ok(part_dists, torch.float32, (P, nq, k)):
        raise ValueError("part_ids (int32) and part_dists (float32) must be contiguous [P, nq, k] tensors on cuda:%d"
                         % device)
    if len(part_base) != P:
        raise ValueError("part_base must hold one global id offset per part (%d), not %d" % (P, len(part_base)))
    if (out_ids is None) != (out_dists is None):
        raise ValueError("pass both out_ids and out_dists, or neither")
    if out_ids is None:
        out_ids = torch.empty((nq, k), dtype=torch.int64, device=part_ids.device)
        out_dists = torch.empty((nq, k), dtype=torch.float32, device=part_ids.device)
    if not tensor_ok(out_ids, torch.int64, (nq, k)) or not tensor_ok(out_dists, torch.float32, (nq, k)):
        raise ValueError("out_ids (int64) and out_dists (float32) must be contiguous [nq, k] tensors on cuda:%d" % device)
    base = np.ascontiguousarray(part_base, dtype=np.uint64)
    _check(load_library().granne_b200_merge_topk_device(
        device, C.c_void_p(part_ids.data_ptr()), C.c_void_p(part_dists.data_ptr()), _ptr(base), P, nq, k,
        C.c_void_p(out_ids.data_ptr()), C.c_void_p(out_dists.data_ptr()),
        C.c_void_p(_raw_stream(stream, part_ids.device))))
    return out_ids, out_dists
