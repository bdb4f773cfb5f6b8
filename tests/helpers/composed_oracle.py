"""ctypes wrapper over tests/helpers/composed_oracle.cpp: checkers composed from the CPU oracle's own pieces.
- Container.exact_search: brute-force k nearest neighbours, the checker of granne_b200_exact_search_batch.
- Filtered.search: the oracle's descent, its bottom-layer search_for_neighbors (recording the scored ids), a filter and
  dist_to_element, the checker of granne_b200_search_filtered_batch.
- compute_embeddings: the oracle's restatement of compute_embeddings_and_save_to_disk
  (src/elements/embeddings/parsing.rs:102-152), the checker of granne_b200_compute_embeddings.

TEST INFRASTRUCTURE ONLY.  The library is compiled with the oracle's flags (oracle/Makefile) into a temporary directory,
so that the source tree is never written to.  It shares no state with oracle/granne_oracle.py's library: the index and
the containers are passed to it as file images."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SOURCES = [os.path.join(_HERE, "composed_oracle.cpp"), os.path.join(_ROOT, "oracle", "granne_oracle.cpp")]
_FLAGS = ["-O3", "-std=c++17", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-pthread", "-shared"]
ANGULAR, ANGULAR_INT, EMBEDDINGS = 0, 1, 2
_KINDS = {"angular": ANGULAR, "angular_int": ANGULAR_INT, "embeddings": EMBEDDINGS}

_lib = None


def build_lib():
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out_dir = os.path.join(tempfile.gettempdir(), "granne_b200_composed_oracle_%d" % os.getuid())
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "lib_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(path):
        tmp = "%s.%d.tmp" % (path, os.getpid())
        subprocess.check_call([os.environ.get("CXX", "g++")] + _FLAGS + ["-o", tmp, _SOURCES[0]])
        os.replace(tmp, path)
    return path


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_lib())
        vp, u64 = C.c_void_p, C.c_uint64
        L.orc_last_error.restype = C.c_char_p
        L.orc_elements_from_bytes.restype = vp
        L.orc_elements_from_bytes.argtypes = [C.c_int, vp, u64, vp, u64]
        L.orc_elements_free.argtypes = [vp]
        L.orc_elements_len.restype = u64
        L.orc_elements_len.argtypes = [vp]
        L.orc_elements_dim.restype = u64
        L.orc_elements_dim.argtypes = [vp]
        L.orc_index_from_bytes.restype = vp
        L.orc_index_from_bytes.argtypes = [vp, u64]
        L.orc_index_free.argtypes = [vp]
        L.orc_index_len.restype = u64
        L.orc_index_len.argtypes = [vp]
        L.orc_exact_search.restype = C.c_int
        L.orc_exact_search.argtypes = [vp, u64, vp, vp, u64, C.c_int, u64, C.c_int, vp, vp, vp]
        L.orc_filtered_search.restype = C.c_int
        L.orc_filtered_search.argtypes = [vp, vp, vp, vp, u64, C.c_int, u64, u64, vp, u64, vp, u64, C.c_int, vp, vp,
                                          vp, vp]
        L.orc_compute_embeddings.restype = C.c_int64
        L.orc_compute_embeddings.argtypes = [vp, C.c_int, C.c_int, vp, u64]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class NotFinite(ValueError):
    """A distance the oracle computes is NaN, or a sum of embeddings is not finite: the reference panics, or the rows
    would hold NaN."""


def _kind(kind):
    return _KINDS[kind] if isinstance(kind, str) else int(kind)


def _queries(queries, already_element):
    """(f32 rows, int8 rows or None, already_element): int8 queries are angular_int elements."""
    q = np.asarray(queries)
    if q.dtype == np.int8:
        return np.zeros(q.shape, dtype=np.float32), np.ascontiguousarray(q), True
    return np.ascontiguousarray(q, dtype=np.float32), None, already_element


def _open_elements(kind, eb, mb):
    L = lib()
    h = L.orc_elements_from_bytes(kind, _ptr(eb), eb.size, _ptr(mb) if mb is not None else None,
                                  mb.size if mb is not None else 0)
    if not h:
        raise ValueError(L.orc_last_error().decode())
    return h


class Container:
    """An oracle element container opened from file images (elements file, and the embeddings table for
    "embeddings")."""

    def __init__(self, kind, elements_bytes, embeddings_bytes=None):
        self.kind = _kind(kind)
        self._eb = np.frombuffer(elements_bytes, dtype=np.uint8)
        self._mb = np.frombuffer(embeddings_bytes, dtype=np.uint8) if embeddings_bytes is not None else None
        self._h = _open_elements(self.kind, self._eb, self._mb)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().orc_elements_free(self._h)
                self._h = None
        except Exception:  # interpreter shutdown
            pass

    def __len__(self):
        return int(lib().orc_elements_len(self._h))

    @property
    def dim(self):
        return int(lib().orc_elements_dim(self._h))

    def exact_search(self, queries, k, index_len=None, already_element=False, threads=16):
        """(ids uint32 [nq,k], dists float32 [nq,k], counts uint32 [nq]): the first min(k, index_len) elements
        i < index_len by (dist_to_element, i).  int8 queries are angular_int elements."""
        n = len(self) if index_len is None else int(index_len)
        qf, qi8, already_element = _queries(queries, already_element)
        nq = qf.shape[0]
        ids = np.empty((nq, k), dtype=np.uint32)
        dists = np.empty((nq, k), dtype=np.float32)
        counts = np.empty(nq, dtype=np.uint32)
        rc = lib().orc_exact_search(self._h, n, _ptr(qf), _ptr(qi8) if qi8 is not None else None, nq,
                                    int(already_element), int(k), max(1, int(threads)), _ptr(ids), _ptr(dists),
                                    _ptr(counts))
        if rc != 0:
            raise NotFinite(lib().orc_last_error().decode())
        return ids, dists, counts


def pack(mask):
    """Bool masks (F, n) -> uint32 words (F, ceil(n / 32)), id i at bit i % 32 of word i // 32 (the C ABI's layout,
    packed here independently of the binding)."""
    mask = np.atleast_2d(np.asarray(mask, dtype=bool))
    f, n = mask.shape
    words = np.zeros((f, (n + 31) // 32), dtype=np.uint32)
    for i in np.nonzero(mask.any(axis=0))[0]:
        words[:, i // 32] |= (mask[:, i].astype(np.uint32) << np.uint32(i % 32))
    return words


class Filtered:
    """An oracle index and element container opened from file images (index, elements, and the embeddings table for
    "embeddings")."""

    def __init__(self, index_bytes, kind, elements_bytes, embeddings_bytes=None):
        self.kind = _kind(kind)
        self._ib = np.frombuffer(bytes(index_bytes), dtype=np.uint8)
        self._eb = np.frombuffer(bytes(elements_bytes), dtype=np.uint8)
        self._mb = np.frombuffer(bytes(embeddings_bytes), dtype=np.uint8) if embeddings_bytes is not None else None
        self._e = _open_elements(self.kind, self._eb, self._mb)
        L = lib()
        self._i = L.orc_index_from_bytes(_ptr(self._ib), self._ib.size)
        if not self._i:
            raise ValueError(L.orc_last_error().decode())

    def __del__(self):
        try:
            if getattr(self, "_e", None):
                lib().orc_elements_free(self._e)
                self._e = None
            if getattr(self, "_i", None):
                lib().orc_index_free(self._i)
                self._i = None
        except Exception:  # interpreter shutdown
            pass

    def __len__(self):
        return int(lib().orc_index_len(self._i))

    def search(self, queries, words, max_search, k, query_filter=None, bit_base=0, already_element=False,
               threads=16):
        """(ids uint32 [nq,k], dists float32 [nq,k], counts uint32 [nq], stats uint64 [nq,3]) of the filtered search
        over the uint32 bitmaps `words` (F, W).  int8 queries are angular_int elements."""
        qf, qi8, already_element = _queries(queries, already_element)
        nq = qf.shape[0]
        words = np.ascontiguousarray(words, dtype=np.uint32)
        sel = None if query_filter is None else np.ascontiguousarray(query_filter, dtype=np.uint32)
        ids = np.empty((nq, k), dtype=np.uint32)
        dists = np.empty((nq, k), dtype=np.float32)
        counts = np.empty(nq, dtype=np.uint32)
        stats = np.empty((nq, 3), dtype=np.uint64)
        rc = lib().orc_filtered_search(self._i, self._e, _ptr(qf), _ptr(qi8) if qi8 is not None else None, nq,
                                       int(already_element), int(max_search), int(k), _ptr(words), words.shape[1],
                                       _ptr(sel) if sel is not None else None, int(bit_base), max(1, int(threads)),
                                       _ptr(ids), _ptr(dists), _ptr(counts), _ptr(stats))
        if rc != 0:
            raise NotFinite(lib().orc_last_error().decode())
        return ids, dists, counts, stats


def table_image(table):
    """FixedWidthSliceVector<f32>::write of an embedding table (u64 width | rows)."""
    table = np.ascontiguousarray(table, dtype=np.float32)
    return np.uint64(table.shape[1]).tobytes() + table.tobytes()


def elements_image(elements):
    """VariableWidthSliceVector<ThreeByteInt, FiveByteInt>::write of term lists: u64 count | (count + 1) five-byte
    offsets | three-byte ids."""
    offsets = np.concatenate([[0], np.cumsum([len(e) for e in elements], dtype=np.uint64)]).astype(np.uint64)
    ids = np.fromiter((t for e in elements for t in e), dtype=np.uint32, count=int(offsets[-1]))
    return elements_image_from_arrays(offsets, ids)


def elements_image_from_arrays(offsets, ids):
    """elements_image of term lists given as n + 1 offsets and the concatenated ids."""
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    off5 = offsets.view(np.uint8).reshape(-1, 8)[:, :5]
    id3 = ids.view(np.uint8).reshape(-1, 4)[:, :3]
    return np.uint64(offsets.size - 1).tobytes() + off5.tobytes() + id3.tobytes()


def compute_embeddings(kind, elements_bytes, embeddings_bytes, threads=1):
    """The elements file image compute_embeddings_and_save_to_disk writes (a uint8 array), for valid images of a
    SumEmbeddings container (elements file, embeddings table); kind "angular_int" (the reference) or "angular"."""
    kind = _kind(kind)
    L = lib()
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    mb = np.frombuffer(embeddings_bytes, dtype=np.uint8)
    h = _open_elements(EMBEDDINGS, eb, mb)
    try:
        n, dim = int(L.orc_elements_len(h)), int(L.orc_elements_dim(h))
        out = np.empty(8 + n * dim * (4 if kind == ANGULAR else 1), dtype=np.uint8)
        size = int(L.orc_compute_embeddings(h, kind, max(1, int(threads)), _ptr(out), out.size))
    finally:
        L.orc_elements_free(h)
    if size < 0:
        raise NotFinite(L.orc_last_error().decode())
    assert size <= out.size
    return out[:size]


def single_layer_index(go, n):
    """An index image with one layer of n nodes, every node listing node 0: Index::len == n, built without a search
    (exact search reads no neighbour list)."""
    import json

    enc = bytes(go.set_encode([0])) if n else b""
    blobs = []
    if n:
        L = len(enc)
        nchunks = 1 + n // 60
        offs = np.arange(n + 1, dtype=np.uint64) * np.uint64(L)  # n + 1 list offsets
        chunk = np.zeros((nchunks, 8 + 120), dtype=np.uint8)
        pad = np.full(nchunks * 60, np.iinfo(np.uint64).max, dtype=np.uint64)
        pad[:n + 1] = offs
        pad = pad.reshape(nchunks, 60)
        initial = pad[:, 0].copy()
        initial[initial == np.iinfo(np.uint64).max] = 0
        chunk[:, :8] = initial.view(np.uint8).reshape(nchunks, 8)
        deltas = np.full((nchunks, 60), 0xFFFF, dtype=np.uint16)
        valid = pad != np.iinfo(np.uint64).max
        prev = np.concatenate([initial[:, None], pad[:, :-1]], axis=1)
        d = (pad - prev).astype(np.uint16)
        deltas[valid] = d[valid]
        chunk[:, 8:] = deltas.view(np.uint8).reshape(nchunks, 120)
        chunks = chunk.tobytes()
        blobs.append(len(chunks).to_bytes(8, "little") + chunks + enc * n)
    meta = "granne" + json.dumps({"compressed": True, "granne_version": "0.5.2",
                                  "layer_counts": [n] if n else [], "layer_sizes": [len(b) for b in blobs],
                                  "num_elements": n, "num_layers": 1 if n else 0,
                                  "num_neighbors": 1 if n else 0, "version": 2}, separators=(",", ":"))
    return meta.encode().ljust(1024, b" ") + b"".join(blobs)
