"""ctypes wrapper over tests/helpers/filtered_oracle.cpp: filtered search composed from the CPU oracle's descent, its
bottom-layer search_for_neighbors (recording the scored ids), a filter and dist_to_element — the checker of
granne_b200_search_filtered_batch.

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
_SOURCES = [os.path.join(_HERE, "filtered_oracle.cpp"), os.path.join(_ROOT, "oracle", "granne_oracle.cpp")]
_FLAGS = ["-O3", "-std=c++17", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-pthread", "-shared"]
_KINDS = {"angular": 0, "angular_int": 1, "embeddings": 2}

_lib = None


def build_lib():
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out_dir = os.path.join(tempfile.gettempdir(), "granne_b200_filtered_oracle_%d" % os.getuid())
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
        L.orc_index_from_bytes.restype = vp
        L.orc_index_from_bytes.argtypes = [vp, u64]
        L.orc_index_free.argtypes = [vp]
        L.orc_index_len.restype = u64
        L.orc_index_len.argtypes = [vp]
        L.orc_filtered_search.restype = C.c_int
        L.orc_filtered_search.argtypes = [vp, vp, vp, vp, u64, C.c_int, u64, u64, vp, u64, vp, u64, C.c_int, vp, vp,
                                          vp, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class NotFinite(ValueError):
    """A distance the search computes is NaN: the reference panics."""


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
        self.kind = _KINDS[kind] if isinstance(kind, str) else int(kind)
        self._ib = np.frombuffer(bytes(index_bytes), dtype=np.uint8)
        self._eb = np.frombuffer(bytes(elements_bytes), dtype=np.uint8)
        self._mb = np.frombuffer(bytes(embeddings_bytes), dtype=np.uint8) if embeddings_bytes is not None else None
        L = lib()
        self._e = L.orc_elements_from_bytes(self.kind, _ptr(self._eb), self._eb.size,
                                            _ptr(self._mb) if self._mb is not None else None,
                                            self._mb.size if self._mb is not None else 0)
        if not self._e:
            raise ValueError(L.orc_last_error().decode())
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
        q = np.asarray(queries)
        qi8 = None
        if q.dtype == np.int8:
            qi8 = np.ascontiguousarray(q)
            qf = np.zeros(q.shape, dtype=np.float32)
            already_element = True
        else:
            qf = np.ascontiguousarray(q, dtype=np.float32)
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
