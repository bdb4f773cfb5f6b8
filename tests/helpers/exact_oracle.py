"""ctypes wrapper over tests/helpers/exact_oracle.cpp: the CPU oracle's brute-force k nearest neighbours, the checker
of granne_b200_exact_search_batch.

TEST INFRASTRUCTURE ONLY.  The library is compiled with the oracle's flags (oracle/Makefile) into a temporary directory,
so that the source tree is never written to.  It shares no state with oracle/granne_oracle.py's library: containers
are passed to it as file images."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SOURCES = [os.path.join(_HERE, "exact_oracle.cpp"), os.path.join(_ROOT, "oracle", "granne_oracle.cpp")]
_FLAGS = ["-O3", "-std=c++17", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-pthread", "-shared"]
_KINDS = {"angular": 0, "angular_int": 1, "embeddings": 2}

_lib = None


def build_lib():
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out_dir = os.path.join(tempfile.gettempdir(), "granne_b200_exact_oracle_%d" % os.getuid())
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
        vp = C.c_void_p
        L.orc_last_error.restype = C.c_char_p
        L.orc_elements_from_bytes.restype = vp
        L.orc_elements_from_bytes.argtypes = [C.c_int, vp, C.c_uint64, vp, C.c_uint64]
        L.orc_elements_free.argtypes = [vp]
        L.orc_elements_len.restype = C.c_uint64
        L.orc_elements_len.argtypes = [vp]
        L.orc_elements_dim.restype = C.c_uint64
        L.orc_elements_dim.argtypes = [vp]
        L.orc_exact_search.restype = C.c_int
        L.orc_exact_search.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint64, C.c_int, C.c_uint64, C.c_int, vp, vp, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class NotFinite(ValueError):
    """A distance is NaN: the reference panics."""


class Container:
    """An oracle element container opened from file images (elements file, and the embeddings table for
    "embeddings")."""

    def __init__(self, kind, elements_bytes, embeddings_bytes=None):
        self.kind = _KINDS[kind] if isinstance(kind, str) else int(kind)
        self._eb = np.frombuffer(elements_bytes, dtype=np.uint8)
        self._mb = np.frombuffer(embeddings_bytes, dtype=np.uint8) if embeddings_bytes is not None else None
        L = lib()
        self._h = L.orc_elements_from_bytes(self.kind, _ptr(self._eb), self._eb.size,
                                            _ptr(self._mb) if self._mb is not None else None,
                                            self._mb.size if self._mb is not None else 0)
        if not self._h:
            raise ValueError(L.orc_last_error().decode())

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
        q = np.asarray(queries)
        qi8 = None
        if q.dtype == np.int8:
            qi8 = np.ascontiguousarray(q)
            qf = np.zeros(q.shape, dtype=np.float32)
            already_element = True
        else:
            qf = np.ascontiguousarray(q, dtype=np.float32)
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


def single_layer_index(go, n):
    """An index image with one layer of n nodes, every node listing node 0: Index::len == n, built without a search
    (exact search reads no neighbour list)."""
    import json

    enc =bytes(go.set_encode([0])) if n else b""
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
