"""ctypes wrapper over tests/helpers/embeddings_oracle.cpp: the CPU oracle plus its restatement of
compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152).

TEST INFRASTRUCTURE ONLY.  The library is compiled with the oracle's flags (oracle/Makefile) into a temporary directory,
so that the source tree is never written to."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SOURCES = [os.path.join(_HERE, "embeddings_oracle.cpp"), os.path.join(_ROOT, "oracle", "granne_oracle.cpp")]
_FLAGS = ["-O3", "-std=c++17", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-pthread", "-shared"]
ANGULAR, ANGULAR_INT = 0, 1
_KINDS = {"angular": ANGULAR, "angular_int": ANGULAR_INT}

_lib = None


def build_lib():
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, "rb") as f:
            h.update(f.read())
    out_dir = os.path.join(tempfile.gettempdir(), "granne_b200_embeddings_oracle_%d" % os.getuid())
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
        L.orc_compute_embeddings.restype = C.c_int64
        L.orc_compute_embeddings.argtypes = [vp, C.c_int, C.c_int, vp, C.c_uint64]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


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


class NotFinite(ValueError):
    """The reference panics (angular_int), or the rows would hold NaN (angular)."""


def compute_embeddings(kind, elements_bytes, embeddings_bytes, threads=1):
    """The elements file image compute_embeddings_and_save_to_disk writes (a uint8 array), for valid images of a
    SumEmbeddings container (elements file, embeddings table); kind "angular_int" (the reference) or "angular"."""
    kind = _KINDS[kind] if isinstance(kind, str) else int(kind)
    L = lib()
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    mb = np.frombuffer(embeddings_bytes, dtype=np.uint8)
    h = L.orc_elements_from_bytes(2, _ptr(eb), eb.size, _ptr(mb), mb.size)
    if not h:
        raise ValueError(L.orc_last_error().decode())
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
