"""ctypes wrapper over oracle/libgranne_oracle.so — the CPU restatement of granne's search path.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` legs.  The product package (granne_b200/) never imports this module.

The class surface mirrors the reference's Python module (py/src/lib.rs:149-344 `Granne`, :346-579
`GranneBuilder`) closely enough that the parity tests read like the reference's own tests.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgranne_oracle.so")

ANGULAR, ANGULAR_INT, EMBEDDINGS = 0, 1, 2
_KINDS = {"angular": ANGULAR, "angular_int": ANGULAR_INT, "embeddings": EMBEDDINGS}
UNUSED = 0xFFFFFFFF


def build_lib(force=False):
    """Compile the oracle with oracle/Makefile (g++ only; no reference sources are compiled)."""
    src = os.path.join(_HERE, "granne_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    build_lib()
    L = C.CDLL(_LIB_PATH)
    vp, u64, i64, f32, i32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_float, C.c_int
    sig = {
        "orc_last_error": (C.c_char_p, []),
        "orc_num_elements_in_layer": (u64, [u64, f32, u64]),
        "orc_dot_f32": (f32, [vp, vp, u64]),
        "orc_normalize_f32": (None, [vp, u64]),
        "orc_sum_into_f32": (None, [vp, vp, u64]),
        "orc_dist_f32": (f32, [vp, vp, u64]),
        "orc_dist_i8": (f32, [vp, vp, u64]),
        "orc_quantize_i8": (None, [vp, u64, vp]),
        "orc_dot_i8": (None, [vp, vp, u64, vp]),
        "orc_read_uint": (u64, [vp, i32]),
        "orc_write_uint": (None, [vp, u64, i32]),
        "orc_set_encode": (u64, [vp, u64, vp, u64]),
        "orc_set_decode": (u64, [vp, u64, vp, u64]),
        "orc_delta_encode": (None, [vp, u64]),
        "orc_elements_new": (vp, [i32, u64]),
        "orc_elements_free": (None, [vp]),
        "orc_elements_len": (u64, [vp]),
        "orc_elements_dim": (u64, [vp]),
        "orc_elements_push_f32": (None, [vp, vp, u64, i32]),
        "orc_elements_push_i8": (None, [vp, vp, u64]),
        "orc_sum_push_embeddings": (None, [vp, vp, u64]),
        "orc_sum_push_element": (None, [vp, vp, u64]),
        "orc_elements_data": (vp, [vp]),
        "orc_sum_num_embeddings": (u64, [vp]),
        "orc_sum_terms": (u64, [vp, u64, vp, u64]),
        "orc_elements_get": (None, [vp, u64, vp]),
        "orc_elements_dist_to": (f32, [vp, u64, vp, i32]),
        "orc_elements_serialize": (u64, [vp, i32, vp, u64]),
        "orc_elements_from_bytes": (vp, [i32, vp, u64, vp, u64]),
        "orc_index_free": (None, [vp]),
        "orc_index_from_bytes": (vp, [vp, u64]),
        "orc_build": (vp, [vp, u64, u64, f32, i32, i64, u64, i32]),
        "orc_index_serialize": (u64, [vp, vp, u64]),
        "orc_index_to_fixed": (vp, [vp]),
        "orc_index_len": (u64, [vp]),
        "orc_index_num_layers": (u64, [vp]),
        "orc_index_layer_len": (u64, [vp, u64]),
        "orc_index_get_neighbors": (u64, [vp, u64, u64, vp, u64]),
        "orc_offsets_roundtrip": (i64, [vp, u64, vp, vp]),
        "orc_multiset_blob": (u64, [vp, vp, u64, vp, u64]),
        "orc_multiset_len": (i64, [vp, u64]),
        "orc_multiset_get": (u64, [vp, u64, u64, vp, u64]),
        "orc_select_neighbors": (u64, [vp, vp, vp, u64, u64, vp, vp]),
        "orc_builder_new": (vp, [vp, u64, u64, f32, i32, i64]),
        "orc_builder_free": (None, [vp]),
        "orc_builder_from_index": (vp, [vp, vp, u64, u64, f32, i32, i64]),
        "orc_builder_build_partial": (i32, [vp, u64, i32]),
        "orc_builder_set_max_batch": (None, [vp, u64]),
        "orc_builder_counters": (None, [vp, vp]),
        "orc_elements_dists": (None, [vp, u64, vp, u64, vp]),
        "orc_builder_get_index": (vp, [vp]),
        "orc_entrypoint_trail": (None, [vp, vp, u64, u64, vp]),
        "orc_compute_order": (None, [vp, vp, vp, i32]),
        "orc_order_by_keys": (None, [vp, vp, u64, vp]),
        "orc_index_apply_order": (vp, [vp, vp, u64]),
        "orc_elements_permute": (None, [vp, vp, u64]),
        "orc_sum_reorder_keys": (None, [vp, vp]),
        "orc_search_batch": (i32, [vp, vp, vp, vp, u64, i32, u64, u64, vp, vp, vp, vp, i32]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


# ---- KAT helpers -------------------------------------------------------------------------------------------------
def num_elements_in_layer(total, multiplier, layer):
    return int(lib().orc_num_elements_in_layer(total, multiplier, layer))


def dot_product_f32(x, y):
    x, y = _f32(x), _f32(y)
    return float(np.float32(lib().orc_dot_f32(_ptr(x), _ptr(y), x.size)))


def normalize_f32(x):
    x = _f32(x).copy()
    lib().orc_normalize_f32(_ptr(x), x.size)
    return x


def sum_into_f32(x, y):
    x, y = _f32(x).copy(), _f32(y)
    lib().orc_sum_into_f32(_ptr(x), _ptr(y), x.size)
    return x


def dist_f32(x, y):
    x, y = _f32(x), _f32(y)
    return np.float32(lib().orc_dist_f32(_ptr(x), _ptr(y), x.size))


def quantize_i8(x):
    x = _f32(x)
    out = np.empty(x.size, dtype=np.int8)
    lib().orc_quantize_i8(_ptr(x), x.size, _ptr(out))
    return out


def dist_i8(x, y):
    x = np.ascontiguousarray(x, dtype=np.int8)
    y = np.ascontiguousarray(y, dtype=np.int8)
    return np.float32(lib().orc_dist_i8(_ptr(x), _ptr(y), x.size))


def dot_i8(x, y):
    x = np.ascontiguousarray(x, dtype=np.int8)
    y = np.ascontiguousarray(y, dtype=np.int8)
    out = np.zeros(3, dtype=np.int32)
    lib().orc_dot_i8(_ptr(x), _ptr(y), x.size, _ptr(out))
    return tuple(int(v) for v in out)


def read_uint(b, nbytes):
    a = np.frombuffer(bytes(b), dtype=np.uint8)
    return int(lib().orc_read_uint(_ptr(a), nbytes))


def write_uint(v, nbytes):
    a = np.zeros(nbytes, dtype=np.uint8)
    lib().orc_write_uint(_ptr(a), v, nbytes)
    return a.tobytes()


def set_encode(sorted_ids):
    ids = np.ascontiguousarray(sorted_ids, dtype=np.uint32)
    out = np.zeros(8 + 5 * max(4, ids.size), dtype=np.uint8)
    n = lib().orc_set_encode(_ptr(ids), ids.size, _ptr(out), out.size)
    return out[:n].tobytes()


def set_decode(enc):
    a = np.frombuffer(bytes(enc), dtype=np.uint8)
    out = np.zeros(260, dtype=np.uint32)
    n = lib().orc_set_decode(_ptr(a), a.size, _ptr(out), out.size)
    return out[:n].tolist()


def delta_encode(ids):
    a = np.ascontiguousarray(ids, dtype=np.uint32).copy()
    lib().orc_delta_encode(_ptr(a), a.size)
    return a.tolist()


def offsets_roundtrip(offsets):
    """Offsets::push for every value, then Offsets::len / get / last (offsets.rs:225-270).  Returns
    (len, values read back, last() after each push), or None where the reference panics."""
    a = np.ascontiguousarray(offsets, dtype=np.uint64)
    out = np.zeros(a.size, dtype=np.uint64)
    last = np.zeros(a.size, dtype=np.uint64)
    n = int(lib().orc_offsets_roundtrip(_ptr(a), a.size, _ptr(out), _ptr(last)))
    if n < 0:
        return None
    return n, out[:n].tolist(), last.tolist()


class MultiSetVector:
    """MultiSetVector written by write_as_multi_set_vector (set_vector.rs:169-221) and loaded with from_bytes."""

    def __init__(self, lists):
        flat = np.ascontiguousarray([v for l in lists for v in l], dtype=np.uint32)
        lens = np.ascontiguousarray([len(l) for l in lists], dtype=np.uint64)
        if flat.size == 0:
            flat = np.zeros(1, dtype=np.uint32)
        if lens.size == 0:
            lens = np.zeros(1, dtype=np.uint64)
        n = lib().orc_multiset_blob(_ptr(flat), _ptr(lens), len(lists), None, 0)
        self.blob = np.zeros(n, dtype=np.uint8)
        lib().orc_multiset_blob(_ptr(flat), _ptr(lens), len(lists), _ptr(self.blob), n)

    def __len__(self):
        return int(lib().orc_multiset_len(_ptr(self.blob), self.blob.size))

    def get(self, idx):
        out = np.zeros(300, dtype=np.uint32)
        n = int(lib().orc_multiset_get(_ptr(self.blob), self.blob.size, idx, _ptr(out), out.size))
        return out[:n].tolist()


def select_neighbors(elements, candidates, max_neighbors):
    """GranneBuilder::select_neighbors (index/mod.rs:849-883); candidates = [(id, dist)] ascending by distance."""
    ids = np.ascontiguousarray([c[0] for c in candidates], dtype=np.uint64)
    ds = np.ascontiguousarray([c[1] for c in candidates], dtype=np.float32)
    oi = np.zeros(max(1, len(candidates)), dtype=np.uint64)
    od = np.zeros(max(1, len(candidates)), dtype=np.float32)
    n = int(lib().orc_select_neighbors(elements._h, _ptr(ids), _ptr(ds), len(candidates), max_neighbors, _ptr(oi),
                                       _ptr(od)))
    return [(int(oi[i]), float(od[i])) for i in range(n)]


# ---- element containers ------------------------------------------------------------------------------------------
class Elements:
    """angular::Vectors / angular_int::Vectors / embeddings::SumEmbeddings (src/elements/)."""

    def __init__(self, kind, dim, _handle=None):
        self.kind = _KINDS[kind] if isinstance(kind, str) else kind
        self._h = _handle if _handle is not None else lib().orc_elements_new(self.kind, dim)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().orc_elements_free(self._h)
                self._h = None
        except Exception:  # interpreter shutdown
            pass

    @classmethod
    def angular(cls, raw, as_is=False):
        raw = _f32(raw)
        e = cls(ANGULAR, raw.shape[1])
        lib().orc_elements_push_f32(e._h, _ptr(raw), raw.shape[0], int(as_is))
        return e

    @classmethod
    def angular_int(cls, raw):
        """raw f32 rows are quantised (angular_int.rs:28-45); int8 rows are stored as is."""
        raw = np.asarray(raw)
        e = cls(ANGULAR_INT, raw.shape[1])
        if raw.dtype == np.int8:
            raw = np.ascontiguousarray(raw)
            lib().orc_elements_push_i8(e._h, _ptr(raw), raw.shape[0])
        else:
            raw = _f32(raw)
            lib().orc_elements_push_f32(e._h, _ptr(raw), raw.shape[0], 0)
        return e

    @classmethod
    def sum_embeddings(cls, embeddings, elements):
        embeddings = _f32(embeddings)
        e = cls(EMBEDDINGS, embeddings.shape[1])
        lib().orc_sum_push_embeddings(e._h, _ptr(embeddings), embeddings.shape[0])
        for el in elements:
            ids = np.ascontiguousarray(el, dtype=np.uint32)
            lib().orc_sum_push_element(e._h, _ptr(ids), ids.size)
        return e

    @classmethod
    def from_bytes(cls, kind, elements_bytes, embeddings_bytes=None):
        kind = _KINDS[kind] if isinstance(kind, str) else kind
        a = np.frombuffer(elements_bytes, dtype=np.uint8)
        if embeddings_bytes is not None:
            b = np.frombuffer(embeddings_bytes, dtype=np.uint8)
            h = lib().orc_elements_from_bytes(kind, _ptr(a), a.size, _ptr(b), b.size)
        else:
            h = lib().orc_elements_from_bytes(kind, _ptr(a), a.size, None, 0)
        if not h:
            raise ValueError(lib().orc_last_error().decode())
        return cls(kind, 0, _handle=h)

    def __len__(self):
        return int(lib().orc_elements_len(self._h))

    @property
    def dim(self):
        return int(lib().orc_elements_dim(self._h))

    def get(self, idx):
        out = np.empty(self.dim, dtype=np.int8 if self.kind == ANGULAR_INT else np.float32)
        lib().orc_elements_get(self._h, idx, _ptr(out))
        return out

    def rows(self):
        """The stored rows (f32/i8 vectors, or the embedding table for SumEmbeddings) as a numpy copy."""
        n = int(lib().orc_sum_num_embeddings(self._h)) if self.kind == EMBEDDINGS else len(self)
        p = lib().orc_elements_data(self._h)
        if self.kind == ANGULAR_INT:
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int8)), shape=(n, self.dim)).copy()
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(n, self.dim)).copy()

    def dists(self, idx, ids):
        """dist(ids[k], element idx) for every k: the distances a builder sorts node idx's row by
        (index/mod.rs:938)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        out = np.zeros(ids.size, dtype=np.float32)
        if ids.size:
            lib().orc_elements_dists(self._h, idx, _ptr(ids), ids.size, _ptr(out))
        return out

    def dist_to_element(self, idx, raw_query, already_element=False):
        q = _f32(raw_query)
        return np.float32(lib().orc_elements_dist_to(self._h, idx, _ptr(q), int(already_element)))

    def push(self, raw, as_is=False):
        """ExtendableElementContainer::push for the vector containers: rows of raw f32 become elements
        (`Vector::from`: normalised / quantised) and are appended (dense_vector.rs:120-136)."""
        raw = _f32(np.atleast_2d(raw))
        lib().orc_elements_push_f32(self._h, _ptr(raw), raw.shape[0], int(as_is))

    def terms(self, idx):
        """SumEmbeddings::get_terms (embeddings/mod.rs:106-108)."""
        out = np.zeros(256, dtype=np.uint32)
        n = int(lib().orc_sum_terms(self._h, idx, _ptr(out), out.size))
        return out[:n].tolist()

    def permute(self, permutation):
        """Permutable::permute (slice_vector/mod.rs:437-458, embeddings/mod.rs:191-217): new i = old permutation[i]."""
        perm = np.ascontiguousarray(permutation, dtype=np.uint64)
        assert perm.size == len(self)
        lib().orc_elements_permute(self._h, _ptr(perm), perm.size)

    def reorder_keys(self):
        """embeddings::compute_keys_for_reordering (embeddings/reorder.rs:31-58) -> uint64 [n, 8]."""
        assert self.kind == EMBEDDINGS
        keys = np.zeros((len(self), 8), dtype=np.uint64)
        lib().orc_sum_reorder_keys(self._h, _ptr(keys))
        return keys

    def to_bytes(self, which=0):
        """io::Writeable::write.  which=1: the SumEmbeddings embeddings table."""
        n = lib().orc_elements_serialize(self._h, which, None, 0)
        out = np.empty(n, dtype=np.uint8)
        lib().orc_elements_serialize(self._h, which, _ptr(out), n)
        return out.tobytes()


# ---- index -------------------------------------------------------------------------------------------------------
class Granne:
    """granne::Granne (src/index/mod.rs:38-160) over the oracle."""

    def __init__(self, handle, elements):
        self._h = handle
        self.elements = elements

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().orc_index_free(self._h)
                self._h = None
        except Exception:  # interpreter shutdown
            pass

    @classmethod
    def from_bytes(cls, index_bytes, elements):
        a = np.frombuffer(index_bytes, dtype=np.uint8)
        h = lib().orc_index_from_bytes(_ptr(a), a.size)
        if not h:
            raise ValueError(lib().orc_last_error().decode())
        return cls(h, elements)

    def to_fixed(self):
        """Pre-decoded adjacency (the 'strong' CPU baseline variant, BASELINE.md §3)."""
        return Granne(lib().orc_index_to_fixed(self._h), self.elements)

    def __len__(self):
        return int(lib().orc_index_len(self._h))

    def num_layers(self):
        return int(lib().orc_index_num_layers(self._h))

    def layer_len(self, layer):
        return int(lib().orc_index_layer_len(self._h, layer))

    def get_neighbors(self, idx, layer=None):
        if layer is None:
            layer = self.num_layers() - 1
        out = np.zeros(256, dtype=np.uint32)
        n = lib().orc_index_get_neighbors(self._h, idx, layer, _ptr(out), out.size)
        return out[:n].tolist()

    def to_bytes(self):
        """Index::write_index (src/index/io.rs:11-70)."""
        n = lib().orc_index_serialize(self._h, None, 0)
        out = np.empty(n, dtype=np.uint8)
        lib().orc_index_serialize(self._h, _ptr(out), n)
        return out.tobytes()

    # ---- reorder (src/index/reorder.rs) ----
    def entrypoint_trail(self, idx, max_layer):
        """find_entrypoint_trail (reorder.rs:180-207) for element idx."""
        out = np.zeros(8, dtype=np.uint32)
        lib().orc_entrypoint_trail(self._h, self.elements._h, idx, max_layer, _ptr(out))
        return out

    def compute_order(self, threads=1):
        """Granne::compute_order (reorder.rs:126-174)."""
        order = np.zeros(len(self), dtype=np.uint64)
        lib().orc_compute_order(self._h, self.elements._h, _ptr(order), threads)
        return order

    def order_by_keys(self, keys):
        """The ordering part of Granne::reorder_by_keys (reorder.rs:96-108); keys uint64 [n] or [n, kw]."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64).reshape(len(self), -1)
        order = np.zeros(len(self), dtype=np.uint64)
        lib().orc_order_by_keys(self._h, _ptr(keys), keys.shape[1], _ptr(order))
        return order

    def _apply(self, order):
        order = np.ascontiguousarray(order, dtype=np.uint64)
        new = lib().orc_index_apply_order(self._h, _ptr(order), order.size)
        lib().orc_index_free(self._h)
        self._h = new
        self.elements.permute(order)
        return order

    def reorder(self, threads=1):
        """Granne::reorder (reorder.rs:59-82): reorders this index AND its elements in place; returns the order."""
        return self._apply(self.compute_order(threads))

    def reorder_by_keys(self, keys):
        """Granne::reorder_by_keys (reorder.rs:89-124)."""
        return self._apply(self.order_by_keys(keys))

    def search_batch(self, queries, max_search=200, num_neighbors=10, already_element=False, threads=1,
                     with_stats=False):
        """Runs Granne::search for every row of `queries` (raw f32; normalised/quantised like the reference's
        Python binding does, py/src/variants/index.rs:15-16,32-33) — or, with already_element, rows that are
        already elements (normalised f32 / int8)."""
        L = lib()
        q = np.asarray(queries)
        qi8 = None
        if q.dtype == np.int8:
            qi8 = np.ascontiguousarray(q)
            qf = np.zeros((q.shape[0], q.shape[1]), dtype=np.float32)
            already_element = True
        else:
            qf = _f32(q)
        nq = qf.shape[0]
        ids = np.empty((nq, num_neighbors), dtype=np.uint32)
        dists = np.empty((nq, num_neighbors), dtype=np.float32)
        counts = np.empty(nq, dtype=np.uint32)
        stats = np.zeros((nq, 3), dtype=np.uint64)
        rc = L.orc_search_batch(self._h, self.elements._h, _ptr(qf), _ptr(qi8) if qi8 is not None else None, nq,
                                int(already_element), max_search, num_neighbors, _ptr(ids), _ptr(dists),
                                _ptr(counts), _ptr(stats), threads)
        if rc != 0:
            raise ValueError(L.orc_last_error().decode())
        if with_stats:
            return ids, dists, counts, stats
        return ids, dists, counts

    def search(self, element, max_search=200, num_elements=10):
        ids, dists, counts = self.search_batch(np.asarray(element)[None, :], max_search, num_elements)
        return [(int(ids[0, i]), float(dists[0, i])) for i in range(counts[0])]


class GranneBuilder:
    """granne::GranneBuilder (src/index/mod.rs:295-531) — fixture generator."""

    def __init__(self, elements, num_neighbors=30, max_search=200, layer_multiplier=15.0, reinsert_elements=True,
                 expected_num_elements=None):
        self.elements = elements
        self.cfg = (num_neighbors, max_search, layer_multiplier, reinsert_elements,
                    -1 if expected_num_elements is None else expected_num_elements)

    def build(self, num_elements=0, threads=1):
        m, ef, mult, re, exp = self.cfg
        h = lib().orc_build(self.elements._h, m, ef, mult, int(re), exp, num_elements, threads)
        return Granne(h, self.elements)

    @classmethod
    def from_index(cls, index, elements, **config):
        """GranneBuilder::from_bytes (index/mod.rs:428-457): continue building from `index` with a new config."""
        b = cls(elements, **config)
        m, ef, mult, re, exp = b.cfg
        b._b = lib().orc_builder_from_index(index._h, elements._h, m, ef, mult, int(re), exp)
        return b

    # stateful use, like the reference's builder: build_partial(n) continues from what is already indexed
    def build_partial(self, num_elements, threads=1, max_batch=0):
        """Builder::build_partial (index/mod.rs:374-402); returns the index built so far (get_index).
        max_batch > 0 follows the product's batch schedule instead (see build_batched)."""
        if getattr(self, "_b", None) is None:
            m, ef, mult, re, exp = self.cfg
            self._b = lib().orc_builder_new(self.elements._h, m, ef, mult, int(re), exp)
        lib().orc_builder_set_max_batch(self._b, max_batch)
        if lib().orc_builder_build_partial(self._b, num_elements, threads) != 0:
            raise ValueError(lib().orc_last_error().decode())
        return Granne(lib().orc_builder_get_index(self._b), self.elements)

    def build_batched(self, max_batch, threads=1):
        """NOT a reference behaviour: the product's batched build (granne_b200.cu builder_index_elements) with its
        link phase serialized.  Each batch of up to `max_batch` insertions searches one snapshot of the layer, then its
        members are linked one after another in batch order.  `threads` only spreads the searches of a batch; the image
        does not depend on it.  Returns the index; counters() tells what the build did."""
        return self.build_partial(len(self.elements), threads, max_batch)

    def counters(self):
        """What the batched builds of this builder did so far (build_batched / build_partial with max_batch)."""
        out = np.zeros(6, dtype=np.uint64)
        if getattr(self, "_b", None) is not None:
            lib().orc_builder_counters(self._b, _ptr(out))
        keys = ("batches", "max_batch", "connect_present", "connect_overflow", "nontrivial_selects",
                "max_batch_in_links")
        return {k: int(v) for k, v in zip(keys, out)}

    def __del__(self):
        try:
            if getattr(self, "_b", None):
                lib().orc_builder_free(self._b)
                self._b = None
        except Exception:  # interpreter shutdown
            pass
