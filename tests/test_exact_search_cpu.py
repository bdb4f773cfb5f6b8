"""Exact k nearest neighbours without a device: the brute-force checker (tests/helpers/exact_oracle.cpp) against a
per-pair restatement with the oracle's own distances, and the host-side statuses of the new C entry points."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers import exact_oracle as xo
from helpers.data import random_vectors

INVALID = -1


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _restated(oracle, kind, rows, queries, k, n):
    """sorted((dist_f32 / dist_i8 of the oracle, i) for i < n)[:k], pair by pair."""
    ids = np.full((len(queries), k), 0xFFFFFFFF, np.uint32)
    ds = np.full((len(queries), k), np.inf, np.float32)
    for qi, q in enumerate(queries):
        if kind == "angular":
            qq = oracle.normalize_f32(np.array(q, np.float32))
            pairs = sorted((float(oracle.dist_f32(rows[i], qq)), i) for i in range(n))
        else:
            qq = q if q.dtype == np.int8 else oracle.quantize_i8(q)
            pairs = sorted((float(oracle.dist_i8(rows[i], qq)), i) for i in range(n))
        for r, (d, i) in enumerate(pairs[:k]):
            ids[qi, r], ds[qi, r] = i, d
    return ids, ds, np.full(len(queries), min(k, n), np.uint32)


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("k,n", [(5, 60), (70, 60), (3, 0), (4, 1)])
def test_checker_equals_a_per_pair_restatement(oracle, kind, k, n):
    raw = random_vectors(60, 37, 3)
    raw[10] = raw[11]  # ties: duplicate rows
    raw[20] = 0.0      # an all-zero row
    el = oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)
    rows = el.rows()
    c = xo.Container(kind, el.to_bytes(0))
    q = np.concatenate([random_vectors(4, 37, 4), raw[10:11]])
    got = c.exact_search(q, k, index_len=n)
    want = _restated(oracle, kind, rows, q, k, n)
    for g, w in zip(got, want):
        assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w).view(np.uint32))


def test_checker_raises_on_nan(oracle):
    raw = random_vectors(30, 16, 1)
    el = oracle.Elements.angular(raw, as_is=True)
    bad = raw.copy()
    bad[7, 2] = np.nan
    c = xo.Container("angular", np.uint64(16).tobytes() + bad.tobytes())
    with pytest.raises(xo.NotFinite):
        c.exact_search(random_vectors(2, 16, 2), 5)
    assert len(el) == 30


def test_symbols_exported():
    L = granne_b200.load_library()
    for name in ("granne_b200_exact_search_batch", "granne_b200_exact_search_batch_device",
                 "granne_b200_multi_exact_search_batch"):
        assert hasattr(L, name)
    assert api.EXACT_MAX_K == 1024


def test_host_side_statuses():
    L = granne_b200.load_library()
    q = np.zeros((2, 8), np.float32)
    ids = np.zeros((2, 2000), np.uint32)
    ds = np.zeros((2, 2000), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert L.granne_b200_exact_search_batch(None, p(q), 2, 0, 10, p(ids), p(ds), None) == INVALID
    assert L.granne_b200_exact_search_batch_device(None, p(q), 2, 0, 10, p(ids), p(ds), None, None) == INVALID
    assert L.granne_b200_multi_exact_search_batch(None, p(q), 2, 0, 10, None, None, None) == INVALID
    # a non-null handle that is never dereferenced: the format and k checks come first and need no device
    fake = C.c_void_p(1)
    assert L.granne_b200_exact_search_batch(fake, p(q), 2, 7, 10, p(ids), p(ds), None) == INVALID
    assert L.granne_b200_exact_search_batch(fake, p(q), 2, 0, 1025, p(ids), p(ds), None) == INVALID
    assert L.granne_b200_exact_search_batch_device(fake, p(q), 2, 0, 1025, p(ids), p(ds), None, None) == INVALID
    assert L.granne_b200_exact_search_batch(fake, None, 2, 0, 10, p(ids), p(ds), None) == INVALID
    assert L.granne_b200_exact_search_batch(fake, p(q), 2, 0, 10, None, p(ds), None) == INVALID
    assert L.granne_b200_exact_search_batch(fake, p(q), 0, 0, 10, None, None, None) == 0  # nq == 0
