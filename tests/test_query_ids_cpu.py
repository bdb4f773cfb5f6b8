"""Queries by element id without a device: which calls accept GRANNE_B200_QUERY_ID (2) and _ID_EXCLUDING (3), the
exclusion rule on k and its place in each call's order, null ids, the new ABI symbols and constants in the C header,
the C++ header and the Rust shim, and the Python argument checks.  The rules are checked before the handle is read,
so a handle that is never dereferenced serves."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.fixtures import compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

INVALID = -1
FAKE = C.c_void_p(1)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMAT = "unknown query format"
NULL = "null buffer"
EXCL_K = "num_neighbors exceeds 1023 with GRANNE_B200_QUERY_ID_EXCLUDING (the call runs k + 1)"
EXACT_K = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)"
OFFSETS_NULL = "offsets is null"
FILTERS = "filters is null or num_filters is 0"


def _call(lib, call, fmt, k=10, nq=2, q=True, offsets=True, filters=True):
    ids = np.array([0, 1], np.uint32)
    out_ids = np.zeros((2, 2000), np.uint32)
    out_d = np.zeros((2, 2000), np.float32)
    offs = np.array([0, 1, 2], np.uint64)
    words = np.ones((1, 4), np.uint32)
    pq, pi, pd = api._ptr(ids) if q else None, api._ptr(out_ids), api._ptr(out_d)
    if call == "search":
        rc = lib.granne_b200_search_batch(FAKE, pq, nq, fmt, 50, k, pi, pd, None, None)
    elif call == "search_device":
        rc = lib.granne_b200_search_batch_device(FAKE, pq, nq, fmt, 50, k, pi, pd, None, None, None)
    elif call == "gather":
        g = api.PeerGather()
        rc = lib.granne_b200_search_batch_device_gather(FAKE, pq, nq, fmt, 50, k, C.byref(g), None, None, None)
    elif call == "exact":
        rc = lib.granne_b200_exact_search_batch(FAKE, pq, nq, fmt, k, pi, pd, None)
    elif call == "exact_device":
        rc = lib.granne_b200_exact_search_batch_device(FAKE, pq, nq, fmt, k, pi, pd, None, None)
    elif call == "rerank":
        rc = lib.granne_b200_search_rerank_batch(FAKE, pq, nq, fmt, 50, 20, k, pi, pd, None, None)
    elif call == "rerank_device":
        rc = lib.granne_b200_search_rerank_batch_device(FAKE, pq, nq, fmt, 50, 20, k, pi, pd, None, None, None)
    elif call == "within":
        rc = lib.granne_b200_exact_search_within_batch(FAKE, pq, nq, fmt, api._ptr(offs) if offsets else None,
                                                       api._ptr(ids), k, pi, pd, None)
    elif call == "within_device":
        rc = lib.granne_b200_exact_search_within_batch_device(FAKE, pq, nq, fmt, api._ptr(offs) if offsets else None,
                                                              api._ptr(ids), k, pi, pd, None, None)
    elif call == "filtered":
        rc = lib.granne_b200_search_filtered_batch(FAKE, pq, nq, fmt, 50, k, api._ptr(words) if filters else None, 1,
                                                   4, None, pi, pd, None, None)
    else:
        rc = lib.granne_b200_search_filtered_batch_device(FAKE, pq, nq, fmt, 50, k,
                                                          api._ptr(words) if filters else None, 1, 4, None, pi, pd,
                                                          None, None, None)
    return rc, lib.granne_b200_last_error().decode()


ACCEPTING = ["search", "search_device", "exact", "exact_device", "within", "within_device", "filtered",
             "filtered_device"]


@pytest.mark.parametrize("call", ACCEPTING)
def test_id_formats_pass_the_shared_rules(library, call):
    # with nq = 0 a call that takes the format returns OK before it reads the handle
    for fmt in (api.QUERY_ID, api.QUERY_ID_EXCLUDING):
        assert _call(library, call, fmt, nq=0, q=False)[0] == 0
        assert _call(library, call, fmt, q=False) == (INVALID, NULL)  # null ids
    assert _call(library, call, 4) == (INVALID, FORMAT)


@pytest.mark.parametrize("call", ["gather", "rerank", "rerank_device"])
def test_gather_and_rerank_reject_id_formats(library, call):
    for fmt in (api.QUERY_ID, api.QUERY_ID_EXCLUDING):
        assert _call(library, call, fmt, nq=0, q=False) == (INVALID, FORMAT)


@pytest.mark.parametrize("call", ["exact", "exact_device", "within", "within_device", "filtered", "filtered_device"])
def test_exclusion_k_rule_and_order(library, call):
    X = api.QUERY_ID_EXCLUDING
    assert _call(library, call, X, k=1024, nq=0, q=False) == (INVALID, EXCL_K)
    assert _call(library, call, X, k=1023, nq=0, q=False)[0] == 0
    assert _call(library, call, api.QUERY_ID, k=1024, nq=0, q=False)[0] == 0
    # after the existing rules: the cap itself, null buffers, null offsets / filters
    assert _call(library, call, X, k=1025) == (INVALID, EXACT_K)
    assert _call(library, call, X, k=1024, q=False) == (INVALID, NULL)
    if call.startswith("within"):
        assert _call(library, call, X, k=1024, offsets=False) == (INVALID, OFFSETS_NULL)
    if call.startswith("filtered"):
        assert _call(library, call, X, k=1024, filters=False) == (INVALID, FILTERS)


def test_search_has_no_exclusion_cap_below_u32(library):
    assert _call(library, "search", api.QUERY_ID_EXCLUDING, k=5000, nq=0, q=False)[0] == 0
    assert _call(library, "search", api.QUERY_ID_EXCLUDING, k=0xFFFFFFFF, nq=0, q=False)[0] == INVALID


def test_get_elements_null_and_empty(library):
    assert library.granne_b200_get_elements(None, None, 0, None) == INVALID
    assert library.granne_b200_get_elements(FAKE, None, 3, None) == INVALID
    assert library.granne_b200_get_elements_device(None, None, 0, None, None) == INVALID
    assert library.granne_b200_get_elements_device(FAKE, None, 0, None, None) == 0


def test_abi_symbols_and_constants(library):
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    assert re.search(r"#define GRANNE_B200_QUERY_ID 2\b", header)
    assert re.search(r"#define GRANNE_B200_QUERY_ID_EXCLUDING 3\b", header)
    assert "#define GRANNE_B200_ABI_VERSION 2 " in header
    raw = C.CDLL(granne_b200.library_path())
    assert hasattr(raw, "granne_b200_get_elements") and hasattr(raw, "granne_b200_get_elements_device")
    shim = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    assert "pub const QUERY_ID: c_int = 2;" in shim and "pub const QUERY_ID_EXCLUDING: c_int = 3;" in shim
    assert "fn granne_b200_get_elements(" in shim and "fn granne_b200_get_elements_device(" in shim
    assert (api.QUERY_ID, api.QUERY_ID_EXCLUDING) == (2, 3)


def test_cxx_ids_client_compiles(library, tmp_path):
    compile_cxx_client("cxx_ids_client.cpp", tmp_path)


class _Fake(api.Granne):
    """A Granne whose handle is never used: the Python checks run before any library call."""

    def __init__(self):
        self._h = None
        self.device = 0

    @property
    def dim(self):
        return 8

    @property
    def element_kind(self):
        return api.ANGULAR


@pytest.mark.parametrize("bad", [np.zeros((2, 2), np.uint32), np.array([1.5, 2.0]), np.array([-1, 2]),
                                 np.array([2**32], np.uint64)])
def test_python_id_checks(bad):
    g = _Fake()
    for fn in (lambda: g.search_batch(bad, by_id=True), lambda: g.exact_search_batch(bad, exclude_self=True),
               lambda: g.exact_search_within(bad, [[0]] * len(np.atleast_1d(bad)), by_id=True),
               lambda: g.search_batch_filtered(bad, np.ones(8, bool), by_id=True), lambda: g.get_elements(bad)):
        with pytest.raises(ValueError):
            fn()


def test_python_exclude_self_implies_ids():
    assert api._id_queries(np.array([1, 2], np.int64), True, np.uint32)[1] == api.QUERY_ID_EXCLUDING
    q, fmt = _Fake()._host_queries(np.array([3, 4]), False, False, True)
    assert fmt == api.QUERY_ID_EXCLUDING and q.dtype == np.uint32
    # multi handles take uint64 global ids
    assert api._id_queries(np.array([2**40]), False, np.uint64)[0].dtype == np.uint64


def test_python_device_ids_must_be_int32_cuda():
    g = _Fake()
    with pytest.raises(ValueError):
        g.search_batch_device(np.array([1, 2], np.int32), by_id=True)
    with pytest.raises(ValueError):
        g.get_elements_device(np.array([1, 2], np.int32))


def test_stream_status_of_and_part_len(library):
    assert library.granne_b200_stream_status_of(None, None) == INVALID
    assert library.granne_b200_multi_part_len(None, 0) == 0
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    assert "int granne_b200_stream_status_of(granne_b200_index* h, void* cuda_stream);" in header
    assert "fn granne_b200_multi_part_len(" in open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()


def test_knn_graph_chunk_must_be_positive():
    m = api.MultiGranne.__new__(api.MultiGranne)
    m._h = None
    with pytest.raises(ValueError):
        m.knn_graph(chunk=0)
    with pytest.raises(ValueError):
        _Fake().knn_graph(chunk=0)
    cxx = open(os.path.join(ROOT, "include", "granne_b200.hpp")).read()
    assert 'if (chunk == 0) throw Error(GRANNE_B200_ERR_INVALID_ARGUMENT, "chunk must be >= 1");' in cxx
