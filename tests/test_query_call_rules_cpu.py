"""The argument rules the five batched query calls share (graph, exact, two-stage, within-lists and filtered search),
without a device: for arguments that break a rule, the status and the granne_b200_last_error text of each call, and each
call's own rules in the order they are reported; and the stream argument of the Python device calls.  The rules are
checked before the handle is read, so a handle that is never dereferenced serves."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from granne_b200 import api

INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
TOO_MANY = 0xFFFFFFF1

FORMAT = "unknown query format"
MAX_SEARCH = "max_search must be >= 1 (the reference panics on 0, src/index/mod.rs:1019)"
EXACT_K = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)"
NQ = "too many queries in one batch"
NULL = "null buffer"
OFFSETS_NULL = "offsets is null"
IDS_NULL = "ids is null"
FILTERS = "filters is null or num_filters is 0"
ALL_CALLS = ["search", "exact", "rerank", "within", "filtered"]


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _call(lib, call, q=True, nq=2, fmt=api.QUERY_RAW_F32, max_search=50, k=10, ids=True, offsets=(0, 2, 3),
          cand=True, filters=True, num_filters=1):
    """Status and message of `call` (one of ALL_CALLS) on the fake handle; q / ids / cand / filters False, offsets None:
    a null pointer (ids: the output ids, cand: the within lists' ids)."""
    queries = np.zeros((2, 8), np.float32)
    out_ids = np.zeros((2, 2000), np.uint32)
    out_d = np.zeros((2, 2000), np.float32)
    offs = None if offsets is None else np.asarray(offsets, np.uint64)
    cand_ids = np.array([0, 1, 2], np.uint32)
    words = np.ones((2, 4), np.uint32)
    pq, pi, pd = api._ptr(queries) if q else None, api._ptr(out_ids) if ids else None, api._ptr(out_d)
    if call == "search":
        rc = lib.granne_b200_search_batch(FAKE, pq, nq, fmt, max_search, k, pi, pd, None, None)
    elif call == "exact":
        rc = lib.granne_b200_exact_search_batch(FAKE, pq, nq, fmt, k, pi, pd, None)
    elif call == "rerank":
        rc = lib.granne_b200_search_rerank_batch(FAKE, pq, nq, fmt, max_search, 20, k, pi, pd, None, None)
    elif call == "within":
        rc = lib.granne_b200_exact_search_within_batch(FAKE, pq, nq, fmt, api._ptr(offs) if offs is not None else None,
                                                       api._ptr(cand_ids) if cand else None, k, pi, pd, None)
    else:
        rc = lib.granne_b200_search_filtered_batch(FAKE, pq, nq, fmt, max_search, k,
                                                   api._ptr(words) if filters else None, num_filters, 4, None, pi, pd,
                                                   None, None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("call", ALL_CALLS)
def test_shared_rules(lib, call):
    assert _call(lib, call, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, call, nq=TOO_MANY) == (INVALID, NQ)
    assert _call(lib, call, q=False) == (INVALID, NULL)
    assert _call(lib, call, ids=False) == (INVALID, NULL)


@pytest.mark.parametrize("call", ["search", "rerank", "filtered"])
def test_max_search_rule(lib, call):
    assert _call(lib, call, max_search=0) == (INVALID, MAX_SEARCH)
    # reported after the format, before the batch size and the buffers
    assert _call(lib, call, max_search=0, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, call, max_search=0, nq=TOO_MANY, q=False) == (INVALID, MAX_SEARCH)


def test_exact_k_rule(lib):
    for call in ("exact", "within", "filtered"):
        assert _call(lib, call, k=1025) == (INVALID, EXACT_K)
        assert _call(lib, call, k=1025, fmt=7) == (INVALID, FORMAT)
        assert _call(lib, call, k=1025, nq=TOO_MANY, q=False) == (INVALID, EXACT_K)


def test_within_rules_in_order(lib):
    # the exact-k rule, then a null offsets with nq > 0, then null ids when offsets[nq] > 0
    assert _call(lib, "within", k=1025, offsets=None, cand=False) == (INVALID, EXACT_K)
    assert _call(lib, "within", q=False, offsets=None, cand=False) == (INVALID, NULL)
    assert _call(lib, "within", offsets=None, cand=False) == (INVALID, OFFSETS_NULL)
    assert _call(lib, "within", cand=False) == (INVALID, IDS_NULL)


def test_filtered_rules_in_order(lib):
    # max_search, then the exact-k rule, then null or zero filters
    assert _call(lib, "filtered", max_search=0, k=1025, filters=False) == (INVALID, MAX_SEARCH)
    assert _call(lib, "filtered", k=1025, filters=False, num_filters=0) == (INVALID, EXACT_K)
    assert _call(lib, "filtered", q=False, filters=False) == (INVALID, NULL)
    assert _call(lib, "filtered", filters=False) == (INVALID, FILTERS)
    assert _call(lib, "filtered", num_filters=0) == (INVALID, FILTERS)


def test_no_queries_is_ok_before_the_handle_is_read(lib):
    for call in ("search", "exact", "within", "filtered"):
        assert _call(lib, call, nq=0, q=False, ids=False, offsets=None, cand=False, filters=False)[0] == 0


def test_raw_stream():
    class Stream:
        cuda_stream = 0x7F00DEAD0000

    assert api._raw_stream(0x1234, None) == 0x1234
    assert api._raw_stream(0, None) == 0  # the legacy default stream, not "no stream given"
    assert api._raw_stream(Stream(), None) == 0x7F00DEAD0000
