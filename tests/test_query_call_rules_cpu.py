"""The argument rules the three batched query calls share (graph, exact and two-stage search), without a device: for
arguments that break a rule, the status and the granne_b200_last_error text of each call; and the stream argument of
the Python device calls.  The rules are checked before the handle is read, so a handle that is never dereferenced
serves."""
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


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _call(lib, call, q=True, nq=2, fmt=api.QUERY_RAW_F32, max_search=50, k=10, ids=True):
    """Status and message of `call` (search | exact | rerank) on the fake handle; q / ids False: a null pointer."""
    queries = np.zeros((2, 8), np.float32)
    out_ids = np.zeros((2, 2000), np.uint32)
    out_d = np.zeros((2, 2000), np.float32)
    pq, pi, pd = api._ptr(queries) if q else None, api._ptr(out_ids) if ids else None, api._ptr(out_d)
    if call == "search":
        rc = lib.granne_b200_search_batch(FAKE, pq, nq, fmt, max_search, k, pi, pd, None, None)
    elif call == "exact":
        rc = lib.granne_b200_exact_search_batch(FAKE, pq, nq, fmt, k, pi, pd, None)
    else:
        rc = lib.granne_b200_search_rerank_batch(FAKE, pq, nq, fmt, max_search, 20, k, pi, pd, None, None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("call", ["search", "exact", "rerank"])
def test_shared_rules(lib, call):
    assert _call(lib, call, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, call, nq=TOO_MANY) == (INVALID, NQ)
    assert _call(lib, call, q=False) == (INVALID, NULL)
    assert _call(lib, call, ids=False) == (INVALID, NULL)


@pytest.mark.parametrize("call", ["search", "rerank"])
def test_max_search_rule(lib, call):
    assert _call(lib, call, max_search=0) == (INVALID, MAX_SEARCH)
    # reported after the format, before the batch size and the buffers
    assert _call(lib, call, max_search=0, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, call, max_search=0, nq=TOO_MANY, q=False) == (INVALID, MAX_SEARCH)


def test_exact_k_rule(lib):
    assert _call(lib, "exact", k=1025) == (INVALID, EXACT_K)
    assert _call(lib, "exact", k=1025, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, "exact", k=1025, nq=TOO_MANY, q=False) == (INVALID, EXACT_K)


def test_no_queries_is_ok_before_the_handle_is_read(lib):
    assert _call(lib, "search", nq=0, q=False, ids=False)[0] == 0
    assert _call(lib, "exact", nq=0, q=False, ids=False)[0] == 0


def test_raw_stream():
    class Stream:
        cuda_stream = 0x7F00DEAD0000

    assert api._raw_stream(0x1234, None) == 0x1234
    assert api._raw_stream(0, None) == 0  # the legacy default stream, not "no stream given"
    assert api._raw_stream(Stream(), None) == 0x7F00DEAD0000
