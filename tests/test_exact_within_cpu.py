"""Exact search within candidate lists without a device: the argument rules of the three C calls (status, message and
the order they are reported in) on a handle that is never dereferenced, and the Python packing of candidate lists
into CSR.  The rules on the ids' range need a real handle's Index::len and are checked in test_exact_within_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from granne_b200 import api

INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
TOO_MANY = 0xFFFFFFF1

FORMAT = "unknown query format"
EXACT_K = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)"
NQ = "too many queries in one batch"
NULL = "null buffer"
OFFSETS_NULL = "offsets is null"
IDS_NULL = "ids is null"
SHAPE = "offsets must start at 0 and not decrease"


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _call(lib, device=False, q=True, nq=2, fmt=api.QUERY_RAW_F32, k=10, out=True, offsets=(0, 2, 3), ids=True):
    """Status and message of the host (or device) call on the fake handle; q / out / ids False, offsets None: a null
    pointer."""
    queries = np.zeros((2, 8), np.float32)
    out_ids = np.zeros((2, 2000), np.uint32)
    out_d = np.zeros((2, 2000), np.float32)
    offs = None if offsets is None else np.asarray(offsets, np.uint64)
    cand = np.array([0, 1, 2], np.uint32)
    pq = api._ptr(queries) if q else None
    po = api._ptr(offs) if offs is not None else None
    pc = api._ptr(cand) if ids else None
    pi = api._ptr(out_ids) if out else None
    if device:
        rc = lib.granne_b200_exact_search_within_batch_device(FAKE, pq, nq, fmt, po, pc, k, pi, api._ptr(out_d), None,
                                                               None)
    else:
        rc = lib.granne_b200_exact_search_within_batch(FAKE, pq, nq, fmt, po, pc, k, pi, api._ptr(out_d), None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("device", [False, True])
def test_shared_rules(lib, device):
    assert _call(lib, device, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, device, k=1025) == (INVALID, EXACT_K)
    assert _call(lib, device, nq=TOO_MANY) == (INVALID, NQ)
    assert _call(lib, device, q=False) == (INVALID, NULL)
    assert _call(lib, device, out=False) == (INVALID, NULL)
    # reported in that order, before the lists' rules
    assert _call(lib, device, fmt=7, k=1025, offsets=None) == (INVALID, FORMAT)
    assert _call(lib, device, k=1025, nq=TOO_MANY, q=False, offsets=None) == (INVALID, EXACT_K)
    assert _call(lib, device, q=False, offsets=None) == (INVALID, NULL)


@pytest.mark.parametrize("device", [False, True])
def test_offsets_null(lib, device):
    assert _call(lib, device, offsets=None) == (INVALID, OFFSETS_NULL)
    assert _call(lib, device, offsets=None, ids=False) == (INVALID, OFFSETS_NULL)


def test_ids_null_when_the_lists_name_ids(lib):
    assert _call(lib, ids=False) == (INVALID, IDS_NULL)
    # before the shape of the offsets
    assert _call(lib, ids=False, offsets=(1, 0, 3)) == (INVALID, IDS_NULL)


@pytest.mark.parametrize("offsets", [(1, 2, 3), (0, 3, 2), (0, 2, 1), (5, 5, 5)])
def test_offsets_shape(lib, offsets):
    assert _call(lib, offsets=offsets) == (INVALID, SHAPE)
    assert _call(lib, offsets=offsets, ids=False) == (INVALID, IDS_NULL)


def test_no_queries_is_ok_before_the_handle_is_read(lib):
    assert _call(lib, nq=0, q=False, out=False, offsets=None, ids=False)[0] == 0
    assert _call(lib, device=True, nq=0, q=False, out=False, offsets=None, ids=False)[0] == 0


def test_multi_null_handle(lib):
    q = np.zeros((1, 8), np.float32)
    rc = lib.granne_b200_multi_exact_search_within_batch(None, api._ptr(q), 1, 0, None, None, 10, None, None, None)
    assert (rc, lib.granne_b200_last_error().decode()) == (INVALID, "multi handle is null")


def test_lists_pack_into_csr():
    lists = [np.array([5, 1, 5], np.int64), np.array([], np.int64), [7], np.arange(3, dtype=np.uint32)]
    offsets, ids = api._candidate_lists(lists, 4, np.uint32)
    assert offsets.dtype == np.uint64 and ids.dtype == np.uint32
    assert offsets.tolist() == [0, 3, 3, 4, 7]
    assert ids.tolist() == [5, 1, 5, 7, 0, 1, 2]
    assert offsets.flags.c_contiguous and ids.flags.c_contiguous


def test_csr_lists_pass_through():
    offsets, ids = api._candidate_lists(api.CsrLists(np.array([0, 2, 2]), np.array([9, 4])), 2, np.uint64)
    assert offsets.dtype == np.uint64 and ids.dtype == np.uint64
    assert offsets.tolist() == [0, 2, 2] and ids.tolist() == [9, 4]
    # a buffer longer than offsets[-1] is fine: the lists end at offsets[-1]
    offsets, ids = api._candidate_lists(api.CsrLists([0, 1], [3, 8, 8]), 1, np.uint32)
    assert offsets.tolist() == [0, 1] and ids.tolist() == [3, 8, 8]


def test_plain_tuple_is_per_query_lists():
    # two queries' lists given as a tuple of two arrays: never read as (offsets, ids)
    offsets, ids = api._candidate_lists((np.array([0, 3, 7]), np.arange(9)), 2, np.uint32)
    assert offsets.tolist() == [0, 3, 12]
    assert ids.tolist() == [0, 3, 7] + list(range(9))


def test_no_lists():
    offsets, ids = api._candidate_lists([], 0, np.uint32)
    assert offsets.tolist() == [0] and ids.size == 0


@pytest.mark.parametrize("cands, nq, msg", [
    ([1, 2], 1, "one candidate list per query"),
    ([np.zeros((2, 2), np.int64)], 1, "1-D"),
    (api.CsrLists(np.array([0, 1]), np.array([3])), 2, "offsets must have shape"),
    (api.CsrLists(np.array([0, 5]), np.array([1, 2])), 1, r"offsets\[-1\] = 5 exceeds the 2 ids given"),
    (api.CsrLists(np.array([0, 1, 3]), np.array([1, 2])), 2, r"offsets\[-1\] = 3 exceeds the 2 ids given"),
    (api.CsrLists(np.array([0, 1]), np.zeros((1, 1), np.int64)), 1, "ids must be 1-D"),
    ([np.array([-1])], 1, "non-negative"),
    ([np.array([1.5])], 1, "integers"),
    ([np.array([1 << 32])], 1, "fit uint32"),
])
def test_list_rejections(cands, nq, msg):
    with pytest.raises(ValueError, match=msg):
        api._candidate_lists(cands, nq, np.uint32)
