"""Filtered search without a device: the argument rules of the three C calls (status, message and the order they are
reported in) on a handle that is never dereferenced, and the Python packing of filters.  The rules that read the
handle's Index::len (filter_words) and the host check of query_filter are checked in test_filtered_search_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.filtered_oracle import pack

INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
TOO_MANY = 0xFFFFFFF1

HANDLE = "index handle is null"
FORMAT = "unknown query format"
MAX_SEARCH = "max_search must be >= 1 (the reference panics on 0, src/index/mod.rs:1019)"
EXACT_K = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)"
NQ = "too many queries in one batch"
NULL = "null buffer"
FILTERS = "filters is null or num_filters is 0"


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _call(lib, which="host", handle=FAKE, q=True, nq=2, fmt=api.QUERY_RAW_F32, ef=50, k=10, out=True, filters=True,
          num_filters=1):
    """Status and message of the host, device or multi call; q / out / filters False: a null pointer."""
    queries = np.zeros((2, 8), np.float32)
    out_ids = np.zeros((2, 2000), np.uint64)
    out_d = np.zeros((2, 2000), np.float32)
    words = np.ones((2, 4), np.uint32)
    pq = api._ptr(queries) if q else None
    pi = api._ptr(out_ids) if out else None
    pf = api._ptr(words) if filters else None
    if which == "host":
        rc = lib.granne_b200_search_filtered_batch(handle, pq, nq, fmt, ef, k, pf, num_filters, 4, None, pi,
                                                   api._ptr(out_d), None, None)
    elif which == "device":
        rc = lib.granne_b200_search_filtered_batch_device(handle, pq, nq, fmt, ef, k, pf, num_filters, 4, None, pi,
                                                          api._ptr(out_d), None, None, None)
    else:
        rc = lib.granne_b200_multi_search_filtered_batch(handle, pq, nq, fmt, ef, k, pf, num_filters, 4, None, pi,
                                                         api._ptr(out_d), None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("which", ["host", "device"])
def test_each_rule(lib, which):
    assert _call(lib, which, handle=None) == (INVALID, HANDLE)
    assert _call(lib, which, fmt=7) == (INVALID, FORMAT)
    assert _call(lib, which, ef=0) == (INVALID, MAX_SEARCH)
    assert _call(lib, which, k=1025) == (INVALID, EXACT_K)
    assert _call(lib, which, nq=TOO_MANY) == (INVALID, NQ)
    assert _call(lib, which, q=False) == (INVALID, NULL)
    assert _call(lib, which, out=False) == (INVALID, NULL)
    assert _call(lib, which, filters=False) == (INVALID, FILTERS)
    assert _call(lib, which, num_filters=0) == (INVALID, FILTERS)


@pytest.mark.parametrize("which", ["host", "device"])
def test_rule_order(lib, which):
    everything = dict(handle=None, fmt=7, ef=0, k=1025, nq=TOO_MANY, q=False, out=False, filters=False)
    order = [("handle", HANDLE), ("fmt", FORMAT), ("ef", MAX_SEARCH), ("k", EXACT_K), ("nq", NQ), ("q", NULL),
             ("out", NULL), ("filters", FILTERS)]
    for i, (_, msg) in enumerate(order):
        broken = {name: everything[name] for name, _ in order[i:]}
        assert _call(lib, which, **broken) == (INVALID, msg), broken


@pytest.mark.parametrize("which", ["host", "device"])
def test_k_may_exceed_max_search(lib, which):
    # k > max_search breaks no rule: the call goes on to the filters' rule
    assert _call(lib, which, ef=5, k=1024, filters=False) == (INVALID, FILTERS)


@pytest.mark.parametrize("which", ["host", "device"])
def test_no_queries_is_ok_before_the_filters_and_the_handle_are_read(lib, which):
    assert _call(lib, which, nq=0, q=False, out=False, filters=False, num_filters=0)[0] == 0


def test_multi_null_handle_first(lib):
    # before every single-device rule (those follow on a real handle: test_filtered_search_gpu.py)
    assert _call(lib, "multi", handle=None, fmt=7, ef=0, filters=False) == (INVALID, "multi handle is null")


def test_bool_mask_packs_lsb_first():
    n = 70
    mask = np.zeros(n, bool)
    mask[[0, 1, 31, 32, 63, 64, 69]] = True
    words = api._filter_words(mask, n)
    assert words.dtype == np.uint32 and words.shape == (1, 3) and words.flags.c_contiguous
    assert words.tolist() == [[0x80000003, 0x80000001, (1 << 0) | (1 << 5)]]
    assert np.array_equal(words, pack(mask))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 4097])
def test_bool_masks_match_the_independent_packing(n):
    rng = np.random.default_rng(n)
    masks = rng.random((3, n)) < 0.3
    words = api._filter_words(masks, n)
    assert words.shape == (3, (n + 31) // 32)
    assert np.array_equal(words, pack(masks))
    # unpacking gives the mask back, and no bit beyond n is set
    bits = np.unpackbits(words.view(np.uint8), axis=1, bitorder="little").astype(bool)
    assert np.array_equal(bits[:, :n], masks) and not bits[:, n:].any()


def test_words_pass_through():
    w = np.arange(12, dtype=np.uint32).reshape(3, 4)
    assert api._filter_words(w, 100) is not None
    assert np.array_equal(api._filter_words(w, 100), w)
    # wider than needed is fine (a bitmap shared with a larger index)
    assert api._filter_words(w, 33).shape == (3, 4)
    # a strided view is made contiguous
    assert api._filter_words(np.ones((4, 8), np.uint32)[:, ::2], 100).flags.c_contiguous


@pytest.mark.parametrize("filters, n, msg", [
    (np.zeros(10, bool), 11, r"shape \(11,\) or \(F, 11\)"),
    (np.zeros((2, 10), bool), 9, r"shape \(9,\) or \(F, 9\)"),
    (np.zeros((1, 2, 3), bool), 3, "shape"),
    (np.zeros((0, 5), bool), 5, "at least one filter"),
    (np.zeros((2, 3), np.uint32), 100, r"W = 3 is less than ceil\(100 / 32\) = 4"),
    (np.zeros(4, np.uint32), 100, r"shape \(F, W\)"),
    (np.zeros((0, 4), np.uint32), 100, "at least one filter"),
    (np.zeros((1, 4), np.int32), 100, "bool mask or uint32 words"),
    (np.zeros((1, 4), np.uint64), 100, "bool mask or uint32 words"),
    ([[1, 0, 1]], 3, "bool mask or uint32 words"),
])
def test_filter_rejections(filters, n, msg):
    with pytest.raises(ValueError, match=msg):
        api._filter_words(filters, n)


def test_query_filter_packing():
    assert api._query_filter(None, 3) is None
    qf = api._query_filter([0, 2, 1], 3)
    assert qf.dtype == np.uint32 and qf.tolist() == [0, 2, 1]
    # entries >= F are the library's to reject (its rule and message)
    assert api._query_filter(np.array([7], np.int64), 1).tolist() == [7]


@pytest.mark.parametrize("qf, nq, msg", [
    ([0, 1], 3, r"shape \(nq,\) = \(3,\)"),
    (np.zeros((1, 1), np.int64), 1, "shape"),
    ([-1], 1, "non-negative"),
    ([1 << 32], 1, "fit uint32"),
    ([0.5], 1, "integers"),
])
def test_query_filter_rejections(qf, nq, msg):
    with pytest.raises(ValueError, match=msg):
        api._query_filter(qf, nq)
