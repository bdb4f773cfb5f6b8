"""Exact filtered search without a device: the argument rules of the host, device and multi calls (status, message and
the order they are reported in) on a handle that is never dereferenced, nq == 0, the new symbols in the C header, the
C++ header and the Rust shim, and the Python checks that run before any library call.  The rules that read the
handle's Index::len (filter_words) and the host check of query_filter are checked in test_exact_filtered_gpu.py."""
import ctypes as C
import os

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.fixtures import compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOO_MANY = 0xFFFFFFF1

HANDLE = "index handle is null"
FORMAT = "unknown query format"
EXACT_K = "num_neighbors exceeds GRANNE_B200_EXACT_MAX_K (1024)"
NQ = "too many queries in one batch"
NULL = "null buffer"
FILTERS = "filters is null or num_filters is 0"
EXCLUDE_K = "num_neighbors exceeds 1023 with GRANNE_B200_QUERY_ID_EXCLUDING (the call runs k + 1)"
NAMES = ["granne_b200_exact_search_filtered_batch", "granne_b200_exact_search_filtered_batch_device",
         "granne_b200_multi_exact_search_filtered_batch"]


def _call(lib, which="host", handle=FAKE, q=True, nq=2, fmt=api.QUERY_RAW_F32, k=10, out=True, filters=True,
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
        rc = lib.granne_b200_exact_search_filtered_batch(handle, pq, nq, fmt, pf, num_filters, 4, None, k, pi,
                                                         api._ptr(out_d), None)
    elif which == "device":
        rc = lib.granne_b200_exact_search_filtered_batch_device(handle, pq, nq, fmt, pf, num_filters, 4, None, k, pi,
                                                                api._ptr(out_d), None, None)
    else:
        rc = lib.granne_b200_multi_exact_search_filtered_batch(handle, pq, nq, fmt, pf, num_filters, 4, None, k, pi,
                                                               api._ptr(out_d), None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("which", ["host", "device"])
def test_each_rule(library, which):
    assert _call(library, which, handle=None) == (INVALID, HANDLE)
    assert _call(library, which, fmt=7) == (INVALID, FORMAT)
    assert _call(library, which, k=1025) == (INVALID, EXACT_K)
    assert _call(library, which, nq=TOO_MANY) == (INVALID, NQ)
    assert _call(library, which, q=False) == (INVALID, NULL)
    assert _call(library, which, out=False) == (INVALID, NULL)
    assert _call(library, which, filters=False) == (INVALID, FILTERS)
    assert _call(library, which, num_filters=0) == (INVALID, FILTERS)
    assert _call(library, which, fmt=api.QUERY_ID_EXCLUDING, k=1024, filters=False) == (INVALID, FILTERS)
    assert _call(library, which, fmt=api.QUERY_ID_EXCLUDING, k=1024) == (INVALID, EXCLUDE_K)


@pytest.mark.parametrize("which", ["host", "device"])
def test_rule_order(library, which):
    everything = dict(handle=None, fmt=7, k=1025, nq=TOO_MANY, q=False, out=False, filters=False)
    order = [("handle", HANDLE), ("fmt", FORMAT), ("k", EXACT_K), ("nq", NQ), ("q", NULL), ("out", NULL),
             ("filters", FILTERS)]
    for i, (_, msg) in enumerate(order):
        broken = {name: everything[name] for name, _ in order[i:]}
        assert _call(library, which, **broken) == (INVALID, msg), broken


@pytest.mark.parametrize("which", ["host", "device"])
def test_every_query_format_passes_the_format_rule(library, which):
    for fmt in (api.QUERY_RAW_F32, api.QUERY_ELEMENT, api.QUERY_ID, api.QUERY_ID_EXCLUDING):
        assert _call(library, which, fmt=fmt, filters=False) == (INVALID, FILTERS)


@pytest.mark.parametrize("which", ["host", "device"])
def test_no_queries_is_ok_before_the_filters_and_the_handle_are_read(library, which):
    assert _call(library, which, nq=0, q=False, out=False, filters=False, num_filters=0)[0] == 0
    assert _call(library, which, nq=0, k=0, q=False, out=False, filters=False)[0] == 0


def test_k_zero_needs_no_output_buffers(library):
    # k == 0 writes no entry: null ids / dists break no rule, the call goes on to the filters' rule
    assert _call(library, "host", k=0, out=False, filters=False) == (INVALID, FILTERS)


def test_multi_null_handle_first(library):
    # before every single-device rule (those follow on a real handle: test_exact_filtered_gpu.py)
    assert _call(library, "multi", handle=None, fmt=7, k=1025, filters=False) == (INVALID, "multi handle is null")
    assert _call(library, "multi", handle=None, nq=0) == (INVALID, "multi handle is null")


def test_symbols_in_the_headers_and_the_shim(library):
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    raw = C.CDLL(granne_b200.library_path())
    for name in NAMES:
        assert "int %s(" % name in header
        assert hasattr(raw, name)
    assert "#define GRANNE_B200_ABI_VERSION 2 " in header
    assert library.granne_b200_abi_version() == 2
    cxx = open(os.path.join(ROOT, "include", "granne_b200.hpp")).read()
    assert cxx.count("exact_search_filtered(") == 2
    shim = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    for name in ("granne_b200_exact_search_filtered_batch", "granne_b200_multi_exact_search_filtered_batch"):
        assert "fn %s(" % name in shim
    assert shim.count("pub fn exact_search_filtered(") == 2


def test_cxx_exact_filtered_client_compiles(library, tmp_path):
    compile_cxx_client("cxx_exact_filtered_client.cpp", tmp_path)


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

    def __len__(self):
        return 40

    def __del__(self):
        pass


@pytest.mark.parametrize("filters, query_filter, msg", [
    (np.ones(41, bool), None, "a bool filter mask must have shape"),
    (np.ones((1, 1), np.uint32), None, "filter words: W = 1 is less than ceil(40 / 32) = 2"),
    (np.ones(40, np.float32), None, "filters must be a bool mask or uint32 words"),
    (np.ones((0, 2), np.uint32), None, "filters must hold at least one filter"),
    (np.ones(40, bool), np.zeros(3, np.uint32), "query_filter must have shape (nq,) = (2,)"),
    (np.ones(40, bool), np.array([0, -1]), "query_filter entries must be non-negative"),
])
def test_python_rejections(filters, query_filter, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        _Fake().exact_search_filtered(np.zeros((2, 8), np.float32), filters, query_filter)


def test_python_device_form_needs_cuda_tensors():
    torch = pytest.importorskip("torch")
    q = torch.zeros((2, 8), dtype=torch.float32)
    with pytest.raises(ValueError, match="CUDA torch tensor"):
        _Fake().exact_search_filtered_device(q, torch.zeros((1, 2), dtype=torch.int32))
