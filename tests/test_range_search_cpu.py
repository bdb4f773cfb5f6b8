"""Exact range search without a device: the argument rules of the count and search calls (host and device forms) and
the order they are reported in, the multi-handle calls' null handle, the new symbols in the C header, the C++ header
and the Rust shim, and the Python packing and rejections.  The rules are checked before the handle is read, so a
handle that is never dereferenced serves."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import granne_b200
from granne_b200 import api

INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOO_MANY = 0xFFFFFFF1
HANDLE = "index handle is null"
FORMAT = "unknown query format"
RADIUS = "radius is NaN"
NQ = "too many queries in one batch"
NULL = "null buffer"
COUNTS_NULL = "counts is null"
OFFSETS_NULL = "offsets is null"
OFFSETS_SHAPE = "offsets must start at 0 and not decrease"
CALLS = ["count", "count_device", "search", "search_device"]


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _call(lib, call, h=FAKE, q=True, nq=2, fmt=api.QUERY_RAW_F32, radius=0.5, counts=True, offsets=(0, 2, 3),
          outs=True):
    """Status and message of `call` (one of CALLS); q / counts / outs False, offsets None: a null pointer."""
    queries = np.zeros((2, 8), np.float32)
    cnt = np.zeros(2, np.uint64)
    offs = None if offsets is None else np.asarray(offsets, np.uint64)
    ids = np.zeros(8, np.uint32)
    d = np.zeros(8, np.float32)
    pq = api._ptr(queries) if q else None
    po = api._ptr(offs) if offs is not None else None
    pi, pd = (api._ptr(ids), api._ptr(d)) if outs else (None, None)
    if call == "count":
        rc = lib.granne_b200_exact_range_count(h, pq, nq, fmt, radius, api._ptr(cnt) if counts else None)
    elif call == "count_device":
        rc = lib.granne_b200_exact_range_count_device(h, pq, nq, fmt, radius, api._ptr(cnt) if counts else None, None)
    elif call == "search":
        rc = lib.granne_b200_exact_range_search(h, pq, nq, fmt, radius, po, pi, pd)
    else:
        rc = lib.granne_b200_exact_range_search_device(h, pq, nq, fmt, radius, po, pi, pd, None)
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("call", CALLS)
def test_rules_in_order(lib, call):
    nan = float("nan")
    # validate_batch's order: handle, format, the NaN radius (the call's own rule), batch size, queries
    assert _call(lib, call, h=None, fmt=7, radius=nan) == (INVALID, HANDLE)
    assert _call(lib, call, fmt=7, radius=nan, nq=TOO_MANY) == (INVALID, FORMAT)
    assert _call(lib, call, radius=nan, nq=TOO_MANY, q=False) == (INVALID, RADIUS)
    assert _call(lib, call, nq=TOO_MANY, q=False) == (INVALID, NQ)
    assert _call(lib, call, q=False, counts=False, offsets=None) == (INVALID, NULL)
    # then the call's own output: counts, or offsets
    if call.startswith("count"):
        assert _call(lib, call, counts=False) == (INVALID, COUNTS_NULL)
    else:
        assert _call(lib, call, offsets=None, outs=False) == (INVALID, OFFSETS_NULL)


@pytest.mark.parametrize("call", CALLS)
def test_nan_radius_is_rejected_even_without_queries(lib, call):
    assert _call(lib, call, radius=float("nan"), nq=0, q=False) == (INVALID, RADIUS)


@pytest.mark.parametrize("call", CALLS)
def test_no_queries_is_ok_before_the_handle_is_read(lib, call):
    for fmt in (api.QUERY_RAW_F32, api.QUERY_ELEMENT, api.QUERY_ID, api.QUERY_ID_EXCLUDING):
        assert _call(lib, call, fmt=fmt, nq=0, q=False, counts=False, offsets=None, outs=False)[0] == 0
    for radius in (float("inf"), float("-inf"), -0.0, 0.0, -1.0):
        assert _call(lib, call, radius=radius, nq=0, q=False, counts=False, offsets=None, outs=False)[0] == 0


def test_host_search_checks_offsets_then_outputs(lib):
    assert _call(lib, "search", offsets=(1, 2, 3)) == (INVALID, OFFSETS_SHAPE)
    assert _call(lib, "search", offsets=(0, 2, 1)) == (INVALID, OFFSETS_SHAPE)
    assert _call(lib, "search", offsets=(0, 2, 1), outs=False) == (INVALID, OFFSETS_SHAPE)
    assert _call(lib, "search", outs=False) == (INVALID, NULL)  # offsets[nq] > 0


def test_multi_null_handle(lib):
    cnt = np.zeros(1, np.uint64)
    offs = np.zeros(2, np.uint64)
    assert lib.granne_b200_multi_exact_range_count(None, None, 0, 0, 0.5, api._ptr(cnt)) == INVALID
    assert lib.granne_b200_multi_exact_range_search(None, None, 0, 0, 0.5, api._ptr(offs), None, None) == INVALID
    assert lib.granne_b200_last_error().decode() == "multi handle is null"


NAMES = ["granne_b200_exact_range_count", "granne_b200_exact_range_count_device", "granne_b200_exact_range_search",
         "granne_b200_exact_range_search_device", "granne_b200_multi_exact_range_count",
         "granne_b200_multi_exact_range_search"]


def test_symbols_in_the_headers_and_the_shim(lib):
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    raw = C.CDLL(granne_b200.library_path())
    for name in NAMES:
        assert "int %s(" % name in header
        assert hasattr(raw, name)
    assert "#define GRANNE_B200_ABI_VERSION 2 " in header
    assert lib.granne_b200_abi_version() == 2
    cxx = open(os.path.join(ROOT, "include", "granne_b200.hpp")).read()
    assert cxx.count("exact_range_search(const void* queries, size_t nq, int query_format, float radius) const") == 2
    shim = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    for name in ("granne_b200_exact_range_count", "granne_b200_exact_range_search",
                 "granne_b200_multi_exact_range_count", "granne_b200_multi_exact_range_search"):
        assert "fn %s(" % name in shim
    assert shim.count("pub fn exact_range_search(") == 2


def test_cxx_range_client_compiles(lib, tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    libdir = os.path.dirname(granne_b200.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", "cxx_range_client.cpp"), "-o",
                           str(tmp_path / "client"), "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])


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


def test_python_radius_packing():
    assert api._radius(1) == 1.0
    assert api._radius(np.float64(0.1)) == float(np.float32(0.1))
    assert api._radius(float("inf")) == float("inf")
    assert np.isnan(api._radius(float("nan")))  # the library rejects it, with its own message
    assert np.signbit(api._radius(-0.0))
    for bad in ("0.5", None, [0.5], True, np.array([0.5])):
        with pytest.raises(ValueError):
            api._radius(bad)


def test_python_offsets_from_counts():
    off = api._csr_offsets(np.array([3, 0, 2], np.uint64))
    assert off.dtype == np.uint64 and off.tolist() == [0, 3, 3, 5]
    assert api._csr_offsets(np.zeros(0, np.uint64)).tolist() == [0]


@pytest.mark.parametrize("bad", [np.zeros((2, 2), np.uint32), np.array([1.5, 2.0]), np.array([-1, 2]),
                                 np.array([2**32], np.uint64)])
def test_python_rejections(bad):
    g = _Fake()
    for fn in (lambda: g.exact_range_count(bad, 0.5, by_id=True),
               lambda: g.exact_range_search(bad, 0.5, exclude_self=True)):
        with pytest.raises(ValueError):
            fn()
    with pytest.raises(ValueError):
        g.exact_range_count(np.zeros((2, 7), np.float32), 0.5)  # wrong width
    with pytest.raises(ValueError):
        g.exact_range_count(np.zeros((2, 8), np.float32), "near")


def test_python_device_forms_need_cuda_tensors():
    g = _Fake()
    with pytest.raises(ValueError):
        g.exact_range_count_device(np.zeros((2, 8), np.float32), 0.5)
    with pytest.raises(ValueError):
        g.exact_range_search_device(np.array([1, 2], np.int32), 0.5, np.zeros(3, np.int64), by_id=True)


def test_python_range_graph_arguments():
    with pytest.raises(ValueError):
        _Fake().range_graph(0.1, chunk=0)
    with pytest.raises(ValueError):
        _Fake().range_graph(0.1, out="disk")
