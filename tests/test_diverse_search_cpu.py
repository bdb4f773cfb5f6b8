"""The diverse search without a device: the selection-by-elimination scheme of diverse_kernel, modelled lane by lane
(helpers/diverse_model.py), against the oracle's select_neighbors on a few hundred random lists of every element
kind; the argument rules of the four calls in the order they are reported, on a handle that is never dereferenced;
and the exported symbols and the candidate cap the header and the Python binding share."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from granne_b200 import api
from helpers import diverse_model as dm
from helpers.data import random_vectors, varied_sum_embeddings
from helpers.fixtures import library  # noqa: F401  (autouse)
from oracle import granne_oracle as go

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1
FAKE = C.c_void_p(1)  # never dereferenced by a call whose arguments break a rule
TOO_MANY = 0xFFFFFFF1

FORMAT = "unknown query format"
MAX_SEARCH = "max_search must be >= 1 (the reference panics on 0, src/index/mod.rs:1019)"
DIVERSE_MAX = "max_search exceeds GRANNE_B200_DIVERSE_MAX_CANDIDATES (1024)"
STRIDE = "the candidate stride exceeds GRANNE_B200_DIVERSE_MAX_CANDIDATES (1024)"
NQ = "too many queries in one batch"
NULL = "null buffer"
SYMBOLS = ("granne_b200_search_diverse_batch", "granne_b200_search_diverse_batch_device",
           "granne_b200_select_neighbors_batch", "granne_b200_select_neighbors_batch_device",
           "granne_b200_multi_search_diverse_batch")


def _containers():
    """Oracle containers of each kind with planted duplicates (ties) and a zero row."""
    f = random_vectors(160, 40, 1)
    f[10:14] = f[9]        # exact duplicates
    f[20] = 0.0            # a zero row
    i8 = random_vectors(160, 48, 2)
    i8[30:33] = i8[29]
    return {"angular": go.Elements.angular(f), "angular_int": go.Elements.angular_int(i8),
            "embeddings": varied_sum_embeddings(go, 36, 60, 160, 3)}


@pytest.fixture(scope="module")
def containers():
    out = {}
    for kind, el in _containers().items():
        n = len(el)
        pair = np.stack([el.dists(s, np.arange(n)) for s in range(n)])  # pair[s, c] = dist(c, element s)
        out[kind] = (el, pair)
    return out


@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_elimination_model_matches_the_oracle(containers, kind):
    el, pair = containers[kind]
    n = len(el)
    rng = np.random.default_rng(7)
    pruned = 0
    for case in range(120):
        s0 = int(rng.integers(0, n))
        d = pair[s0].copy()  # the candidates' distances to element s0, as the query
        order = np.lexsort((np.arange(n), d))
        order = order[order != s0]
        c = int(rng.choice([0, 1, 5, 31, 32, 33, 64, 100, n - 1]))
        cand = order[:c]
        k = int(rng.choice([1, 2, 5, 10, 40, c, c + 1, max(c - 1, 0)]))
        want = go.select_neighbors(el, [(int(i), float(d[i])) for i in cand], k)
        got_i, got_d, pairs = dm.select_by_elimination([int(i) for i in cand], [float(d[i]) for i in cand], k,
                                                      lambda s, cc: pair[s, cc])
        seq_i, _ = dm.select_sequential([int(i) for i in cand], [float(d[i]) for i in cand], k,
                                        lambda s, cc: pair[s, cc])
        assert got_i == [w[0] for w in want] == seq_i, (kind, case, c, k)
        assert np.array_equal(np.float32(got_d), np.float32([w[1] for w in want]))
        assert pairs <= k * c
        pruned += len(got_i) < min(k, c)
    assert pruned > 0  # the cases exercise pruning, not only the unpruned return


def test_elimination_model_edges():
    # C <= k: unpruned, even when the list would be pruned; ties kept (d <= d); all-equal rows collapse to one
    far = lambda s, c: 1.0  # noqa: E731
    same = lambda s, c: 0.0  # noqa: E731
    assert dm.select_by_elimination([3, 1, 2], [0.1, 0.2, 0.3], 3, same)[0] == [3, 1, 2]
    assert dm.select_by_elimination([3, 1, 2, 5], [0.1, 0.2, 0.3, 0.4], 3, same)[0] == [3]
    assert dm.select_by_elimination([3, 1, 2, 5], [0.5, 0.5, 0.5, 0.5], 2, lambda s, c: 0.5)[0] == [3, 1]
    assert dm.select_by_elimination(list(range(100)), [0.5] * 100, 40, far)[0] == list(range(40))
    assert dm.select_by_elimination([], [], 0, far)[0] == []
    assert dm.select_by_elimination([4, 5], [0.1, 0.2], 0, far)[0] == []


def _diverse(lib, fmt=api.QUERY_RAW_F32, nq=2, max_search=50, k=10, q=True, ids=True, device=False):
    queries = np.zeros((2, 8), np.float32)
    out_i, out_d = np.zeros((2, 64), np.uint32), np.zeros((2, 64), np.float32)
    args = [FAKE, api._ptr(queries) if q else None, nq, fmt, max_search, k, api._ptr(out_i) if ids else None,
            api._ptr(out_d), None, None]
    fn = lib.granne_b200_search_diverse_batch_device if device else lib.granne_b200_search_diverse_batch
    rc = fn(*(args + [None] if device else args))
    return rc, lib.granne_b200_last_error().decode()


def _select(lib, nq=2, stride=8, k=4, cand=True, counts=True, ids=True, handle=FAKE, device=False):
    ci, cd = np.zeros((2, 8), np.uint32), np.zeros((2, 8), np.float32)
    cc = np.zeros(2, np.uint32)
    out_i, out_d = np.zeros((2, 8), np.uint32), np.zeros((2, 8), np.float32)
    args = [handle, api._ptr(ci) if cand else None, api._ptr(cd), api._ptr(cc) if counts else None, nq, stride, k,
            api._ptr(out_i) if ids else None, api._ptr(out_d), None]
    fn = lib.granne_b200_select_neighbors_batch_device if device else lib.granne_b200_select_neighbors_batch
    rc = fn(*(args + [None] if device else args))
    return rc, lib.granne_b200_last_error().decode()


@pytest.mark.parametrize("device", [False, True])
def test_diverse_rules_in_order(library, device):
    call = lambda **kw: _diverse(library, device=device, **kw)  # noqa: E731
    assert call(fmt=7, max_search=0) == (INVALID, FORMAT)
    assert call(max_search=0, nq=TOO_MANY, q=False) == (INVALID, MAX_SEARCH)
    assert call(max_search=1025, nq=TOO_MANY, q=False) == (INVALID, DIVERSE_MAX)
    assert call(nq=TOO_MANY, q=False) == (INVALID, NQ)
    assert call(q=False) == (INVALID, NULL)
    assert call(ids=False) == (INVALID, NULL)
    assert call(ids=False, k=0, nq=0)[0] == 0
    for fmt in (api.QUERY_ELEMENT, api.QUERY_ID, api.QUERY_ID_EXCLUDING):
        assert call(fmt=fmt, ids=False) == (INVALID, NULL)  # every query format gets past the format rule
    assert library.granne_b200_search_diverse_batch(None, None, 0, 0, 50, 10, None, None, None, None) == INVALID
    assert b"index handle is null" in library.granne_b200_last_error()
    assert library.granne_b200_multi_search_diverse_batch(None, None, 0, 0, 50, 10, None, None, None) == INVALID
    assert b"multi handle is null" in library.granne_b200_last_error()


@pytest.mark.parametrize("device", [False, True])
def test_select_rules_in_order(library, device):
    call = lambda **kw: _select(library, device=device, **kw)  # noqa: E731
    assert call(handle=None, stride=2000) == (INVALID, "index handle is null")
    assert call(stride=1025, nq=TOO_MANY, counts=False) == (INVALID, STRIDE)
    assert call(nq=TOO_MANY, counts=False) == (INVALID, NQ)
    assert call(counts=False, cand=False) == (INVALID, NULL)
    assert call(ids=False) == (INVALID, NULL)
    assert call(cand=False) == (INVALID, NULL)
    assert call(nq=0, cand=False, counts=False, ids=False)[0] == 0


def test_symbols_and_cap(library):
    for name in SYMBOLS:
        assert hasattr(library, name), name
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    m = re.search(r"#define GRANNE_B200_DIVERSE_MAX_CANDIDATES (\d+)", header)
    assert m and int(m.group(1)) == api.DIVERSE_MAX_CANDIDATES
    for name in SYMBOLS:
        assert name + "(" in header
    rust = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    for name in SYMBOLS:
        assert "fn " + name + "(" in rust, name
