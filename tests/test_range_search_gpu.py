"""Exact range search on the GPU (granne_b200_exact_range_count* / granne_b200_exact_range_search*): offsets, ids,
distance bits and counts equal a composed oracle — the CPU oracle's exact search over the whole index
(tests/helpers/exact_oracle.cpp) cut at d <= r, with the NumPy model (tests/helpers/ref_model.py) as a second
statement — for every engine, radii at their edges, results spanning slabs and windows, queries by id, mismatched
offsets, NaN elements, concurrent streams, both multi modes, range_graph and a C++ client; and at scale, without an
oracle, the identity with exact_search_batch(k = 1024)."""
import ctypes as C
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers import embeddings_oracle as eo
from helpers import exact_oracle as xo
from helpers import ref_model as rm
from helpers.data import clustered_vectors, random_vectors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NOT_FINITE, OUT_OF_RANGE = -1, -6, -8
U32_MAX = 0xFFFFFFFF


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _rows(kind, raw):
    image = granne_b200.elements_from_raw(kind, raw)
    dim = int(np.frombuffer(bytes(image[:8]), dtype=np.uint64)[0])
    return np.frombuffer(bytes(image[8:]), dtype=np.float32 if kind == "angular" else np.int8).reshape(-1, dim)


def _dense(go, kind, rows, index_len=None):
    """(GPU handle, oracle container) over the given element rows; the index covers index_len of them."""
    rows = np.ascontiguousarray(rows)
    eb = np.uint64(rows.shape[1]).tobytes() + rows.tobytes()
    n = rows.shape[0] if index_len is None else index_len
    return granne_b200.Granne.from_bytes(xo.single_layer_index(go, n), kind, eb), xo.Container(kind, eb)


def _want(c, q, r, n, k=None, already_element=False, self_ids=None):
    """The oracle's range: the exact search over [0, n) (its first k entries: k must exceed every |R(q)|) cut at
    d <= r, without each query's own id when self_ids is given.  Returns (offsets, ids, dists)."""
    k = n if k is None else min(n, k)
    if n == 0 or q.shape[0] == 0:
        return np.zeros(q.shape[0] + 1, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.float32)
    ids, d, cnt = c.exact_search(q, max(k, 1), index_len=n, already_element=already_element, threads=32)
    keep = (np.arange(ids.shape[1])[None, :] < cnt[:, None]) & (d <= np.float32(r))
    if self_ids is not None:
        keep &= ids != np.asarray(self_ids, np.uint32)[:, None]
    if k < n:
        assert not keep[:, -1].any(), "the oracle's k does not cover the range"
    offsets = np.zeros(q.shape[0] + 1, np.uint64)
    np.cumsum(keep.sum(1), out=offsets[1:])
    return offsets, ids[keep], d[keep]


def _same(got, want):
    go, gi, gd = (np.asarray(x) for x in got)
    wo, wi, wd = want
    assert np.array_equal(go.astype(np.uint64), wo)
    assert np.array_equal(gi.astype(np.uint32), wi)
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))


def _check(g, c, q, r, n=None, already_element=False, **kw):
    """The host calls against the oracle; the count equals the segment lengths.  Returns the offsets."""
    n = len(g) if n is None else n
    got = g.exact_range_search(q, r, already_element=already_element, **kw)
    counts = g.exact_range_count(q, r, already_element=already_element, **kw)
    assert np.array_equal(np.diff(got[0]), counts)
    k = int(counts.max()) + 1 if counts.size else 1
    _same(got, _want(c, q, r, n, k=k, already_element=already_element))
    return got[0]


def _kth(c, q, j, already_element=False):
    """The exact distance of query 0's j-th nearest element (an element's distance: the tie at the bound)."""
    return c.exact_search(q[:1], j + 1, already_element=already_element)[1][0, j]


@pytest.mark.parametrize("dim", [1, 31, 32, 33, 64, 100, 128, 256, 300, 1000])
def test_f32_every_engine_layout(oracle, dim):
    rows = _rows("angular", random_vectors(700, dim, dim))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(40, dim, dim + 1)
    r = _kth(c, q, 50)
    assert np.diff(_check(g, c, q, r))[0] >= 51  # the element at the bound is in
    below = np.nextafter(r, np.float32(-np.inf), dtype=np.float32)
    _check(g, c, q, below)
    qe = rows[[3, 500, 699]]  # ELEMENT queries
    _check(g, c, qe, _kth(c, qe, 20, already_element=True), already_element=True)


@pytest.mark.parametrize("dim", [1, 16, 100, 511, 512, 513, 1000])
def test_i8_every_width(oracle, dim):
    rows = _rows("angular_int", random_vectors(600, dim, dim))
    g, c = _dense(oracle, "angular_int", rows)
    q = random_vectors(30, dim, dim + 1)
    _check(g, c, q, _kth(c, q, 40))
    _check(g, c, rows[[0, 599]], _kth(c, rows[[0, 599]], 10))


def _sum_case(dim, n, seed, num_rows=300):
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((num_rows, dim))).astype(np.float32)
    counts = [0, 1, 2, 7, 33, 40]
    elements = [[int(t) for t in rng.integers(0, num_rows, counts[i % len(counts)])] for i in range(n)]
    return eo.table_image(table), eo.elements_image(elements)


@pytest.mark.parametrize("dim,n", [(20, 700), (2048, 20000)])
def test_embeddings_across_windows(oracle, dim, n):
    ti, ei = _sum_case(dim, n, dim)
    m = n - 3  # an index shorter than its container
    g = granne_b200.Granne.from_bytes(xo.single_layer_index(oracle, m), "embeddings", ei, ti)
    c = xo.Container("embeddings", ei, ti)
    q = random_vectors(5, dim, 1)
    r = c.exact_search(q[:1], 300, index_len=m)[1][0, 299]
    off = _check(g, c, q, r, n=m)
    assert int(off[1]) >= 300
    _check(g, c, q, np.float32(np.inf), n=m)  # every element: the results of one query across all windows


def test_radius_edges_with_duplicates_and_zero_rows(oracle):
    base = _rows("angular", random_vectors(40, 64, 1))
    rows = np.concatenate([base, base, np.zeros((30, 64), np.float32), base[:1].repeat(50, 0), base]).astype(np.float32)
    g, c = _dense(oracle, "angular", rows)
    n = len(rows)
    q = np.concatenate([base[:5], np.zeros((1, 64), np.float32)])
    for r in (0.0, -0.0, np.float32(np.inf), -1.0, 1.0, np.nextafter(np.float32(1), np.float32(0))):
        _check(g, c, q, r, already_element=True)
    assert np.array_equal(g.exact_range_count(q, np.inf, already_element=True), np.full(6, n, np.uint64))
    assert not g.exact_range_count(q, -1.0, already_element=True).any()
    # the all-zero query: every distance is exactly 1
    assert g.exact_range_count(q[5:], 1.0, already_element=True)[0] == n
    assert g.exact_range_count(q[5:], np.nextafter(np.float32(1), np.float32(0)), already_element=True)[0] == 0
    # distance 0 of an element to its copies is at the bound of r = +-0.0 (the model agrees on the bits)
    d = rm.distances("angular", rows, q[:1])[0]
    cnt0 = int(np.count_nonzero(d <= 0.0))
    assert g.exact_range_count(q[:1], -0.0, already_element=True)[0] == cnt0
    rows8 = np.concatenate([_rows("angular_int", random_vectors(40, 64, 2))] * 3 + [np.zeros((20, 64), np.int8)])
    g8, c8 = _dense(oracle, "angular_int", rows8)
    q8 = np.concatenate([rows8[:4], np.zeros((1, 64), np.int8)])
    for r in (0.0, -0.0, 1.0, np.float32(np.inf), -0.5):
        _check(g8, c8, q8, r)
    for gg, qq in ((g, q), (g8, q8)):
        for fn in (gg.exact_range_count, gg.exact_range_search):
            with pytest.raises(granne_b200.GranneError) as e:
                fn(qq, np.nan)
            assert e.value.code == INVALID


def test_model_is_a_second_statement(oracle):
    rows = _rows("angular", random_vectors(500, 48, 3))
    g, _ = _dense(oracle, "angular", rows)
    q = rows[[1, 2, 3]]
    d = rm.distances("angular", rows, q)
    r = np.sort(d[0])[70]
    off, ids, dists = g.exact_range_search(q, r, already_element=True)
    for i in range(3):
        want = rm.rank(d[i], np.flatnonzero(d[i] <= r), len(rows))
        seg = slice(int(off[i]), int(off[i + 1]))
        assert ids[seg].tolist() == [w[0] for w in want]
        assert dists[seg].view(np.uint32).tolist() == np.array([w[1] for w in want], np.float32).view(np.uint32).tolist()


def test_segments_across_slabs_and_chunks(oracle):
    # 1025 queries: two chunks; a slab of the first holds 65536 rows, so every query's range spans a full slab and a
    # short one; ranges of about 6000 entries sort past one shared-memory tile
    n, dim = 65536 + 129, 8
    rows = _rows("angular", random_vectors(n, dim, 8))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(1025, dim, 9)
    off = _check(g, c, q, _kth(c, q, 6000))
    assert np.diff(off).max() > 4096
    # the whole index per query: segments of 65665, the global steps of the sort
    _check(g, c, q[:2], np.float32(np.inf))


@pytest.mark.parametrize("nq", [1, 63, 64, 65, 1023, 1024, 1025])
def test_nq_around_the_query_block_and_chunk(oracle, nq):
    rows = _rows("angular_int", random_vectors(300, 100, 2))
    g, c = _dense(oracle, "angular_int", rows)
    q = random_vectors(nq, 100, 3)
    _check(g, c, q, _kth(c, q, 30))


@pytest.mark.parametrize("n", [1, 5, 127, 128, 129, 255, 257])
def test_n_around_the_row_tile(oracle, n):
    rows = _rows("angular", random_vectors(n, 128, n))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(3, 128, 1)
    _check(g, c, q, np.float32(np.inf))
    _check(g, c, q, _kth(c, q, min(n - 1, 9)))


def test_index_shorter_than_container_and_empty(oracle):
    rows = _rows("angular", random_vectors(500, 96, 4))
    q = random_vectors(20, 96, 5)
    for n in (0, 1, 300):
        g, c = _dense(oracle, "angular", rows, index_len=n)
        assert np.array_equal(g.exact_range_count(q, np.inf), np.full(20, n, np.uint64))
        off, ids, _ = g.exact_range_search(q, np.inf)
        assert (ids < n).all() and int(off[-1]) == 20 * n
        _check(g, c, q, np.float32(1.0), n=n)
    g, _ = _dense(oracle, "angular", rows)
    off, ids, dists = g.exact_range_search(np.zeros((0, 96), np.float32), 1.0)
    assert off.tolist() == [0] and ids.size == 0 and dists.size == 0


def test_by_id_and_excluding(oracle):
    base = _rows("angular", random_vectors(200, 32, 6))
    rows = np.concatenate([base, base[:10]])  # duplicates of 0..9 at 200..209
    g, c = _dense(oracle, "angular", rows)
    ids = np.array([0, 5, 150, 209, 0], np.uint32)
    r = _kth(c, rows[ids], 25, already_element=True)
    want = g.exact_range_search(rows[ids], r, already_element=True)
    _same(g.exact_range_search(ids, r, by_id=True), want)
    k = int(np.diff(want[0]).max()) + 1
    exc = _want(c, rows[ids], r, len(rows), k=k, already_element=True, self_ids=ids)
    _same(g.exact_range_search(ids, r, exclude_self=True), exc)
    assert np.array_equal(g.exact_range_count(ids, r, exclude_self=True), np.diff(exc[0]))
    # the duplicate stays: query 0 finds 200, query 209 finds 9, both at distance 0
    seg = exc[1][int(exc[0][0]):int(exc[0][1])]
    assert 200 in seg.tolist() and 0 not in seg.tolist()
    # a radius below the self distance: nothing to remove
    assert np.array_equal(g.exact_range_count(ids, -1.0, exclude_self=True), np.zeros(5, np.uint64))
    for fn in (g.exact_range_count, g.exact_range_search):
        with pytest.raises(granne_b200.GranneError) as e:
            fn(np.array([3, len(rows)], np.uint32), r, by_id=True)
        assert e.value.code == OUT_OF_RANGE


def test_device_calls_and_bad_ids(oracle):
    import torch

    rows = _rows("angular", random_vectors(300, 32, 7))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(50, 32, 8)
    r = float(_kth(c, q, 40))
    want = g.exact_range_search(q, r)
    s = torch.cuda.Stream()
    dq = torch.from_numpy(q).cuda()
    with torch.cuda.stream(s):
        cnt = g.exact_range_count_device(dq, r, stream=s)
        off = torch.zeros(51, dtype=torch.int64, device="cuda")
        torch.cumsum(cnt, 0, out=off[1:])
        ids, dists = g.exact_range_search_device(dq, r, off, stream=s)
    g.stream_status(s)
    _same((off.cpu().numpy(), ids.cpu().numpy().view(np.uint32), dists.cpu().numpy()), want)
    # by id with a bad id: count 0, an empty segment, ERR_OUT_OF_RANGE from the stream; the others unaffected
    qid = torch.tensor([4, 300, 7, -1], dtype=torch.int32, device="cuda")
    host_ok = g.exact_range_search(np.array([4, 7], np.uint32), r, exclude_self=True)
    with torch.cuda.stream(s):
        cnt = g.exact_range_count_device(qid, r, exclude_self=True, stream=s)
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status(s)
    assert e.value.code == OUT_OF_RANGE
    ch = cnt.cpu().numpy()
    assert ch[1] == 0 and ch[3] == 0 and ch[0] == host_ok[0][1] and ch[2] == host_ok[0][2] - host_ok[0][1]
    with torch.cuda.stream(s):
        off = torch.zeros(5, dtype=torch.int64, device="cuda")
        torch.cumsum(cnt, 0, out=off[1:])
        ids, dists = g.exact_range_search_device(qid, r, off, exclude_self=True, stream=s)
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status(s)
    assert e.value.code == OUT_OF_RANGE
    o = off.cpu().numpy()
    got_ids = ids.cpu().numpy().view(np.uint32)
    assert o[2] == o[1] and o[4] == o[3]
    assert np.array_equal(got_ids, host_ok[1]) and np.array_equal(dists.cpu().numpy(), host_ok[2])
    g.release_stream(s)


def test_mismatched_offsets_pad_and_stay_inside(oracle):
    import torch

    rows = _rows("angular", random_vectors(400, 16, 9))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(4, 16, 10)
    r = float(_kth(c, q, 30))
    good = g.exact_range_search(q, r)
    cnt = np.diff(good[0]).astype(np.int64)
    lens = cnt.copy()
    lens[1] -= 1  # too short
    lens[2] += 3  # too long
    off = np.zeros(5, np.uint64)
    np.cumsum(lens, out=off[1:])
    total = int(off[-1])
    guard = 0xA5A5A5A5
    ids = np.full(total + 2, guard, np.uint32)
    d = np.full(total + 2, guard, np.uint32)
    lib = granne_b200.load_library()
    rc = lib.granne_b200_exact_range_search(g._h, api._ptr(q), 4, api.QUERY_RAW_F32, r, api._ptr(off),
                                            C.c_void_p(ids.ctypes.data + 4), C.c_void_p(d.ctypes.data + 4))
    assert rc == INVALID
    assert ids[0] == guard and ids[-1] == guard and d[0] == guard and d[-1] == guard

    def check(ids_in, d_in):
        for qi in range(4):
            seg = slice(int(off[qi]), int(off[qi + 1]))
            gseg = slice(int(good[0][qi]), int(good[0][qi + 1]))
            if qi in (1, 2):
                assert (ids_in[seg] == U32_MAX).all() and (d_in[seg].view(np.float32) == np.inf).all()
            else:
                assert np.array_equal(ids_in[seg], good[1][gseg])
                assert np.array_equal(d_in[seg], good[2][gseg].view(np.uint32))

    check(ids[1:-1], d[1:-1])
    # the device call: the same segments, reported by the stream
    s = torch.cuda.Stream()
    dq = torch.from_numpy(q).cuda()
    tid = torch.full((total + 2,), guard - 2**32, dtype=torch.int64, device="cuda").to(torch.int32)
    td = torch.from_numpy(np.full(total + 2, guard, np.uint32).view(np.int32)).cuda().view(torch.float32)
    toff = torch.from_numpy(off.view(np.int64)).cuda()
    with torch.cuda.stream(s):
        g.exact_range_search_device(dq, r, toff, out=(tid[1:-1], td[1:-1]), stream=s)
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status(s)
    assert e.value.code == INVALID
    hi, hd = tid.cpu().numpy().view(np.uint32), td.cpu().numpy().view(np.uint32)
    assert hi[0] == guard and hi[-1] == guard and hd[0] == guard and hd[-1] == guard
    check(hi[1:-1], hd[1:-1])
    # offsets that go backwards write nothing
    back = torch.tensor([0, 5, 2, 2, 2], dtype=torch.int64, device="cuda")
    tid2 = torch.full((8,), 7, dtype=torch.int32, device="cuda")
    td2 = torch.zeros(8, dtype=torch.float32, device="cuda")
    with torch.cuda.stream(s):
        g.exact_range_search_device(dq, r, back, out=(tid2, td2), stream=s)
    with pytest.raises(granne_b200.GranneError):
        g.stream_status(s)
    assert (tid2.cpu().numpy()[5:] == 7).all()
    g.release_stream(s)


def test_nan_element(oracle):
    rows = _rows("angular", random_vectors(200, 32, 1)).copy()
    rows[77, 3] = np.nan
    g, _ = _dense(oracle, "angular", rows)
    q = random_vectors(2, 32, 2)
    for r in (0.5, -1.0, np.inf):  # the scan runs whatever the radius
        for fn in (g.exact_range_count, g.exact_range_search):
            with pytest.raises(granne_b200.GranneError) as e:
                fn(q, r)
            assert e.value.code == NOT_FINITE


def test_device_calls_on_two_streams_concurrent_with_search(oracle):
    import torch

    el = oracle.Elements.angular(random_vectors(2000, 64, 3))
    gb = oracle.GranneBuilder(el, num_neighbors=10, max_search=50).build()
    g = granne_b200.Granne.from_bytes(gb.to_bytes(), "angular", el.to_bytes(0))
    q = random_vectors(300, 64, 4)
    r = float(g.exact_search_batch(q[:1], 100)[1][0, 99])
    want_range = g.exact_range_search(q, r)
    want_search = g.search_batch(q, 50, 10)
    streams = [torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()]
    dq = torch.from_numpy(q).cuda()
    outs = []

    def run_range(s):
        for _ in range(4):
            with torch.cuda.stream(s):
                cnt = g.exact_range_count_device(dq, r, stream=s)
                off = torch.zeros(301, dtype=torch.int64, device="cuda")
                torch.cumsum(cnt, 0, out=off[1:])
                total = int(want_range[0][-1])  # the output is sized without waiting for the device
                out = (torch.empty(total, dtype=torch.int32, device="cuda"),
                       torch.empty(total, dtype=torch.float32, device="cuda"))
                ids, dists = g.exact_range_search_device(dq, r, off, out=out, stream=s)
                s.synchronize()
                outs.append(("r", (off.cpu().numpy(), ids.cpu().numpy().view(np.uint32), dists.cpu().numpy())))

    def run_search(s):
        for _ in range(4):
            with torch.cuda.stream(s):
                res = g.search_batch_device(dq, 50, 10, stream=s)
                s.synchronize()
                outs.append(("s", [t.cpu().numpy() for t in res]))

    ts = [threading.Thread(target=run_range, args=(streams[0],)), threading.Thread(target=run_range, args=(streams[1],)),
          threading.Thread(target=run_search, args=(streams[2],))]
    [t.start() for t in ts]
    [t.join() for t in ts]
    g.stream_status()
    assert len(outs) == 12
    for tag, got in outs:
        if tag == "r":
            _same(got, want_range)
        else:
            i, d, c = got
            assert np.array_equal(i.view(np.uint32), want_search[0]) and np.array_equal(c.view(np.uint32), want_search[2])
            assert np.array_equal(d.view(np.uint32), want_search[1].view(np.uint32))


def test_multi_partitioned_and_replicated(oracle):
    sizes = [300, 1, 450]
    parts = [_rows("angular", random_vectors(s, 48, 10 + i)).copy() for i, s in enumerate(sizes)]
    parts[2][:5] = parts[0][:5]  # duplicates across shards: ties broken by global id
    shards = [(xo.single_layer_index(oracle, s), np.uint64(48).tobytes() + p.tobytes()) for s, p in zip(sizes, parts)]
    allrows = np.concatenate(parts)
    g, c = _dense(oracle, "angular", allrows)
    q = random_vectors(30, 48, 2)
    r = float(_kth(c, q, 60))
    want = g.exact_range_search(q, r)
    gids = np.array([0, 300, 301, 750, 3], np.uint64)
    want_id = g.exact_range_search(gids.astype(np.uint32), r, by_id=True)
    want_ex = g.exact_range_search(gids.astype(np.uint32), r, exclude_self=True)
    m = granne_b200.MultiGranne.partitioned(shards, "angular", [0, 0, 0])
    rep = granne_b200.MultiGranne.replicated(xo.single_layer_index(oracle, 751), "angular",
                                             np.uint64(48).tobytes() + allrows.tobytes(), [0, 0])
    for h in (m, rep):
        for got, w, kw in ((h.exact_range_search(q, r), want, {}),
                           (h.exact_range_search(gids, r, by_id=True), want_id, {"by_id": True}),
                           (h.exact_range_search(gids, r, exclude_self=True), want_ex, {"exclude_self": True})):
            assert got[1].dtype == np.uint64
            _same(got, (w[0], w[1], w[2]))
            assert np.array_equal(h.exact_range_count(gids if kw else q, r, **kw), np.diff(w[0]))
        with pytest.raises(granne_b200.GranneError) as e:
            h.exact_range_count(np.array([751], np.uint64), r, by_id=True)
        assert e.value.code == OUT_OF_RANGE
        with pytest.raises(granne_b200.GranneError) as e:
            h.exact_range_count(q, np.nan)
        assert e.value.code == INVALID
    # a mismatched segment is padded and reported, the others are written
    lib = granne_b200.load_library()
    off = want[0].copy()
    off[1:] += 1  # query 0's segment is one too long
    ids = np.zeros(int(off[-1]), np.uint64)
    d = np.zeros(int(off[-1]), np.float32)
    for h in (m, rep):
        assert lib.granne_b200_multi_exact_range_search(h._h, api._ptr(q), 30, 0, r, api._ptr(off), api._ptr(ids),
                                                        api._ptr(d)) == INVALID
        assert (ids[:int(off[1])] == 2**64 - 1).all()
        assert np.array_equal(ids[int(off[1]):], want[1][int(want[0][1]):].astype(np.uint64))
    m.close()
    rep.close()


def test_range_graph(oracle):
    raw = clustered_vectors(400, 32, 11)
    raw[200:210] = raw[:10]  # near duplicates
    rows = _rows("angular", raw)
    g, c = _dense(oracle, "angular", rows)
    r = 0.05
    for exclude in (True, False):
        off, ids, dists = g.range_graph(r, exclude_self=exclude, chunk=150)
        allq = np.arange(400, dtype=np.uint32)
        host = g.exact_range_search(allq, r, exclude_self=exclude, by_id=not exclude)
        _same((off, ids, dists), host)
        k = int(np.diff(host[0]).max()) + 2
        _same((off, ids, dists), _want(c, rows, r, 400, k=k, already_element=True,
                                       self_ids=allq if exclude else None))
    doff, dids, dd = g.range_graph(r, chunk=1000, out="device")
    _same((doff.cpu().numpy(), dids.cpu().numpy().view(np.uint32), dd.cpu().numpy()), g.range_graph(r))


def test_cxx_client(tmp_path, oracle):
    if shutil.which("g++") is None:
        pytest.skip("no C++ compiler")
    rows = _rows("angular", clustered_vectors(500, 64, 1))
    (tmp_path / "index").write_bytes(xo.single_layer_index(oracle, 500))
    (tmp_path / "elements").write_bytes(np.uint64(64).tobytes() + rows.tobytes())
    exe = tmp_path / "client"
    libdir = os.path.dirname(granne_b200.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", "cxx_range_client.cpp"), "-o", str(exe),
                           "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe), str(tmp_path / "index"), str(tmp_path / "elements"), "0.2"], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr
    g, _ = _dense(oracle, "angular", rows)
    assert int(out.stdout.split()[1]) == int(g.exact_range_count(np.arange(500, dtype=np.uint32), 0.2, by_id=True).sum())


def _identity_at_scale(g, q, r):
    """counts == segment lengths, and the first min(1024, |R(q)|) entries are exact_search_batch(q, 1024)'s within r."""
    cnt = g.exact_range_count(q, r)
    off, ids, dists = g.exact_range_search(q, r)
    assert np.array_equal(np.diff(off), cnt)
    ei, ed, ec = g.exact_search_batch(q, 1024)
    for i in range(q.shape[0]):
        keep = (np.arange(1024) < ec[i]) & (ed[i] <= np.float32(r))
        m = min(1024, int(cnt[i]))
        seg = slice(int(off[i]), int(off[i]) + m)
        assert keep.sum() == m and np.array_equal(ids[seg], ei[i][keep])
        assert np.array_equal(dists[seg].view(np.uint32), ed[i][keep].view(np.uint32))
    return cnt


def test_at_size_f32_1m():
    import torch

    n, dim = 1_000_000, 128
    rows = torch.from_numpy(clustered_vectors(n, dim, 11)).cuda()
    el = granne_b200.elements_from_raw_device("angular", rows)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(xo.single_layer_index(go, n), "angular", el)
    q = clustered_vectors(256, dim, 12)
    ed = g.exact_search_batch(q, 1024)[1]
    for r in (float(ed[0, 500]), float(np.median(ed[:, 1023]))):  # ranges below and past 1024 entries
        cnt = _identity_at_scale(g, q, r)
    assert cnt.min() < 1024 < cnt.max()


def test_at_size_i8_10m():
    import torch

    n, dim = 10_000_000, 100
    rng = np.random.default_rng(5)
    host = rng.integers(-128, 128, (n, dim), dtype=np.int8)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(xo.single_layer_index(go, n), "angular_int",
                                                torch.from_numpy(host).cuda())
    q = random_vectors(32, dim, 13)
    ed = g.exact_search_batch(q, 1024)[1]
    cnt = _identity_at_scale(g, q, float(np.median(ed[:, 1023])))
    assert cnt.min() < 1024 < cnt.max()
