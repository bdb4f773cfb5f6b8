"""Queries by element id on the GPU (GRANNE_B200_QUERY_ID / GRANNE_B200_QUERY_ID_EXCLUDING), batched element reads
(granne_b200_get_elements*) and the k-NN graph built on them.  A call by id equals the same call with
get_elements(ids) as ELEMENT queries (ids, distance bits, counts, stats 0..2) for every call, element kind and
distance engine, and the graph search equals the oracle's search of Elements.get(i); exclusion equals "k + 1, drop
self, cut to k".  Also: bad ids (host: before any launch; device: only that row blanked), builder snapshots, repeated
ids, nq = 0 and k = 0, concurrency, the multi handle and knn_graph."""
import threading

import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co
from helpers.data import build_fixture, index_from_lists, random_vectors
from helpers.fixtures import assert_same, cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

UNUSED = 0xFFFFFFFF
OUT_OF_RANGE = -8
CALLS = ["search", "exact", "within", "filtered"]


_CACHE = {}


def _index(oracle, kind, dim, n=600, dup=False):
    """(GPU handle, oracle Elements, oracle Granne) of a small built index; dup: rows 1 and 2 equal rows 0 and 3."""
    key = (kind, dim, n, dup)
    if key not in _CACHE:
        if dup:
            raw = random_vectors(n, dim, seed=dim)
            raw[1], raw[2] = raw[0], raw[3]
            el = oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)
            g = oracle.GranneBuilder(el, num_neighbors=10, max_search=40).build(threads=1)
            ib, eb, mb = g.to_bytes(), el.to_bytes(0), None
            og = oracle.Granne.from_bytes(ib, el)
        else:
            el, og, ib, eb, mb = build_fixture(oracle, kind, n, dim, seed=dim + n, num_neighbors=10, max_search=40)
        _CACHE[key] = (granne_b200.Granne.from_bytes(ib, kind, eb, mb), el, og)
    return _CACHE[key]


# every DistF32<FULL> width (FULL = 0, 1, 2, 3, 4, 6, 8), DistF32Generic, several i8 widths, embeddings
ENGINES = [("angular", d) for d in (8, 32, 64, 96, 128, 192, 256, 100)] + \
          [("angular_int", d) for d in (20, 100, 128)] + [("embeddings", 24)]


def _lists(rng, n, nq):
    return [rng.integers(0, n, size=int(rng.integers(0, 60))).astype(np.uint32) for _ in range(nq)]


def _host(g, call, q, k, lists=None, words=None, **kw):
    """(ids, dists, counts, stats or None) of a host call; q: rows (already_element) or ids (by_id / exclude_self)."""
    if call == "search":
        return g.search_batch(q, 40, k, with_stats=True, **kw)
    if call == "exact":
        return (*g.exact_search_batch(q, k, **kw), None)
    if call == "within":
        return (*g.exact_search_within(q, lists, k, **kw), None)
    return g.search_batch_filtered(q, words, max_search=40, num_elements=k, with_stats=True, **kw)


def _device(g, call, q, k, lists=None, words=None, **kw):
    import torch

    dev = torch.device("cuda", g.device)
    stats = torch.zeros((q.shape[0], 4), dtype=torch.int64, device=dev) if call in ("search", "filtered") else None
    if call == "search":
        r = g.search_batch_device(q, 40, k, stats=stats, **kw)
    elif call == "exact":
        r = g.exact_search_batch_device(q, k, **kw)
    elif call == "within":
        offs = np.zeros(len(lists) + 1, np.int64)
        np.cumsum([len(x) for x in lists], out=offs[1:])
        flat = np.concatenate(lists).astype(np.uint32) if lists else np.zeros(0, np.uint32)
        r = g.exact_search_within_device(q, torch.from_numpy(offs).to(dev),
                                         torch.from_numpy(flat.view(np.int32)).to(dev), k, **kw)
    else:
        r = g.search_batch_filtered_device(q, torch.from_numpy(words.view(np.int32)).to(dev), max_search=40,
                                           num_elements=k, stats=stats, **kw)
    torch.cuda.synchronize(dev)
    out = [t.cpu().numpy() for t in r]
    return (out[0].view(np.uint32), out[1], out[2].view(np.uint32),
            stats.cpu().numpy().view(np.uint64) if stats is not None else None)


def _exclude_model(res, ids, k):
    """QUERY_ID_EXCLUDING from the QUERY_ID result with k + 1 columns: self removed, cut to k (ids of the result's
    own dtype: u32, or u64 global ids, padded with its maximum)."""
    ri, rd, rc, rs = res
    nq = len(ids)
    oi = np.full((nq, k), np.iinfo(ri.dtype).max, ri.dtype)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for q in range(nq):
        keep = [j for j in range(int(rc[q])) if ri[q, j] != ids[q]][:k]
        oi[q, :len(keep)] = ri[q, keep]
        od[q, :len(keep)] = rd[q, keep]
        oc[q] = len(keep)
    return oi, od, oc, rs


@pytest.mark.parametrize("kind,dim", ENGINES)
def test_get_elements_equal_get_element(oracle, kind, dim):
    import torch

    g, el, _ = _index(oracle, kind, dim)
    ids = np.array([0, 5, 599, 5, 17, 300], np.uint32)
    want = np.stack([g.get_element(int(i)) for i in ids])
    got = g.get_elements(ids)
    assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8))
    assert np.array_equal(got.view(np.uint8), np.stack([el.get(int(i)) for i in ids]).view(np.uint8))
    dev = g.get_elements_device(torch.from_numpy(ids.view(np.int32)).cuda(g.device))
    assert np.array_equal(dev.cpu().numpy().view(np.uint8), want.view(np.uint8))
    assert g.get_elements(np.zeros(0, np.uint32)).shape == (0, g.dim)


@pytest.mark.parametrize("call", CALLS)
@pytest.mark.parametrize("kind,dim", ENGINES)
def test_id_call_equals_element_call(oracle, kind, dim, call):
    import torch

    g, _, _ = _index(oracle, kind, dim)
    rng = np.random.default_rng(dim)
    ids = np.concatenate([rng.integers(0, 600, size=70), [3, 3, 599]]).astype(np.uint32)  # repeated ids too
    lists = _lists(rng, 600, len(ids))
    words = rng.integers(0, 2**32, size=(1, 19), dtype=np.uint64).astype(np.uint32)
    rows = g.get_elements(ids)
    for k in (0, 1, 10, 45):
        want = _host(g, call, rows, k, lists, words, already_element=True)
        assert_same(_host(g, call, ids, k, lists, words, by_id=True), want, stats=True)
        d_ids = torch.from_numpy(ids.view(np.int32)).cuda(g.device)
        assert_same(_device(g, call, d_ids, k, lists, words, by_id=True), want, stats=True)
        kk = min(k + 1, 1024)
        model = _exclude_model(_host(g, call, ids, kk, lists, words, by_id=True), ids, k)
        assert_same(_host(g, call, ids, k, lists, words, exclude_self=True), model, stats=True)
        assert_same(_device(g, call, d_ids, k, lists, words, exclude_self=True), model, stats=True)
    g.stream_status()


@pytest.mark.parametrize("kind,dim", [("angular", 32), ("angular_int", 100), ("embeddings", 24)])
def test_search_by_id_equals_the_oracle(oracle, kind, dim):
    g, el, og = _index(oracle, kind, dim)
    ids = np.arange(0, 600, 7, dtype=np.uint32)
    rows = np.stack([el.get(int(i)) for i in ids])
    wi, wd, wc, ws = og.search_batch(rows, 40, 12, already_element=True, with_stats=True)
    gi, gd, gc, gs = g.search_batch(ids, 40, 12, by_id=True, with_stats=True)
    assert_same((gi, gd, gc, gs), (wi, wd, wc, np.c_[ws, np.zeros(len(ids), np.uint64)]), stats=True)
    c = co.Container(kind, el.to_bytes(0), el.to_bytes(1) if kind == "embeddings" else None)
    assert_same((*g.exact_search_batch(ids, 12, by_id=True), None),
                (*c.exact_search(rows, 12, index_len=len(g), already_element=True), None), stats=True)


def test_exclusion_edges(oracle):
    import torch

    g, _, _ = _index(oracle, "angular", 32, dup=True)
    ids = np.array([0, 1, 2, 3, 10], np.uint32)
    # duplicates: the twin stays at distance 0, self is dropped
    ei, ed, ec = g.exact_search_batch(ids, 5, exclude_self=True)
    assert ei[0, 0] == 1 and ei[1, 0] == 0 and ei[2, 0] == 3 and ei[3, 0] == 2 and ed[0, 0] == 0
    assert not any(ids[q] in ei[q, :ec[q]] for q in range(len(ids)))
    # self not among the first k + 1 of a within list that does not hold it: plain cut to k
    lists = [np.array([5, 6, 7, 8], np.uint32)] * len(ids)
    wi = g.exact_search_within(ids, lists, 2, exclude_self=True)
    assert np.array_equal(wi[0], g.exact_search_within(ids, lists, 2, by_id=True)[0])
    # k > max_search: at most max_search results exist; without self one fewer when self is found
    got = g.search_batch(ids, 5, 20, exclude_self=True, with_stats=True)
    assert_same(got, _exclude_model(g.search_batch(ids, 5, 21, by_id=True, with_stats=True), ids, 20), stats=True)
    assert (got[2] <= 5).all()
    # k = 1023 on the capped calls
    words = np.full((1, 19), 0xFFFFFFFF, np.uint32)
    for call in ("exact", "within", "filtered"):
        res = _host(g, call, ids, 1023, [np.arange(600, dtype=np.uint32)] * len(ids), words, exclude_self=True)
        model = _exclude_model(_host(g, call, ids, 1024, [np.arange(600, dtype=np.uint32)] * len(ids), words,
                                     by_id=True), ids, 1023)
        assert_same(res, model, stats=True)
        with pytest.raises(granne_b200.GranneError):
            _host(g, call, ids, 1024, [np.arange(600, dtype=np.uint32)] * len(ids), words, exclude_self=True)
    # nq = 0 in every call, host and device
    for call in CALLS:
        assert _host(g, call, np.zeros(0, np.uint32), 5, [], words, exclude_self=True)[0].shape == (0, 5)
        d0 = torch.zeros(0, dtype=torch.int32, device="cuda:%d" % g.device)
        assert _device(g, call, d0, 5, [], words, by_id=True)[0].shape == (0, 5)


@pytest.mark.parametrize("kind,dim", [("angular", 64), ("angular_int", 100), ("embeddings", 24)])
def test_bad_ids(oracle, kind, dim):
    # the zero row a bad id reads goes through each engine's query path (DistF32, DistI8's qnorm, DistSum)
    import torch

    g, _, _ = _index(oracle, kind, dim)
    bad = np.array([1, 600, 2], np.uint32)
    before = g.launch_count()
    for call in CALLS:
        with pytest.raises(granne_b200.GranneError) as ei:
            _host(g, call, bad, 5, _lists(np.random.default_rng(0), 600, 3), np.ones((1, 19), np.uint32),
                  by_id=True)
        assert ei.value.code == OUT_OF_RANGE
    with pytest.raises(granne_b200.GranneError) as ei:
        g.get_elements(bad)
    assert ei.value.code == OUT_OF_RANGE
    assert g.launch_count() == before  # rejected before any launch
    words = np.ones((1, 19), np.uint32) * 0xFFFFFFFF
    lists = [np.arange(50, dtype=np.uint32)] * 3
    good = np.array([1, 2], np.uint32)
    d_bad = torch.from_numpy(bad.view(np.int32)).cuda(g.device)
    for call in CALLS:
        for excl in (False, True):
            kw = {"exclude_self": True} if excl else {"by_id": True}
            got = _device(g, call, d_bad, 5, lists, words, **kw)
            want = _host(g, call, good, 5, lists[:2], words, **kw)
            assert got[2][1] == 0 and (got[0][1] == UNUSED).all() and np.isinf(got[1][1]).all()
            if got[3] is not None:
                assert (got[3][1] == 0).all()
            assert_same(tuple(None if x is None else x[[0, 2]] for x in got), want, stats=True)
            with pytest.raises(granne_b200.GranneError) as ei:
                g.stream_status()
            assert ei.value.code == OUT_OF_RANGE
    rows = g.get_elements_device(d_bad)
    torch.cuda.synchronize()
    assert (rows[1] == 0).all() and np.array_equal(rows[[0, 2]].cpu().numpy(), g.get_elements(good))
    with pytest.raises(granne_b200.GranneError):
        g.stream_status()
    g.stream_status()  # reported once


def test_builder_snapshot_ids_past_len():
    raw = random_vectors(1500, 32, seed=5)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw[:1000]), num_neighbors=10,
                                  max_search=40)
    b.build()
    for r in raw[1000:]:
        b.append(r)
    g = b.get_index()
    assert len(g) == 1000 and g.num_elements() == 1500
    ids = np.array([999, 1000, 1499, 1200], np.uint32)
    rows = g.get_elements(ids)
    assert_same(_host(g, "search", ids, 8, by_id=True), _host(g, "search", rows, 8, already_element=True), stats=True)
    assert_same(_host(g, "exact", ids, 8, exclude_self=True),
                _exclude_model(_host(g, "exact", ids, 9, by_id=True), ids, 8), stats=True)
    with pytest.raises(granne_b200.GranneError):
        g.search_batch(np.array([1500], np.uint32), 40, 8, by_id=True)


def test_retry_and_slow_passes(oracle):
    # uniform data on a fresh handle (test_parity_regimes_gpu's mixed ladder): the visited tables start at their base
    # size, so part of the batch overflows the fast pass into the retry or slow pass (stats column 3 >= 1)
    n, dim, ef = 20_000, 24, 40
    el = oracle.Elements.angular(random_vectors(n, dim, seed=41))
    ib = oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8).to_bytes()
    g = granne_b200.Granne.from_bytes(ib, "angular", el.to_bytes(0))
    ids = np.arange(n, dtype=np.uint32)
    got = g.search_batch(ids, ef, 10, by_id=True, with_stats=True)
    flags = got[3][:, 3]
    assert (flags == 0).any() and (flags >= 1).any(), np.bincount(flags.astype(np.int64))
    assert_same(got, g.search_batch(g.get_elements(ids), ef, 10, already_element=True, with_stats=True), stats=True)
    assert_same(g.search_batch(ids, ef, 10, exclude_self=True, with_stats=True),
                _exclude_model(g.search_batch(ids, ef, 11, by_id=True, with_stats=True), ids, 10), stats=True)
    g.close()
    # the all-identical plateau (test_parity_regimes_gpu): every query is answered by the slow pass
    n, dim = 400, 8
    el = oracle.Elements.angular(np.tile(random_vectors(1, dim, seed=5), (n, 1)))
    nb = [sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]
    ib = index_from_lists(oracle, [nb])
    og = oracle.Granne.from_bytes(ib, el)
    g = granne_b200.Granne.from_bytes(ib, "angular", el.to_bytes(0))
    ids = np.arange(0, n, 3, dtype=np.uint32)
    got = g.search_batch(ids, 20, 10, by_id=True, with_stats=True)
    assert (got[3][:, 3] == 2).all()
    wi, wd, wc, ws = og.search_batch(np.stack([el.get(int(i)) for i in ids]), 20, 10, already_element=True,
                                     with_stats=True)
    assert_same(got, (wi, wd, wc, ws), stats=True)
    got = g.search_batch(ids, 20, 10, exclude_self=True, with_stats=True)
    assert (got[3][:, 3] == 2).all()
    assert_same(got, _exclude_model((*og.search_batch(np.stack([el.get(int(i)) for i in ids]), 20, 11,
                                                      already_element=True), None), ids, 10), stats=True)
    g.close()


def test_concurrent_device_calls(oracle):
    import torch

    g, _, _ = _index(oracle, "angular", 128)
    ids = np.arange(600, dtype=np.uint32)
    raw = random_vectors(300, 128, seed=9)
    want_id = g.search_batch(ids, 40, 10, exclude_self=True)
    want_raw = g.search_batch(raw, 40, 10)
    errors = []

    def worker(t):
        try:
            s = torch.cuda.Stream(device=g.device)
            d_ids = torch.from_numpy(ids.view(np.int32)).cuda(g.device)
            d_raw = torch.from_numpy(raw).cuda(g.device)
            for _ in range(4):
                with torch.cuda.stream(s):
                    r1 = g.search_batch_device(d_ids, 40, 10, exclude_self=True, stream=s)
                    r2 = g.search_batch_device(d_raw, 40, 10, stream=s)
                s.synchronize()
                assert np.array_equal(r1[0].cpu().numpy().view(np.uint32), want_id[0])
                assert np.array_equal(r2[0].cpu().numpy().view(np.uint32), want_raw[0])
            g.release_stream(s)
        except Exception as e:  # noqa: BLE001 - reported on the main thread
            errors.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    g.stream_status()


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_multi_handle(oracle, mode):
    parts = []
    for s in range(3):
        el, _, ib, eb, _ = build_fixture(oracle, "angular", 400 + 50 * s, 32, seed=70 + s, num_neighbors=10,
                                         max_search=40)
        parts.append((ib, eb))
    if mode == "replicated":
        m = granne_b200.MultiGranne.replicated(parts[0][0], "angular", parts[0][1], [0, 0, 0])
        singles = [granne_b200.Granne.from_bytes(parts[0][0], "angular", parts[0][1])]
        bases = [0]
    else:
        m = granne_b200.MultiGranne.partitioned(parts, "angular", [0, 0])
        singles = [granne_b200.Granne.from_bytes(ib, "angular", eb) for ib, eb in parts]
        bases = [m.shard_base(s) for s in range(3)]
    gids = np.concatenate([b + np.arange(0, len(g), 37) for b, g in zip(bases, singles)]).astype(np.uint64)
    rows = np.concatenate([g.get_elements(np.arange(0, len(g), 37, dtype=np.uint32)) for g in singles])
    words = np.full((1, (max(b + len(g) for b, g in zip(bases, singles)) + 31) // 32), 0xFFFFFFFF, np.uint32)
    lists = [np.array([0, 5, bases[-1] + 3, gid], np.uint64) for gid in gids]

    def run(call, q, k, **kw):
        if call == "search":
            return (*m.search_batch(q, 40, k, **kw), None)
        if call == "exact":
            return (*m.exact_search_batch(q, k, **kw), None)
        if call == "within":
            return (*m.exact_search_within(q, lists, k, **kw), None)
        return (*m.search_batch_filtered(q, words, max_search=40, num_elements=k, **kw), None)

    for call in CALLS:
        assert_same(run(call, gids, 10, by_id=True), run(call, rows, 10, already_element=True), stats=True)
        ri, rd, rc, _ = run(call, rows, 11, already_element=True)
        want = _exclude_model((ri, rd, rc, None), gids, 10)
        assert_same(run(call, gids, 10, exclude_self=True), want, stats=True)
    with pytest.raises(granne_b200.GranneError) as ei:
        m.search_batch(np.array([10**9], np.uint64), 40, 10, by_id=True)
    assert ei.value.code == OUT_OF_RANGE
    m.close()


def test_knn_graph(oracle):
    import glob
    import os

    golden = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))
    handles = []
    for path in golden:
        z = np.load(path)
        emb = z["embeddings"].tobytes() if z["embeddings"].size else None
        kind, eb = str(z["kind"]), z["elements"].tobytes()
        handles.append((granne_b200.Granne.from_bytes(z["index"].tobytes(), kind, eb, emb),
                        (oracle.Elements.from_bytes(kind, eb, emb), co.Container(kind, eb, emb))))
    raw = random_vectors(20000, 32, seed=11)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw), num_neighbors=16,
                                  max_search=60)
    b.build()
    handles.append((b.get_index(), None))
    for g, el in handles:
        n = len(g)
        ids = np.arange(n, dtype=np.uint32)
        gi, gd, gc = g.knn_graph(max_search=60, num_elements=8, chunk=777)
        assert_same((gi, gd, gc, None), (*g.search_batch(ids, 60, 8, exclude_self=True), None), stats=True)
        assert not (gi == ids[:, None]).any()
        xi, xd, xc = g.knn_graph(num_elements=8, exact=True, chunk=4096)
        assert_same((xi, xd, xc, None), (*g.exact_search_batch(ids, 8, exclude_self=True), None), stats=True)
        if el is not None:
            rows = np.stack([el[0].get(int(i)) for i in ids])
            wi, wd, wc = el[1].exact_search(rows, 9, index_len=n, already_element=True)
            assert_same((xi, xd, xc, None), _exclude_model((wi, wd, wc, None), ids, 8), stats=True)
        di, dd, dc = g.knn_graph(max_search=60, num_elements=8, exclude_self=False, out="device")
        assert_same((di.cpu().numpy().view(np.uint32), dd.cpu().numpy(), dc.cpu().numpy().view(np.uint32), None),
                    (*g.search_batch(ids, 60, 8, by_id=True), None), stats=True)


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_multi_knn_graph(oracle, mode):
    # MultiGranne.knn_graph against the merged exact oracle: every shard's exact list of each element, merged by
    # (distance, global id), self dropped, cut to k
    shards = []
    for s in range(3):
        el, _, ib, eb, _ = build_fixture(oracle, "angular", 300 + 40 * s, 16, seed=90 + s, num_neighbors=10,
                                         max_search=40)
        shards.append((ib, eb, el))
    if mode == "replicated":
        shards = shards[:1]
        m = granne_b200.MultiGranne.replicated(shards[0][0], "angular", shards[0][1], [0, 0])
        bases = [0]
    else:
        m = granne_b200.MultiGranne.partitioned([(ib, eb) for ib, eb, _ in shards], "angular", [0, 0])
        bases = [m.shard_base(s) for s in range(len(shards))]
    gids = m.global_ids()
    assert gids.size == len(m) and np.array_equal(gids, np.arange(len(m), dtype=np.uint64))
    rows = np.concatenate([np.stack([el.get(i) for i in range(len(el))]) for _, _, el in shards])
    k = 6
    per = []
    for (_, eb, el), b in zip(shards, bases):
        li, ld, lc = co.Container("angular", eb).exact_search(rows, k + 1, index_len=len(el), already_element=True)
        per.append((np.where(li == UNUSED, np.uint64(2**64 - 1), li.astype(np.uint64) + np.uint64(b)), ld, lc))
    wi = np.full((len(gids), k + 1), np.uint64(2**64 - 1))
    wd = np.full((len(gids), k + 1), np.inf, np.float32)
    wc = np.zeros(len(gids), np.uint32)
    for q in range(len(gids)):
        cand = [(d, i) for pi, pd, pc in per for i, d in zip(pi[q, :pc[q]], pd[q, :pc[q]])]
        cand.sort(key=lambda t: (t[0], int(t[1])))
        cand = cand[:k + 1]
        wc[q] = len(cand)
        wi[q, :len(cand)] = [i for _, i in cand]
        wd[q, :len(cand)] = [d for d, _ in cand]
    want = _exclude_model((wi, wd, wc, None), gids, k)
    xi, xd, xc = m.knn_graph(num_elements=k, exact=True, chunk=97)
    assert_same((xi, xd, xc, None), want, stats=True)
    assert not (xi == gids[:, None]).any()
    gi, gd, gc = m.knn_graph(max_search=40, num_elements=k, chunk=128)
    assert_same((gi, gd, gc, None), (*m.search_batch(gids, 40, k, exclude_self=True), None), stats=True)
    assert not (gi == gids[:, None]).any()
    m.close()


def test_knn_graph_reports_only_its_own_stream(oracle):
    import torch

    g, _, _ = _index(oracle, "angular", 64)
    d_bad = torch.tensor([1, 600], dtype=torch.int32, device="cuda:%d" % g.device)
    g.search_batch_device(d_bad, 40, 5, by_id=True)  # an error left on the current stream
    g.knn_graph(max_search=40, num_elements=5)       # does not consume it, nor fail because of it
    with pytest.raises(granne_b200.GranneError) as ei:
        g.stream_status()
    assert ei.value.code == OUT_OF_RANGE


def test_cxx_ids_client(oracle, tmp_path):
    el, _, ib, eb, _ = build_fixture(oracle, "angular", 1500, 32, seed=21, num_neighbors=12, max_search=50)
    (tmp_path / "index").write_bytes(ib)
    (tmp_path / "elements").write_bytes(eb)
    out = cxx_client("cxx_ids_client.cpp", [tmp_path / "index", tmp_path / "elements"], tmp_path, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stdout + out.stderr
    assert float(out.stdout.split()[1]) > 0.95  # verify_search's bar (src/index/tests.rs:50-62)
