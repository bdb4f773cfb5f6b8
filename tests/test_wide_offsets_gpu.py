"""Every query call on containers past the 32-bit row offsets, bit for bit against the NumPy model (ref_model.py).

The headline configuration (50M x 128 f32) holds 25.6 GB of rows: an id above 2^22 starts past 2^31 bytes, one above
2^25 past 2^32 floats.  Each case below opens a container of n = 2^25 + 4096 rows whose ids past each boundary hold
rows of their own (helpers/wide_fixture.py), so a row address computed in 32 bits anywhere on a call's path reads
another id's row and the call's ids or distance bits differ from the model's.

  case                      engine and layout                       row     container   ids past
  angular 128               DistF32<4>, lane-permuted               512 B   17.2 GB     2^31 B .. 2^32 floats (2^25)
  angular_int 513           DistI8, one row at a time               544 B   18.3 GB     2^31 B .. 2^34 B (31.6M)
  angular_int 100           DistI8, sub-warp groups (128-byte rows) 128 B    4.3 GB     2^31 B, 2^32 B (2^25)
  re-rank: angular_int 128  DistI8 stage 1, DistF32<4> stage 2      128 B + 512 B       stage 2 past 2^32 floats
  with angular 128 rows

The cases run one after another, each on a fresh handle whose tensors are dropped before the next; a case needs the
caller's rows and the library's copy at once (up to about 42 GB in use on the device) and is skipped, saying
so, when the device has less free."""
import time

import numpy as np
import pytest

import granne_b200
from helpers import ref_model as M
from helpers.fixtures import library  # noqa: F401  (autouse)
from helpers.model_checks import assert_same, assert_within_f64_bound, bits
from helpers.wide_fixture import (NUM_QUERIES, Bits, Wide, first_id_at, rank, row_bytes, sparse_graph, sparse_index,
                                  words_of)

pytestmark = pytest.mark.gpu

N = (1 << 25) + 4096
GB = 10 ** 9
# (kind, dim, (engine, layout), the byte boundaries 2^k that n rows of the case cross)
CASES = [
    ("angular", 128, ("DistF32<4>", "no tail"), (1 << 31, 1 << 32, 1 << 33, 1 << 34)),
    ("angular_int", 513, ("DistI8", "one row at a time"), (1 << 31, 1 << 32, 1 << 33, 1 << 34)),
    ("angular_int", 100, ("DistI8", "sub-warp groups"), (1 << 31, 1 << 32)),
]
# the two-stage case: the angular_int index (stage 1) and the attached angular rows (stage 2)
RERANK = [("angular_int", 128, ("DistI8", "sub-warp groups"), (1 << 31, 1 << 32)),
          ("angular", 128, ("DistF32<4>", "no tail"), (1 << 31, 1 << 32, 1 << 33, 1 << 34))]
EF, K = 64, 10             # graph search
KW, KF = 100, 64           # within lists, filtered
MARGIN = 3 * GB            # layers, workspaces and the model's device tensors


def _host(t):
    return t.cpu().numpy()


def _need(torch, what, nbytes):
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("%s needs %.1f GB of free device memory; %.1f GB of %.1f GB are free"
                    % (what, nbytes / GB, free / GB, total / GB))


def _used(torch):
    free, total = torch.cuda.mem_get_info()
    return total - free


def _members(m, seed):
    """C of the sparse graph: the planted ids and about 2000 palette ids spread over [0, n)."""
    rng = np.random.default_rng(seed)
    return np.concatenate([m.planted, rng.integers(0, m.n, size=2000)])


def _open(torch, oracle, m, seed):
    """(handle, layers, used device bytes while the caller's rows and the library's copy coexist)."""
    layers = sparse_graph(m.n, _members(m, seed), seed)
    image = sparse_index(oracle, layers)
    rows = m.device_rows(torch, torch.device("cuda", 0))
    p = granne_b200.Granne.from_device_elements(image, m.kind, rows)
    torch.cuda.synchronize()
    peak = _used(torch)
    del rows
    torch.cuda.empty_cache()
    return p, layers, peak


def _layer_bytes(layers):
    return sum(len(adj) * max(len(l) for l in adj.lists.values()) * 4 for adj in layers)


def _assert_range(got, want, what):
    """got: (offsets, ids, dists) of a range search; want: [[(id, dist)]] per query."""
    offsets, ids, dists = (np.asarray(x) for x in got)
    offsets = offsets.view(np.uint64) if offsets.dtype == np.int64 else offsets
    assert np.array_equal(np.diff(offsets.astype(np.int64)), [len(w) for w in want]), "%s: counts" % what
    for q, w in enumerate(want):
        seg = slice(int(offsets[q]), int(offsets[q + 1]))
        assert np.array_equal(ids[seg].view(np.uint32), np.array([i for i, _ in w], dtype=np.uint32)), \
            "%s: ids of query %d" % (what, q)
        assert np.array_equal(bits(dists[seg]), bits(np.array([x for _, x in w], dtype=np.float32))), \
            "%s: distance bits of query %d" % (what, q)


def _in_range(d, r):
    ids = np.flatnonzero(d <= r)
    return rank(d, ids.size, ids)


@pytest.mark.parametrize("kind,dim,engine,boundaries", CASES, ids=["%s-%d" % (c[0], c[1]) for c in CASES])
def test_query_calls_past_32_bit_offsets(oracle, kind, dim, engine, boundaries):
    import torch

    t0 = time.time()
    stride = row_bytes(kind, dim)
    _need(torch, "%s dim %d" % (kind, dim), 2 * N * stride + MARGIN)
    seed = dim
    m = Wide(kind, dim, N, boundaries, seed)
    p, layers, peak = _open(torch, oracle, m, seed)
    f32 = kind == "angular"
    qarg = dict(already_element=True) if f32 else {}
    nq = NUM_QUERIES
    qe, raw = m.queries, m.raw_queries
    tq, traw = torch.from_numpy(qe).cuda(), torch.from_numpy(raw).cuda()
    try:
        assert len(p) == N and p.dim == dim
        assert p.device_bytes() >= N * stride + _layer_bytes(layers)

        # elements as stored, at every boundary and both ends
        probe = np.concatenate([m.boundary, [0, 1, N - 2, N - 1, m.copy_id]]).astype(np.uint32)
        want_rows = m.rows(probe)
        for i, w in zip(probe, want_rows):
            assert p.get_element(int(i)).tobytes() == w.tobytes(), "get_element(%d)" % i
        assert p.get_elements(probe).tobytes() == want_rows.tobytes()
        got = _host(p.get_elements_device(torch.from_numpy(probe.astype(np.int32)).cuda()))
        assert got.tobytes() == want_rows.tobytes()

        # the model's answers, one query's distance vector at a time
        lab = m.all_labels()
        planted_d = [m.D[q, m.planted_label[m.planted_query == q]] for q in range(nq)]
        r_small = float(max(d.max() for d in planted_d))               # only the planted rows
        r_large = float(max(m.D[q, q] for q in range(nq)))              # and each query's nearest palette row
        rng = np.random.default_rng(seed + 5)
        top = first_id_at(boundaries[-1], stride)
        lists = [np.concatenate([m.boundary, m.boundary[:3], m.planted[m.planted_query == q],
                                 rng.integers(0, N, size=50)]) for q in range(nq)]
        lists[1] = np.concatenate([np.arange(top, top + 2800), rng.integers(top, N, size=400)])
        lists = [rng.permutation(l).astype(np.uint32) for l in lists]
        admitted = [np.arange((1 << 25) - 64, N), np.unique(rng.integers(0, N, size=N // 100)), None, m.planted]
        words = np.stack([words_of(a, N) if a is not None else np.full((N + 31) // 32, 0xFFFFFFFF, np.uint32)
                          for a in admitted])
        qf = np.arange(nq) % len(admitted)
        want = {key: [] for key in ("exact", "small", "large", "within", "search", "fsearch")}
        want_f = [[] for _ in admitted]
        for q in range(nq):
            d = m.D[q][lab]
            want["exact"].append(rank(d, 1024))
            want["small"].append(_in_range(d, np.float32(r_small)))
            want["large"].append(_in_range(d, np.float32(r_large)))
            want["within"].append(rank(d, KW, lists[q]))
            for f, a in enumerate(admitted):
                want_f[f].append(want["exact"][q][:KF] if a is None else rank(d, KF, a))
            want["search"].append(M.search(layers, d, EF, K))
            want["fsearch"].append(M.filtered(layers, d, EF, K, Bits(words[qf[q]])))
        # the planted rows first, then the nearest palette rows' ids, across the whole range
        assert all(len(w) == 1024 and w[-1][0] not in set(m.planted.tolist()) for w in want["exact"])
        assert all(len(s) < 16 < len(l) for s, l in zip(want["small"], want["large"]))
        assert max(i for w in want["large"] for i, _ in w) >= top

        # exact k-NN: raw and element queries, host and device
        for k in (1, 10, 1024):
            w = [x[:k] for x in want["exact"]]
            assert_same(p.exact_search_batch(raw, k), w, k, "exact raw k=%d" % k)
            assert_same(p.exact_search_batch(qe, k, **qarg), w, k, "exact element k=%d" % k)
            got = p.exact_search_batch_device(tq, k, **qarg)
            assert_same([_host(t) for t in got], w, k, "exact device k=%d" % k)
        got = p.exact_search_batch_device(traw, 10)
        assert_same([_host(t) for t in got], [x[:10] for x in want["exact"]], 10, "exact device raw")
        if f32:
            assert_within_f64_bound(m, qe, p.exact_search_batch(qe, 1024, already_element=True))

        # exact range: planted rows only, then also each query's nearest palette row (~n / P ids across the range)
        for r, key in ((r_small, "small"), (r_large, "large")):
            w = want[key]
            assert np.array_equal(p.exact_range_count(qe, r, **qarg), [len(x) for x in w]), "range count %s" % key
            _assert_range(p.exact_range_search(qe, r, **qarg), w, "range %s" % key)
            _assert_range(p.exact_range_search(raw, r), w, "range raw %s" % key)
            cnt = p.exact_range_count_device(tq, r, **qarg)
            offsets = torch.zeros(nq + 1, dtype=torch.int64, device=cnt.device)
            torch.cumsum(cnt, 0, out=offsets[1:])
            got = p.exact_range_search_device(tq, r, offsets, **qarg)
            _assert_range((_host(offsets), _host(got[0]), _host(got[1])), w, "range device %s" % key)

        # within lists: boundary ids with duplicates, and one list of 3200 ids past the last boundary
        assert_same(p.exact_search_within(qe, lists, KW, **qarg), want["within"], KW, "within")
        offs = np.zeros(nq + 1, dtype=np.int64)
        np.cumsum([len(l) for l in lists], out=offs[1:])
        got = p.exact_search_within_device(tq, torch.from_numpy(offs).cuda(),
                                           torch.from_numpy(np.concatenate(lists).view(np.int32)).cuda(), KW, **qarg)
        assert_same([_host(t) for t in got], want["within"], KW, "within device")

        # exact filtered: each filter alone, then all four named in one chunk; the all-admitting one is exact k-NN
        for f in range(len(admitted)):
            assert_same(p.exact_search_filtered(qe, words, np.full(nq, f), KF, **qarg), want_f[f], KF,
                        "exact filtered %d" % f)
        assert_same(p.exact_search_filtered(raw, words[2:3], None, KF), want_f[2], KF, "exact filtered all, raw")
        mixed = [want_f[qf[q]][q] for q in range(nq)]
        assert_same(p.exact_search_filtered(qe, words, qf, KF, **qarg), mixed, KF, "exact filtered mixed")
        got = p.exact_search_filtered_device(tq, torch.from_numpy(words.view(np.int32)).cuda(),
                                             torch.from_numpy(qf.astype(np.int32)).cuda(), KF, **qarg)
        assert_same([_host(t) for t in got], mixed, KF, "exact filtered mixed device")
        all_f = p.exact_search_filtered(qe, words[2:3], None, KF, **qarg)
        full = p.exact_search_batch(qe, KF, **qarg)
        assert all(np.array_equal(a, b) for a, b in zip(all_f, full))

        # graph search over the sparse graph, with its counters; filtered search with four filters in one chunk
        ws = ([w[0] for w in want["search"]], [w[1] for w in want["search"]])
        assert_same(p.search_batch(qe, EF, K, with_stats=True, **qarg), ws, K, "search")
        assert_same(p.search_batch(raw, EF, K, with_stats=True), ws, K, "search raw")
        stats = torch.zeros((nq, 4), dtype=torch.int64, device="cuda")
        got = p.search_batch_device(tq, EF, K, stats=stats, **qarg)
        assert_same([_host(t) for t in got] + [_host(stats)], ws, K, "search device")
        wf = ([w[0] for w in want["fsearch"]], [w[1] for w in want["fsearch"]])
        assert_same(p.search_batch_filtered(qe, words, qf, EF, K, with_stats=True, **qarg), wf, K, "filtered search")

        # by element id at the boundary ids and both ends, with and without the element itself
        qid = np.unique(np.concatenate([m.boundary, [0, 1, N - 2, N - 1]])).astype(np.uint32)
        dq = M.distances(kind, m.distinct, m.distinct[m.labels(qid)])
        by_exact, by_search = [], []
        for j, i in enumerate(qid):
            d = dq[j][lab]
            by_exact.append(rank(d, K + 1))
            by_search.append(M.search(layers, d, EF, K + 1))
        tid = torch.from_numpy(qid.view(np.int32)).cuda()
        for excl in (False, True):
            def cut(res, i):
                return M.excluding_self(res, int(i), K) if excl else res[:K]

            w = [cut(r, i) for r, i in zip(by_exact, qid)]
            assert_same(p.exact_search_batch(qid, K, by_id=True, exclude_self=excl), w, K, "exact by id %s" % excl)
            got = p.exact_search_batch_device(tid, K, by_id=True, exclude_self=excl)
            assert_same([_host(t) for t in got], w, K, "exact by id device %s" % excl)
            w = ([cut(r[0], i) for r, i in zip(by_search, qid)], [r[1] for r in by_search])
            assert_same(p.search_batch(qid, EF, K, with_stats=True, by_id=True, exclude_self=excl), w, K,
                        "search by id %s" % excl)
    finally:
        p.close()
        del tq, traw
        torch.cuda.empty_cache()
    print("\n%s dim %d: n = %d, rows %.1f GB, device memory in use at most %.1f GB, %.0f s"
          % (kind, dim, N, N * stride / GB, peak / GB, time.time() - t0))


def test_rerank_past_32_bit_offsets(oracle):
    import torch

    (k1, dim, _, _), (k2, _, _, boundaries) = RERANK
    s1, s2 = row_bytes(k1, dim), row_bytes(k2, dim)
    t0 = time.time()
    _need(torch, "the re-rank case", N * s1 + 2 * N * s2 + MARGIN)
    seed = 7
    m = Wide(k1, dim, N, boundaries, seed, stride=s2)
    p, layers, peak = _open(torch, oracle, m, seed)
    try:
        rows = m.device_rows(torch, torch.device("cuda", 0), kind=k2)
        p.set_rerank_elements_device(rows)
        torch.cuda.synchronize()
        peak = max(peak, _used(torch))
        del rows
        torch.cuda.empty_cache()
        assert p.device_bytes() >= N * (s1 + s2) + _layer_bytes(layers)
        el2 = m.elements(k2)
        d2_all = M.distances(k2, el2, M.element_rows(k2, m.raw_queries))
        lab = m.all_labels()
        ef, c = EF, 48
        want = []
        for q in range(NUM_QUERIES):
            want.append(M.rerank(layers, m.D[q][lab], d2_all[q][lab], ef, c, K))
        # stage 2 gathers the planted rows past 2^32 floats
        assert any(i >= first_id_at(boundaries[-1], s2) for w in want for i, _ in w[0])
        w = ([x[0] for x in want], [x[1] for x in want])
        assert_same(p.search_batch_rerank(m.raw_queries, c, ef, K, with_stats=True), w, K, "rerank")
        stats = torch.zeros((NUM_QUERIES, 4), dtype=torch.int64, device="cuda")
        got = p.search_batch_rerank_device(torch.from_numpy(m.raw_queries).cuda(), c, ef, K, stats=stats)
        assert_same([_host(t) for t in got] + [_host(stats)], w, K, "rerank device")
    finally:
        p.close()
        torch.cuda.empty_cache()
    print("\nre-rank %s %d + %s %d: n = %d, device memory in use at most %.1f GB, %.0f s"
          % (k1, dim, k2, dim, N, peak / GB, time.time() - t0))
