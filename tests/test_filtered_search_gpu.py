"""Filtered search on the GPU (granne_b200_search_filtered_batch*).  Ids, distance bits, counts and stats[:, :3] equal an
oracle composed from the CPU oracle's own pieces (tests/helpers/composed_oracle.cpp: its descent, its bottom-layer
search recording the scored ids, the filter, dist_to_element, a sort by (distance, id)).  Also: every engine, every
list variant and the slow pass, many queries per warp through the pass ladder, per-query filters, stray bits beyond
len, ties and NaN, the identities with search_batch, the rejections, the device variant under concurrency, every
handle source, both multi modes and a C++ client."""
import threading

import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co
from helpers.data import build_fixture, index_from_lists, random_vectors
from helpers.fixtures import assert_same, cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

INVALID, NOT_FINITE = -1, -6
UNUSED = 0xFFFFFFFF
MAX_CTAS_PER_SM = 32


class Case:
    """A GPU handle and the filtered oracle over the same index and elements."""

    def __init__(self, index_bytes, kind, eb, mb=None, g=None):
        self.ib, self.kind, self.eb, self.mb = index_bytes, kind, eb, mb
        self.g = g if g is not None else granne_b200.Granne.from_bytes(index_bytes, kind, eb, mb)
        self.o = co.Filtered(index_bytes, kind, eb, mb)
        self.n = len(self.g)
        assert len(self.o) == self.n


def _case(oracle, kind, n, dim, seed, num_neighbors=16, max_search=40, **kw):
    _, _, ib, eb, mb = build_fixture(oracle, kind, n, dim, seed=seed, num_neighbors=num_neighbors,
                                     max_search=max_search, threads=8, **kw)
    return Case(ib, kind, eb, mb)


def _masks(n, densities, seed):
    """One bool mask per density: 0 admits nothing, "one" a single id, a fraction that share of the ids at random."""
    rng = np.random.default_rng(seed)
    out = np.zeros((len(densities), n), bool)
    for f, d in enumerate(densities):
        if d == "one":
            out[f, rng.integers(0, n)] = True
        elif d > 0:
            out[f] = rng.random(n) < d
    return out


DENSITIES = [0, "one", 0.01, 0.1, 0.5, 1.0]


def check(c, q, masks, ef, k, query_filter=None, already_element=False, what=""):
    words = co.pack(masks)
    want = c.o.search(q, words, ef, k, query_filter, already_element=already_element)
    got = c.g.search_batch_filtered(q, masks, query_filter, ef, k, already_element=already_element, with_stats=True)
    assert_same(got, want, what, stats=True)
    # every returned id is admitted by its query's filter
    qf = np.zeros(len(q), np.int64) if query_filter is None else np.asarray(query_filter)
    m = np.atleast_2d(masks)
    for i in range(len(q)):
        ids = got[0][i, :got[2][i]].astype(np.int64)
        assert m[qf[i], ids].all()
    return got


def _per_query(nq, f):
    return (np.arange(nq) % f).astype(np.uint32)


# ---- every engine layout ---------------------------------------------------------------------------------------------
# DistF32<FULL> for FULL = 0, 1, 2, 3, 4, 6, 8; DistF32Generic staged (160) and loading directly (2100)
@pytest.mark.parametrize("dim", [24, 32, 64, 96, 128, 192, 256, 160, 2100])
def test_every_f32_engine_layout(oracle, dim):
    c = _case(oracle, "angular", 1500, dim, seed=dim)
    q = random_vectors(36, dim, dim + 1)
    masks = _masks(c.n, DENSITIES, dim)
    check(c, q, masks, 40, 10, _per_query(36, len(DENSITIES)), what="angular dim=%d" % dim)
    e = c.g.get_element(5)[None, :].repeat(6, axis=0)
    check(c, e, masks, 40, 10, np.arange(6, dtype=np.uint32), already_element=True, what="element dim=%d" % dim)


@pytest.mark.parametrize("dim", [16, 100, 513])
def test_i8_widths(oracle, dim):
    c = _case(oracle, "angular_int", 1500, dim, seed=dim)
    q = random_vectors(24, dim, dim + 1)
    check(c, q, _masks(c.n, DENSITIES, dim), 40, 10, _per_query(24, len(DENSITIES)), what="i8 dim=%d" % dim)
    e = np.stack([c.g.get_element(i) for i in (0, 9, 1499)])
    check(c, e, _masks(c.n, [0.5], 1), 40, 10, what="i8 elements dim=%d" % dim)


def test_embeddings_with_empty_elements_and_repeated_terms(oracle):
    emb = random_vectors(64, 48, 1)
    terms = [[], list(range(40)), [5, 5, 5, 9], [63] * 70, [1, 2]] * 300
    el = oracle.Elements.sum_embeddings(emb, terms)
    g = oracle.GranneBuilder(el, num_neighbors=16, max_search=40).build(threads=8)
    c = Case(g.to_bytes(), "embeddings", el.to_bytes(0), el.to_bytes(1))
    q = random_vectors(24, 48, 2)
    check(c, q, _masks(c.n, DENSITIES, 3), 40, 10, _per_query(24, len(DENSITIES)), what="embeddings edges")
    d = _case(oracle, "embeddings", 2000, 50, seed=4)
    check(d, random_vectors(24, 50, 5), _masks(d.n, DENSITIES, 6), 40, 10, _per_query(24, len(DENSITIES)),
          what="embeddings")


# ---- every list variant, k and density -------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shared(oracle):
    return _case(oracle, "angular", 5000, 32, seed=61)


# max_search 40 / 150 / 400 / 900: fast lists of 3, 7, 15 and 31 rows; 1500: the generic list
@pytest.mark.parametrize("ef", [40, 150, 400, 900, 1500])
@pytest.mark.parametrize("k", [1, 10, 100, 1024])
def test_list_variants_k_and_densities(shared, ef, k):
    c = shared
    nq = 3 * len(DENSITIES)
    q = random_vectors(nq, 32, ef + k)
    check(c, q, _masks(c.n, DENSITIES, ef), ef, k, _per_query(nq, len(DENSITIES)), what="ef=%d k=%d" % (ef, k))


def test_slow_pass_with_ties_and_zero_distances(oracle):
    # every element is the same vector: one plateau of equal distances, wider than the fast and retry lists, so every
    # query runs on the slow pass; ties are broken by id, and an element query sits at distance 0 from everything
    n, dim = 400, 8
    raw = np.tile(random_vectors(1, dim, seed=5), (n, 1))
    el = oracle.Elements.angular(raw)
    nb = [sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]
    c = Case(index_from_lists(oracle, [nb]), "angular", el.to_bytes())
    q = np.concatenate([random_vectors(60, dim, seed=6), el.rows()[:12]])
    masks = _masks(n, DENSITIES, 7)
    got = check(c, q, masks, 20, 100, _per_query(72, len(DENSITIES)), what="plateau")
    assert (got[3][:, 3] == 2).all()


def test_many_queries_per_warp_through_the_pass_ladder(oracle):
    # uniform data on a fresh handle (test_parity_regimes_gpu.py): part of the batch overflows the fast pass and is
    # answered by the retry or slow pass, while each persistent warp serves several queries
    import torch

    n, dim = 20_000, 24
    el = oracle.Elements.angular(random_vectors(n, dim, seed=41))
    ib = oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8).to_bytes()
    c = Case(ib, "angular", el.to_bytes(0))
    nq = 4 * MAX_CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    q = random_vectors(nq, dim, seed=42)
    got = check(c, q, _masks(n, DENSITIES, 43), 40, 10, _per_query(nq, len(DENSITIES)), what="ladder")
    flags = got[3][:, 3]
    assert (flags == 0).any() and (flags >= 1).any(), "batch not mixed: %s" % np.bincount(flags.astype(np.int64))


def test_three_filters_per_query(shared):
    c = shared
    masks = _masks(c.n, [0.05, 0.3, 0.9], 8)
    qf = np.random.default_rng(9).integers(0, 3, size=200).astype(np.uint32)
    check(c, random_vectors(200, 32, 10), masks, 80, 20, qf, what="F=3")


def test_len_not_a_multiple_of_32_with_stray_bits(oracle):
    c = _case(oracle, "angular", 1000, 32, seed=12)
    assert c.n % 32 != 0
    masks = _masks(c.n, [0.2, 0.6], 13)
    words = co.pack(masks)
    stray = np.concatenate([words, np.full((2, 3), 0xFFFFFFFF, np.uint32)], axis=1)
    stray[:, c.n // 32] |= np.uint32(0xFFFFFFFF) << np.uint32(c.n % 32)
    q = random_vectors(40, 32, 14)
    qf = _per_query(40, 2)
    want = c.o.search(q, words, 40, 10, qf)
    assert_same(c.g.search_batch_filtered(q, stray, qf, 40, 10, with_stats=True), want, "stray bits", stats=True)
    assert_same(c.g.search_batch_filtered(q, masks, qf, 40, 10, with_stats=True), want, "bool masks", stats=True)


def test_nan_as_search_batch(shared):
    c = shared
    q = random_vectors(4, 32, 15)
    q[2, 3] = np.nan
    with pytest.raises(granne_b200.GranneError) as plain:
        c.g.search_batch(q, 40, 10)
    with pytest.raises(granne_b200.GranneError) as filt:
        c.g.search_batch_filtered(q, np.ones(c.n, bool), None, 40, 10)
    assert plain.value.code == filt.value.code == NOT_FINITE


# ---- identities without the oracle -----------------------------------------------------------------------------------
@pytest.mark.parametrize("ef", [40, 400, 1500])
def test_identities_with_search_batch(shared, ef):
    c = shared
    nq = 300
    q = random_vectors(nq, 32, 16 + ef)
    pi, pd, pc, ps = c.g.search_batch(q, ef, ef, with_stats=True)
    for f, masks in enumerate([_masks(c.n, [0.3], 17)[0], np.zeros(c.n, bool), np.ones(c.n, bool)]):
        gi, gd, gc, gs = c.g.search_batch_filtered(q, masks, None, ef, 10, with_stats=True)
        assert np.array_equal(gs[:, :3], ps[:, :3])  # the traversal does not move, whatever the filter
        for i in range(nq):
            assert masks[gi[i, :gc[i]].astype(np.int64)].all()
        if f == 1:
            assert (gc == 0).all() and (gi == UNUSED).all() and np.isinf(gd).all()
    # all admitted: search_batch(q, ef, k) wherever no tie at the ef-th place can tell them apart
    ki, kd, kc = c.g.search_batch(q, ef, 10)
    gi, gd, gc = c.g.search_batch_filtered(q, np.ones(c.n, bool), None, ef, 10)
    sure = (pc < ef) | (pd[:, 9].view(np.uint32) < pd[np.arange(nq), np.maximum(pc.astype(np.int64), 1) - 1]
                         .view(np.uint32))
    assert sure.mean() > 0.9
    assert np.array_equal(gi[sure], ki[sure]) and np.array_equal(gc[sure], kc[sure])
    assert np.array_equal(gd[sure].view(np.uint32), kd[sure].view(np.uint32))


# ---- rejections ------------------------------------------------------------------------------------------------------
def test_host_rejections(shared):
    c = shared
    q = random_vectors(3, 32, 18)
    lib = granne_b200.load_library()
    words = co.pack(np.ones(c.n, bool))
    ids = np.zeros((3, 10), np.uint32)
    d = np.zeros((3, 10), np.float32)

    def call(w, nwords, qf):
        rc = lib.granne_b200_search_filtered_batch(c.g._h, q.ctypes.data, 3, 0, 40, 10, w.ctypes.data, w.shape[0],
                                                   nwords, qf.ctypes.data if qf is not None else None, ids.ctypes.data,
                                                   d.ctypes.data, None, None)
        return rc, lib.granne_b200_last_error().decode()

    narrow = (INVALID, "filter_words is less than ceil(Index::len / 32)")
    assert call(words, words.shape[1] - 1, None) == narrow
    bad_qf = np.array([0, 1, 0], np.uint32)
    assert call(words, words.shape[1], bad_qf) == (INVALID, "a query_filter entry is >= num_filters")
    # the width rule comes first
    assert call(words, words.shape[1] - 1, bad_qf) == narrow
    two = np.concatenate([words, words])
    assert call(two, two.shape[1], bad_qf)[0] == 0
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.search_batch_filtered(q, np.ones(c.n, bool), [0, 0, 3], 40, 10)
    assert e.value.code == INVALID


def _device(c, q, masks, ef, k, qf=None, stream=None):
    import torch

    dev = torch.device("cuda", 0)
    tq = torch.from_numpy(q).to(dev)
    tw = torch.from_numpy(co.pack(masks).view(np.int32)).to(dev)
    tqf = None if qf is None else torch.from_numpy(np.asarray(qf, np.uint32).view(np.int32)).to(dev)
    stats = torch.empty((q.shape[0], 4), dtype=torch.int64, device=dev)
    ids, d, cnt = c.g.search_batch_filtered_device(tq, tw, tqf, ef, k, stats=stats, stream=stream)
    return ids, d, cnt, stats, (tq, tw, tqf)


def _host(out):
    ids, d, cnt, stats = (t.cpu().numpy() for t in out[:4])
    return ids.view(np.uint32), d, cnt.view(np.uint32), stats.view(np.uint64)


def test_device_bad_query_filter(shared):
    import torch

    c = shared
    q = random_vectors(6, 32, 19)
    masks = _masks(c.n, [0.5, 1.0], 20)
    qf = np.array([0, 1, 2, 1, 7, 0], np.uint32)
    out = _device(c, q, masks, 40, 10, qf)
    torch.cuda.synchronize()
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.stream_status()
    assert e.value.code == INVALID
    gi, gd, gc, gs = _host(out)
    bad = np.array([2, 4])
    assert (gc[bad] == 0).all() and (gi[bad] == UNUSED).all() and np.isinf(gd[bad]).all()
    good = np.array([0, 1, 3, 5])
    want = c.o.search(q[good], co.pack(masks), 40, 10, qf[good])
    assert_same((gi[good], gd[good], gc[good], gs[good]), want, "device, good queries", stats=True)
    c.g.stream_status()  # the error was reported once


def test_device_streams_and_threads(shared):
    import torch

    c = shared
    plans = [(2000, 40, 10, 0.5), (1500, 300, 100, 0.05), (3000, 10, 1, 1.0), (1000, 990, 1024, 0.2)]
    streams = [torch.cuda.Stream() for _ in plans]
    outs, wants = [], []
    for s, (nq, ef, k, dens) in enumerate(plans):
        q = random_vectors(nq, 32, 30 + s)
        masks = _masks(c.n, [dens, 0.01, 1.0], 40 + s)
        qf = _per_query(nq, 3)
        with torch.cuda.stream(streams[s]):
            outs.append(_device(c, q, masks, ef, k, qf, stream=streams[s]))
        wants.append(c.o.search(q, co.pack(masks), ef, k, qf))
    torch.cuda.synchronize()
    for s in range(len(plans)):
        assert_same(_host(outs[s]), wants[s], "stream %d" % s, stats=True)
    c.g.stream_status()
    for st in streams:
        c.g.release_stream(st)
    # host calls from several threads at once
    errors = []

    def worker(t):
        try:
            q = random_vectors(700, 32, 50 + t)
            masks = _masks(c.n, [0.1 * (t + 1), 1.0], 60 + t)
            check(c, q, masks, 60 + 20 * t, 10, _per_query(700, 2), what="thread %d" % t)
        except Exception as e:  # reported on the main thread
            errors.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


# ---- handle sources, multi handle, C++ -------------------------------------------------------------------------------
def test_handle_sources(oracle, tmp_path):
    import torch

    c = _case(oracle, "angular", 3000, 64, seed=31)
    q = random_vectors(24, 64, 33)
    masks = _masks(c.n, DENSITIES, 34)
    qf = _per_query(24, len(DENSITIES))
    want = c.o.search(q, co.pack(masks), 60, 10, qf)
    idx, el = tmp_path / "index.bin", tmp_path / "elements.bin"
    idx.write_bytes(c.ib)
    el.write_bytes(c.eb)
    f = granne_b200.Granne(str(idx), "angular", str(el))
    assert_same(f.search_batch_filtered(q, masks, qf, 60, 10, with_stats=True), want, "file images", stats=True)
    rows = np.frombuffer(bytes(c.eb[8:]), np.float32).reshape(-1, 64)
    d = granne_b200.Granne.from_device_elements(c.ib, "angular", torch.from_numpy(rows.copy()).to("cuda:0"))
    assert_same(d.search_batch_filtered(q, masks, qf, 60, 10, with_stats=True), want, "device elements", stats=True)
    # a builder's get_index: checked against the oracle over the builder's own index image
    raw = random_vectors(2500, 64, 35)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw), num_neighbors=12,
                                  max_search=40)
    b.build()
    snap = b.get_index()
    bc = Case(b.index_bytes(), "angular", granne_b200.elements_from_raw("angular", raw), g=snap)
    bm = _masks(bc.n, DENSITIES, 36)
    check(bc, q, bm, 60, 10, qf, what="builder get_index")


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_multi_handle(oracle, mode):
    dim = 32
    q = random_vectors(30, dim, 37)
    cuts = [0, 1000, 2500]  # shard 1's base 1000 is not a multiple of 32
    raw = random_vectors(2500, dim, 38)
    masks = _masks(2500, [0.02, 0.3, 1.0], 39)
    qf = _per_query(30, 3)
    words = co.pack(masks)
    k = 10
    if mode == "replicated":
        c = _case(oracle, "angular", 2500, dim, seed=38)
        m = granne_b200.MultiGranne.replicated(c.ib, "angular", c.eb, [0, 0])
        wi, wd, wc, _ = c.o.search(q, words, 50, k, qf)
        wi = np.where(wi == UNUSED, np.iinfo(np.uint64).max, wi.astype(np.uint64))
    else:
        shards, parts = [], []
        for a, b in zip(cuts, cuts[1:]):
            el = oracle.Elements.angular(raw[a:b])
            ib = oracle.GranneBuilder(el, num_neighbors=16, max_search=40).build(threads=8).to_bytes()
            shards.append((ib, el.to_bytes()))
            parts.append((a, co.Filtered(ib, "angular", el.to_bytes())))
        m = granne_b200.MultiGranne.partitioned(shards, "angular", [0, 0])
        assert m.shard_base(1) == 1000
        res = [(base, o.search(q, words, 50, k, qf, bit_base=base)) for base, o in parts]
        wi = np.full((30, k), np.iinfo(np.uint64).max, np.uint64)
        wd = np.full((30, k), np.inf, np.float32)
        wc = np.zeros(30, np.uint32)
        for i in range(30):
            keys = sorted((float(r[1][i, j]), base + int(r[0][i, j])) for base, r in res for j in range(int(r[2][i])))
            keys = keys[:k]
            wc[i] = len(keys)
            for j, (dd, gid) in enumerate(keys):
                wi[i, j], wd[i, j] = gid, dd
    gi, gd, gc = m.search_batch_filtered(q, masks, qf, 50, k)
    assert np.array_equal(gc, wc)
    assert np.array_equal(gi, wi)
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
    for i in range(30):
        assert masks[qf[i], gi[i, :gc[i]].astype(np.int64)].all()
    lib = granne_b200.load_library()
    ids, d = np.zeros((1, k), np.uint64), np.zeros((1, k), np.float32)
    rc = lib.granne_b200_multi_search_filtered_batch(m._h, q.ctypes.data, 1, 0, 50, k, words.ctypes.data,
                                                     words.shape[0], words.shape[1] - 1, None, ids.ctypes.data,
                                                     d.ctypes.data, None)
    assert (rc, lib.granne_b200_last_error().decode()) == (INVALID, "filter_words is less than ceil(Index::len / 32)")
    with pytest.raises(granne_b200.GranneError) as e:
        m.search_batch_filtered(q[:2], masks, [0, 3], 50, k)
    assert e.value.code == INVALID
    m.close()


def test_cxx_client(oracle, tmp_path):
    c = _case(oracle, "angular", 2000, 64, seed=44)
    idx, el = tmp_path / "index.bin", tmp_path / "elements.bin"
    idx.write_bytes(c.ib)
    el.write_bytes(c.eb)
    out = cxx_client("cxx_filtered_client.cpp", [idx, el], tmp_path)
    assert out.returncode == 0, out.stdout + out.stderr
    odd = (np.arange(c.n) % 2 == 1)
    wi, wd, wc, _ = c.o.search(c.g.get_element(7)[None, :], co.pack(odd), 40, 5, already_element=True)
    lines = out.stdout.split()
    assert [int(x) for x in lines[0::2]] == wi[0, :wc[0]].tolist()
    assert [np.float32(x).view(np.uint32) for x in lines[1::2]] == wd[0, :wc[0]].view(np.uint32).tolist()
