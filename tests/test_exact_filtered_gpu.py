"""Exact filtered search on the GPU (granne_b200_exact_search_filtered_batch*).  Ids, distance bits and counts equal an
oracle composed from the CPU oracle's exact ranking (tests/helpers/composed_oracle.py: every element i < Index::len by
(dist_to_element, i)) cut to the ids each query's filter admits.  Also: every f32 engine layout, i8 widths, embeddings,
densities, k, n and nq edges, id windows, stray bits and containers larger than their index, the identities with
exact_search_batch, exact_search_within and filtered search, queries by id, NaN, the device variant under
concurrency and with bad query_filter entries, every handle source, both multi modes and a C++ client."""
import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co
from helpers.composed_oracle import pack
from helpers.data import clustered_vectors, random_sum_embeddings, random_vectors
from helpers.fixtures import ExactCase, assert_same, cxx_client, elements_from_raw, elements_image, sum_images
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

INVALID, NOT_FINITE = -1, -6
UNUSED = 0xFFFFFFFF


class Case(ExactCase):
    """An exact call's case; want() cuts the oracle's full exact ranking to the ids each query's filter admits."""

    def want(self, q, masks, k, query_filter=None, already_element=False, skip=None):
        """The first min(k, |A|) of the oracle's full exact ranking that the query's mask admits (masks: bool (F, m),
        m >= n; bits at or beyond n ignored); skip[q]: an id left out (exclude_self)."""
        masks = np.atleast_2d(masks)
        nq = len(q)
        ids = np.full((nq, k), UNUSED, np.uint32)
        dists = np.full((nq, k), np.inf, np.float32)
        counts = np.zeros(nq, np.uint32)
        if nq == 0 or self.n == 0:
            return ids, dists, counts
        ri, rd, rc = self.o.exact_search(q, self.n, index_len=self.n, already_element=already_element)
        for i in range(nq):
            f = 0 if query_filter is None else int(query_filter[i])
            r = ri[i, :rc[i]]
            keep = masks[f][r.astype(np.int64)]
            if skip is not None:
                keep &= r != skip[i]
            sel = np.nonzero(keep)[0][:k]
            ids[i, :sel.size] = r[sel]
            dists[i, :sel.size] = rd[i, sel]
            counts[i] = sel.size
        return ids, dists, counts


def _masks(n, densities, seed, width=None):
    """One bool mask of `width` (default n) ids per density: 0 admits nothing, "one" a single id, a fraction that share
    of the ids at random."""
    rng = np.random.default_rng(seed)
    out = np.zeros((len(densities), width or n), bool)
    for f, d in enumerate(densities):
        if d == "one":
            out[f, rng.integers(0, n)] = True
        elif d > 0:
            out[f, :n] = rng.random(n) < d
    return out


DENSITIES = [0, "one", 0.001, 0.01, 0.1, 0.5, 1.0]


def _check(c, q, masks, k, query_filter=None, already_element=False, what=""):
    got = c.g.exact_search_filtered(q, masks, query_filter, k, already_element=already_element)
    assert_same(got, c.want(q, masks, k, query_filter, already_element), what)
    return got


# DistF32<FULL> layouts (lane-permuted rows) and the natural layout of the generic engine
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 100, 128, 300, 1000])
def test_every_f32_engine_layout(oracle, dim):
    rows = elements_from_raw("angular", random_vectors(1500, dim, dim))
    c = Case(oracle, "angular", rows)
    masks = _masks(1500, DENSITIES, dim)
    q = random_vectors(len(DENSITIES), dim, dim + 1)
    _check(c, q, masks, 10, np.arange(len(DENSITIES)))
    _check(c, rows[[3, 700]], masks, 10, [4, 5], already_element=True)


@pytest.mark.parametrize("dim", [1, 16, 100, 512, 513, 1000])
def test_i8_every_width(oracle, dim):
    rows = elements_from_raw("angular_int", random_vectors(1500, dim, dim))
    c = Case(oracle, "angular_int", rows)
    masks = _masks(1500, DENSITIES, dim)
    q = random_vectors(len(DENSITIES), dim, dim + 1)
    _check(c, q, masks, 10, np.arange(len(DENSITIES)))
    _check(c, rows[[0, 1499]], masks, 10, [3, 6])  # int8 rows are elements


def test_sum_embeddings(oracle):
    # elements with 0 terms, more than 32 terms and repeated terms
    emb = random_vectors(64, 48, 1)
    terms = [[], list(range(40)), [5, 5, 5, 9], [63] * 70, [1, 2]] * 300
    el = oracle.Elements.sum_embeddings(emb, terms)
    c = Case(oracle, "embeddings", images=sum_images(el))
    masks = _masks(c.n, DENSITIES, 2)
    q = random_vectors(len(DENSITIES), 48, 3)
    _check(c, q, masks, 20, np.arange(len(DENSITIES)))
    el2 = random_sum_embeddings(oracle, 128, 50, 1200, 4)
    c2 = Case(oracle, "embeddings", images=sum_images(el2))
    _check(c2, random_vectors(4, 128, 5), _masks(1200, [0.01, 0.3], 6), 10, [0, 1, 1, 0])


@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings", "embeddings_4096"])
def test_all_admitting_filter_is_exact_search(oracle, kind):
    if kind == "embeddings":
        c = Case(oracle, kind, images=sum_images(random_sum_embeddings(oracle, 100, 300, 5000, 7)))
    elif kind == "embeddings_4096":  # 4096 materialised rows per list: two lists and a short one
        c = Case(oracle, "embeddings", images=sum_images(random_sum_embeddings(oracle, 4096, 8, 9000, 7)))
    else:
        c = Case(oracle, kind, elements_from_raw(kind, random_vectors(5000, 100, 7)))
    q = random_vectors(70, c.o.dim, 8)
    for k in (1, 10, 1024):
        got = c.g.exact_search_filtered(q, np.ones(c.n, bool), None, k)
        assert_same(got, c.g.exact_search_batch(q, k), "k=%d" % k)


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("k", [0, 1, 10, 1024])
def test_k(oracle, kind, k):
    rows = elements_from_raw(kind, random_vectors(3000, 64, 9))
    c = Case(oracle, kind, rows)
    masks = _masks(3000, [0.001, 0.01, 0.5, 1.0], 10)  # |A| below and above k
    q = random_vectors(8, 64, 11)
    _check(c, q, masks, k, [0, 1, 2, 3, 3, 2, 1, 0])


@pytest.mark.parametrize("n", [1, 31, 33, 127, 129])
def test_n_around_the_word_and_the_tile(oracle, n):
    rows = elements_from_raw("angular", random_vectors(n + 40, 32, n))
    c = Case(oracle, "angular", rows, index_len=n)  # ids [n, n + 40) are in the container but not the index
    masks = np.ones((3, n + 40), bool)
    masks[1, ::2] = False
    masks[2, :n] = False  # admits only ids >= n: nothing
    q = random_vectors(3, 32, n + 1)
    want = c.want(q, masks, 50, [0, 1, 2])
    got = c.g.exact_search_filtered(q, pack(masks), [0, 1, 2], 50)
    assert_same(got, want)
    assert (got[0][got[0] != UNUSED] < n).all() and got[2][2] == 0
    # stray bits past the container, and filter_words larger than needed
    words = np.concatenate([pack(masks), np.full((3, 5), 0xFFFFFFFF, np.uint32)], axis=1)
    assert_same(c.g.exact_search_filtered(q, words, [0, 1, 2], 50), want)
    assert_same(c.g.exact_search_filtered(q, pack(masks[:, :n]), [0, 1, 2], 50), want)


@pytest.mark.parametrize("nq", [0, 1, 64, 65, 1024, 1025])
def test_nq_and_several_filters(oracle, nq):
    rows = elements_from_raw("angular_int", random_vectors(300, 100, 12))
    c = Case(oracle, "angular_int", rows)
    masks = _masks(300, [0.01, 0.1, 0.5, 1.0, 0], 13)
    q = random_vectors(nq, 100, 14)
    rng = np.random.default_rng(nq)
    got = c.g.exact_search_filtered(q, masks, None, 10)
    assert got[0].shape == (nq, 10)
    if nq == 0:
        return
    assert_same(got, c.want(q, masks, 10))
    # per-query filters: several in one chunk, different mixes across chunks, and one filter per chunk
    _check(c, q, masks, 10, rng.integers(0, 5, size=nq))
    _check(c, q, masks, 10, np.repeat(np.arange(5), (nq + 4) // 5)[:nq])


def test_lists_longer_than_a_slab(oracle):
    # 1024 queries scan lists of at most 65536 ids (a slab): dense filters over 200 000 ids need several, each cut at a
    # word of the bitmap; sparse ones fit in one, whose ids straddle the slab boundaries
    n = 200_000
    rows = elements_from_raw("angular", clustered_vectors(n, 32, 15))
    c = Case(oracle, "angular", rows)
    masks = np.zeros((5, n), bool)
    for b in range(65536, n, 65536):
        masks[0, b - 3:b + 3] = True
    masks[1] = _masks(n, [0.01], 16)[0]
    masks[2, -1] = True
    masks[3] = _masks(n, [0.9], 17)[0]
    masks[4] = True
    q = clustered_vectors(1024, 32, 17)
    rng = np.random.default_rng(18)
    _check(c, q[:64], masks, 10, rng.integers(0, 5, size=64))
    for f in range(4):
        got = c.g.exact_search_filtered(q, masks, np.full(1024, f, np.uint32), 20)
        assert_same(tuple(x[:50] for x in got), c.want(q[:50], masks, 20, np.full(50, f)), "filter %d" % f)
    assert_same(c.g.exact_search_filtered(q, masks, np.full(1024, 1, np.uint32), 20),
                c.g.exact_search_within(q, [np.nonzero(masks[1])[0]] * 1024, 20))
    assert_same(c.g.exact_search_filtered(q, masks, np.full(1024, 4, np.uint32), 20), c.g.exact_search_batch(q, 20))
    # several filters per chunk: the union is listed, each query keeps its own filter's ids
    _check(c, q[:300], masks, 10, rng.integers(0, 5, size=300))


def test_bitmap_of_a_list_is_exact_search_within(oracle):
    rows = elements_from_raw("angular", random_vectors(6000, 96, 19))
    c = Case(oracle, "angular", rows)
    rng = np.random.default_rng(20)
    lists = [rng.permutation(6000)[:m].astype(np.uint32) for m in (0, 1, 7, 100, 3000, 6000)]
    masks = np.zeros((len(lists), 6000), bool)
    for f, lst in enumerate(lists):
        masks[f, lst] = True
    q = random_vectors(len(lists), 96, 21)
    assert_same(c.g.exact_search_filtered(q, masks, np.arange(len(lists)), 50), c.g.exact_search_within(q, lists, 50))


def test_filtered_search_agrees_with_exact(oracle):
    n, dim = 4000, 32
    raw = random_vectors(n, dim, 22)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw), num_neighbors=20,
                                  max_search=100)
    b.build()
    g = b.get_index()
    masks = _masks(n, [0.01, 0.1, 0.5, 1.0], 23)
    q = random_vectors(200, dim, 24)
    qf = np.arange(200) % 4
    ei, ed, ec = g.exact_search_filtered(q, masks, qf, 10)
    # any graph: rank by rank the filtered search's keys are >= the exact ones, and it finds no more
    fi, fd, fc = g.search_batch_filtered(q, masks, qf, 40, 10)
    assert (ec >= fc).all()
    for i in range(len(q)):
        for r in range(fc[i]):
            assert (fd[i, r], fi[i, r]) >= (ed[i, r], ei[i, r])
    # max_search >= n on a GPU-built graph whose every node is reachable: the search scores every element
    assert g.search_batch(q[:1], n, n)[2][0] == n
    assert_same(g.search_batch_filtered(q, masks, qf, n, 10), (ei, ed, ec))


def test_queries_by_id(oracle):
    rows = elements_from_raw("angular", random_vectors(2000, 64, 25))
    c = Case(oracle, "angular", rows)
    masks = _masks(2000, [0.05, 0.5], 26)
    ids = np.array([0, 5, 999, 1999, 1234, 77], np.uint32)
    masks[0, ids[:3]] = True   # the filter admits self for the first three queries
    masks[0, ids[3:]] = False  # and not for the others
    qf = np.zeros(len(ids), np.uint32)
    by_rows = c.g.exact_search_filtered(rows[ids], masks, qf, 10, already_element=True)
    assert_same(c.g.exact_search_filtered(ids, masks, qf, 10, by_id=True), by_rows)
    got = c.g.exact_search_filtered(ids, masks, qf, 10, exclude_self=True)
    assert_same(got, c.want(rows[ids], masks, 10, qf, already_element=True, skip=ids))
    import torch

    dev = torch.device("cuda", 0)
    td = torch.from_numpy(ids.view(np.int32)).to(dev)
    tw = torch.from_numpy(pack(masks).view(np.int32)).to(dev)
    dg = c.g.exact_search_filtered_device(td, tw, None, 10, exclude_self=True)
    c.g.stream_status()
    assert_same(tuple(t.cpu().numpy() for t in dg), got)


def test_nan(oracle):
    rows = elements_from_raw("angular", random_vectors(2000, 32, 27)).copy()
    rows[777] = np.nan
    c = Case(oracle, "angular", rows)
    clean = rows.copy()
    clean[777] = 0
    cc = Case(oracle, "angular", clean)
    q = random_vectors(3, 32, 28)
    masks = np.ones((3, 2000), bool)
    masks[0, 777] = False
    masks[1, :] = False
    masks[1, 5] = True
    masks[2, 700:800] = False
    # a NaN element no query's filter admits: OK and exact, also when a filter no query uses admits it
    assert_same(c.g.exact_search_filtered(q, masks, [0, 1, 2], 10), cc.want(q, masks, 10, [0, 1, 2]))
    both = np.concatenate([masks[:1], np.ones((1, 2000), bool)])
    assert_same(c.g.exact_search_filtered(q[:1], both, [0], 10), cc.want(q[:1], both, 10, [0]))
    # a filter that admits it
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.exact_search_filtered(q, both, [0, 1, 0], 10)
    assert e.value.code == NOT_FINITE
    # a NaN query: fails with a non-empty filter, not with an empty one (f32 and i8)
    qn = q.copy()
    qn[1, 4] = np.nan
    empty = np.zeros((2, 2000), bool)
    empty[1, 3] = True
    got = c.g.exact_search_filtered(qn[1:2], empty, [0], 10)
    assert got[2][0] == 0 and (got[0] == UNUSED).all()
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.exact_search_filtered(qn, empty, [0, 1, 0], 10)
    assert e.value.code == NOT_FINITE
    c8 = Case(oracle, "angular_int", elements_from_raw("angular_int", random_vectors(100, 32, 29)))
    e8 = np.zeros((2, 100), bool)
    e8[1, 3] = True
    got = c8.g.exact_search_filtered(qn[:2], e8, [0, 0], 10)
    assert (got[2] == 0).all()
    with pytest.raises(granne_b200.GranneError) as e:
        c8.g.exact_search_filtered(qn[:2], e8, [0, 1], 10)
    assert e.value.code == NOT_FINITE


def test_host_rejections(oracle):
    rows = elements_from_raw("angular", random_vectors(500, 32, 30))
    c = Case(oracle, "angular", rows, index_len=300)
    q = random_vectors(2, 32, 31)
    lib = granne_b200.load_library()
    launches = c.g.launch_count()
    words = np.ones((2, 10), np.uint32)
    ids, d = np.zeros((2, 10), np.uint32), np.zeros((2, 10), np.float32)
    rc = lib.granne_b200_exact_search_filtered_batch(c.g._h, q.ctypes.data, 2, 0, words.ctypes.data, 2, 9, None, 10,
                                                     ids.ctypes.data, d.ctypes.data, None)
    assert (rc, lib.granne_b200_last_error().decode()) == (INVALID, "filter_words is less than ceil(Index::len / 32)")
    qf = np.array([0, 2], np.uint32)
    rc = lib.granne_b200_exact_search_filtered_batch(c.g._h, q.ctypes.data, 2, 0, words.ctypes.data, 2, 10,
                                                     qf.ctypes.data, 10, ids.ctypes.data, d.ctypes.data, None)
    assert (rc, lib.granne_b200_last_error().decode()) == (INVALID, "a query_filter entry is >= num_filters")
    assert c.g.launch_count() == launches  # rejected before any device call


def test_device_variant(oracle):
    import torch

    rows = elements_from_raw("angular_int", random_vectors(20000, 100, 32))
    c = Case(oracle, "angular_int", rows, index_len=19000)
    dev = torch.device("cuda", 0)
    masks = _masks(19000, [0.01, 0.2, 1.0], 33, width=20000)
    masks[:, 19000:] = True  # ids past Index::len: ignored
    tw = torch.from_numpy(pack(masks).view(np.int32)).to(dev)
    # a bad query_filter entry: count 0 and padding for its query, the others answered, ERR_INVALID_ARGUMENT
    q = random_vectors(4, 100, 34)
    qf = np.array([0, 3, 2, 1], np.uint32)
    ri, rd, rc = c.g.exact_search_filtered_device(torch.from_numpy(q).to(dev), tw,
                                                  torch.from_numpy(qf.view(np.int32)).to(dev), 10)
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.stream_status()
    assert e.value.code == INVALID
    want = c.want(q, masks, 10, [0, 0, 2, 1])
    ri, rd, rc = ri.cpu().numpy().view(np.uint32), rd.cpu().numpy(), rc.cpu().numpy()
    assert rc[1] == 0 and (ri[1] == UNUSED).all() and np.isinf(rd[1]).all()
    for i in (0, 2, 3):
        assert np.array_equal(ri[i], want[0][i]) and rc[i] == want[2][i]
    # on a side stream, concurrent with graph searches on another stream
    qs = [random_vectors(300, 100, 40 + s) for s in range(4)]
    wants = [c.g.exact_search_filtered(x, pack(masks), np.arange(300) % 3, 20) for x in qs]
    assert_same(wants[0], c.want(qs[0], masks, 20, np.arange(300) % 3))
    s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    outs = []
    qf_d = torch.from_numpy((np.arange(300) % 3).astype(np.int32)).to(dev)
    for x in qs:
        qd = torch.from_numpy(x).to(dev)
        with torch.cuda.stream(s2):
            c.g.search_batch_device(qd, 50, 10, stream=s2)
        with torch.cuda.stream(s1):
            outs.append(c.g.exact_search_filtered_device(qd, tw, qf_d, 20, stream=s1))
    torch.cuda.synchronize(dev)
    c.g.stream_status()
    for got, want in zip(outs, wants):
        assert_same(tuple(t.cpu().numpy() for t in got), want)
    for s in (s1, s2):
        c.g.release_stream(s)


def test_handle_sources(oracle, tmp_path):
    import torch

    raw = random_vectors(3000, 128, 35)
    rows = elements_from_raw("angular", raw)
    c = Case(oracle, "angular", rows)
    masks = _masks(3000, [0.001, 0.05, 0.5], 36)
    q = random_vectors(6, 128, 37)
    qf = [0, 1, 2, 2, 1, 0]
    want = c.want(q, masks, 10, qf)
    assert_same(c.g.exact_search_filtered(q, masks, qf, 10), want)
    (tmp_path / "i").write_bytes(c.index_bytes)
    (tmp_path / "e").write_bytes(c.eb)
    f = granne_b200.Granne(str(tmp_path / "i"), "angular", str(tmp_path / "e"))
    assert_same(f.exact_search_filtered(q, masks, qf, 10), want)
    d = granne_b200.Granne.from_device_elements(c.index_bytes, "angular",
                                                torch.from_numpy(rows.copy()).to(torch.device("cuda", 0)))
    assert_same(d.exact_search_filtered(q, masks, qf, 10), want)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw[:2000]), num_neighbors=10,
                                  max_search=40)
    b.build()
    for v in raw[2000:]:
        b.append(v)
    b.build()
    snap = b.get_index()
    assert len(snap) == 3000
    assert_same(snap.exact_search_filtered(q, masks, qf, 10), want)


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_multi_handle(oracle, mode):
    dim = 64
    rows = elements_from_raw("angular", random_vectors(3000, dim, 38))
    full = Case(oracle, "angular", rows)
    masks = _masks(3000, [0.002, 0.05, 0.5, 1.0], 39)
    q = random_vectors(9, dim, 40)
    qf = np.arange(9) % 4
    want = full.want(q, masks, 10, qf)
    if mode == "replicated":
        m = granne_b200.MultiGranne.replicated(full.index_bytes, "angular", full.eb, [0, 0])
    else:
        cuts = [0, 1001, 2203, 3000]  # shard bases that are not multiples of 32
        shards = [(co.single_layer_index(oracle, b - a), elements_image(rows[a:b])) for a, b in zip(cuts, cuts[1:])]
        m = granne_b200.MultiGranne.partitioned(shards, "angular", [0, 0])
    gi, gd, gc = m.exact_search_filtered(q, masks, qf, 10)
    assert np.array_equal(gc, want[2])
    assert np.array_equal(gi, np.where(want[0] == UNUSED, np.iinfo(np.uint64).max, want[0].astype(np.uint64)))
    assert np.array_equal(gd.view(np.uint32), want[1].view(np.uint32))
    gids = np.array([5, 1500, 2999], np.uint64)
    xi, xd, xc = m.exact_search_filtered(gids, masks, [3, 3, 3], 10, exclude_self=True)
    wx = full.want(rows[gids.astype(np.int64)], masks, 10, [3, 3, 3], already_element=True,
                   skip=gids.astype(np.uint32))
    assert np.array_equal(xc, wx[2]) and np.array_equal(xi, wx[0].astype(np.uint64))
    with pytest.raises(granne_b200.GranneError) as e:
        m.exact_search_filtered(q[:2], masks, [0, 4], 10)
    assert e.value.code == INVALID
    m.close()


def test_at_size():
    import torch

    from oracle import granne_oracle as go

    dev = torch.device("cuda", 0)
    for kind, n, dim in (("angular", 1_000_000, 128), ("angular_int", 10_000_000, 100)):
        raw = torch.rand((n, dim), generator=torch.Generator(device=dev).manual_seed(41), device=dev) - 0.5
        g = granne_b200.Granne.from_device_elements(co.single_layer_index(go, n), kind,
                                                    granne_b200.elements_from_raw_device(kind, raw))
        del raw
        q = random_vectors(256, dim, 42)
        rng = np.random.default_rng(43)
        half = rng.random(n) < 0.5
        got = g.exact_search_filtered(q, half, None, 10)
        ai, ad, ac = g.exact_search_batch(q, 1024)
        wi = np.full((256, 10), UNUSED, np.uint32)
        wd = np.full((256, 10), np.inf, np.float32)
        for i in range(256):
            keep = np.nonzero(half[ai[i].astype(np.int64)])[0][:10]
            assert keep.size == 10  # 1024 entries at density 1/2 hold 10 admitted ones
            wi[i], wd[i] = ai[i, keep], ad[i, keep]
        assert_same(got, (wi, wd, np.full(256, 10, np.uint32)), kind + " 50%")
        sparse = rng.random(n) < 0.001
        got = g.exact_search_filtered(q[:16], sparse, None, 10)
        assert_same(got, g.exact_search_within(q[:16], [np.nonzero(sparse)[0].astype(np.uint32)] * 16, 10),
                    kind + " 0.1%")
        g.close()
        torch.cuda.empty_cache()


def test_cxx_client(oracle, tmp_path):
    rows = elements_from_raw("angular", random_vectors(2000, 64, 44))
    c = Case(oracle, "angular", rows)
    idx, el = tmp_path / "index.bin", tmp_path / "elements.bin"
    idx.write_bytes(c.index_bytes)
    el.write_bytes(c.eb)
    out = cxx_client("cxx_exact_filtered_client.cpp", [idx, el], tmp_path)
    assert out.returncode == 0, out.stdout + out.stderr
    odd = np.arange(2000) % 2 == 1
    wi, wd, wc = c.want(rows[7:8], odd, 5, already_element=True)
    lines = out.stdout.split()
    assert [int(x) for x in lines[0::2]] == wi[0, :wc[0]].tolist()
    assert [np.float32(x).view(np.uint32) for x in lines[1::2]] == wd[0, :wc[0]].view(np.uint32).tolist()
