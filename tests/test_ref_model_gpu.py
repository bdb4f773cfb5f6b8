"""The GPU against the NumPy model of the reference (tests/helpers/ref_model.py), bit for bit: ids, distance bits,
counts, padding and stats columns 0..2, for every query call, at the widths the library accepts up to its limits
(f32 up to 16384, i8 up to 16384, embedding tables up to 4096) and on rows at the edges of the reference's
arithmetic.  Every f32 distance is also checked against float64 within a derived bound, so a model and a kernel that
agree and are both wrong still fail.  The model shares no code with the oracle, so these tests also catch a
misreading of the reference made in both the oracle and the kernels."""
import numpy as np
import pytest

import granne_b200
from helpers import ref_model as M
from helpers.data import edge_i8_rows, edge_raw_f32, index_from_lists, random_vectors
from helpers.index_image import assert_same_index
from helpers.model_checks import assert_same, assert_within_f64_bound

pytestmark = pytest.mark.gpu

F32_WIDTHS = [1, 33, 2101, 4096, 8192, 16384]
I8_WIDTHS = [1041, 4096, 16384]


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _image(rows):
    rows = np.ascontiguousarray(rows)
    return np.uint64(rows.shape[1]).tobytes() + rows.tobytes()


def _host(t):
    return t.cpu().numpy()


def graph(n, seed, degree=10, layer_lens=None):
    """Neighbour lists, top layer first: layers of n/40, n/6 and n elements, each node linked to `degree` random
    lower ids and its successor, so every node is reachable from node 0."""
    rng = np.random.default_rng(seed)
    lens = layer_lens or [max(2, n // 40), max(3, n // 6), n]
    layers = []
    for m in lens:
        layers.append([sorted((set(rng.integers(0, m, size=degree).tolist()) | {(i + 1) % m}) - {i})
                       for i in range(m)])
    return layers


def f32_rows(n, dim, seed):
    """Normalised rows at the edges (edge_raw_f32) plus, at the end, two ELEMENT rows that are not unit length."""
    rows = M.normalize_f32(edge_raw_f32(n, dim, seed))
    rows[n - 2] = rows[20] * np.float32(1.5)
    rows[n - 1] = rows[21] * np.float32(-0.75)
    return rows.astype(np.float32)


def f32_queries(dim, seed, rows):
    raw = np.concatenate([random_vectors(10, dim, seed), edge_raw_f32(12, dim, seed + 1)[[0, 1, 3, 4, 5, 6, 7]]])
    return raw, M.element_rows("angular", raw)


def i8_queries(dim, seed, rows):
    raw = random_vectors(10, dim, seed)
    return raw, np.concatenate([M.quantize(raw), rows[:8]])  # the second form: saturated, -128 and zero rows


def _case(kind, dim):
    n = 260 if dim <= 4096 else 160
    if kind == "angular":
        rows = f32_rows(n, dim, dim)
    else:
        rows = edge_i8_rows(n, dim, dim)
    layers = graph(n, dim)
    return rows, layers


def _open(oracle, kind, rows, layers):
    return granne_b200.Granne.from_bytes(index_from_lists(oracle, layers), kind, _image(rows))


# ---- every query call on dense indexes at every width -------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim", [("angular", d) for d in F32_WIDTHS] + [("angular_int", d) for d in I8_WIDTHS])
def test_query_calls_at_width(oracle, kind, dim):
    import torch

    rows, layers = _case(kind, dim)
    n = rows.shape[0]
    p = _open(oracle, kind, rows, layers)
    raw, qe = (f32_queries if kind == "angular" else i8_queries)(dim, dim + 7, rows)
    nq = qe.shape[0]
    d = M.distances(kind, rows, qe)  # [q, i]
    f32 = kind == "angular"

    # elements as stored
    ids = np.array([0, n - 1, 5, 3, 5], dtype=np.uint32)
    assert np.array_equal(p.get_elements(ids).view(np.uint8), rows[ids].view(np.uint8))
    assert np.array_equal(p.get_element(n - 2).view(np.uint8), rows[n - 2].view(np.uint8))
    got = _host(p.get_elements_device(torch.from_numpy(ids.astype(np.int32)).cuda()))
    assert np.array_equal(got.view(np.uint8), rows[ids].view(np.uint8))

    # exact k-NN, raw and element queries, k below, at and above n (k = 1024 > n)
    for k in (1, 10, 1024):
        want = [M.rank_prefix(d[q], n, k) for q in range(nq)]
        if f32:
            assert_same(p.exact_search_batch(raw, k), want[:raw.shape[0]], k, "exact raw k=%d" % k)
            assert_same(p.exact_search_batch(qe, k, already_element=True), want, k, "exact element k=%d" % k)
        else:
            assert_same(p.exact_search_batch(raw, k), want[:raw.shape[0]], k, "exact raw k=%d" % k)
            assert_same(p.exact_search_batch(qe, k), want, k, "exact element k=%d" % k)
    if f32:
        assert_within_f64_bound(rows, qe, p.exact_search_batch(qe, 1024, already_element=True))
    qarg = dict(already_element=True) if f32 else {}

    # graph search with its counters
    for ef, k in ((1, 1), (12, 10), (80, 40)):
        want = [M.search(layers, d[q], ef, k) for q in range(nq)]
        assert_same(p.search_batch(qe, ef, k, with_stats=True, **qarg), ([w[0] for w in want], [w[1] for w in want]),
                    k, "search ef=%d k=%d" % (ef, k))

    # filtered: S(q) ∩ A
    admit = (np.arange(n) % 3 != 1)
    want = [M.filtered(layers, d[q], 30, 20, admit) for q in range(nq)]
    assert_same(p.search_batch_filtered(qe, admit, max_search=30, num_elements=20, with_stats=True, **qarg),
                ([w[0] for w in want], [w[1] for w in want]), 20, "filtered")

    # within lists: duplicates count once; host and device forms
    rng = np.random.default_rng(dim)
    lists = [np.concatenate([rng.integers(0, n, size=int(rng.integers(0, 90))), [q % n, q % n]]).astype(np.uint32)
             for q in range(nq)]
    want = [M.within(d[q], lists[q], 16) for q in range(nq)]
    assert_same(p.exact_search_within(qe, lists, 16, **qarg), want, 16, "within")
    offs = np.zeros(nq + 1, dtype=np.int64)
    np.cumsum([len(c) for c in lists], out=offs[1:])
    tq = torch.from_numpy(qe).cuda()
    got = p.exact_search_within_device(tq, torch.from_numpy(offs).cuda(),
                                       torch.from_numpy(np.concatenate(lists).astype(np.int32)).cuda(), 16, **qarg)
    torch.cuda.synchronize()
    assert_same([_host(t) for t in got], want, 16, "within device")

    # by element id, with and without the element itself, on every call that takes ids
    qid = np.array([0, 1, 2, 3, 4, 5, 6, n - 2, n - 1, 100], dtype=np.uint32)
    dq = M.distances(kind, rows, rows[qid])  # by-id queries: the query of id i is row i
    for excl in (False, True):
        k = 8
        kk = k + 1 if excl else k

        def cut(res, i):
            return M.excluding_self(res, int(i), k) if excl else res

        want = [M.search(layers, dq[j], 20, kk) for j in range(len(qid))]
        assert_same(p.search_batch(qid, 20, k, with_stats=True, by_id=True, exclude_self=excl),
                    ([cut(w[0], i) for w, i in zip(want, qid)], [w[1] for w in want]), k, "search by id %s" % excl)
        want = [cut(M.rank_prefix(dq[j], n, kk), i) for j, i in enumerate(qid)]
        assert_same(p.exact_search_batch(qid, k, by_id=True, exclude_self=excl), want, k, "exact by id %s" % excl)
        want = [cut(M.within(dq[j], lists[j], kk), i) for j, i in enumerate(qid)]
        assert_same(p.exact_search_within(qid, lists[:len(qid)], k, by_id=True, exclude_self=excl), want, k,
                    "within by id %s" % excl)
        want = [M.filtered(layers, dq[j], 20, kk, admit) for j in range(len(qid))]
        assert_same(p.search_batch_filtered(qid, admit, max_search=20, num_elements=k, with_stats=True, by_id=True,
                                            exclude_self=excl),
                    ([cut(w[0], i) for w, i in zip(want, qid)], [w[1] for w in want]), k, "filtered by id %s" % excl)
    p.close()


# ---- Vector::from on the GPU, up to its limits ---------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 33, 2101, 8192, 12000])
def test_elements_from_raw_and_compute_distances(dim):
    raw = edge_raw_f32(24, dim, dim)
    for kind in ("angular", "angular_int"):
        img = granne_b200.elements_from_raw(kind, raw)
        want = M.element_rows(kind, raw)
        assert bytes(img) == _image(want), kind
    a, b = raw, np.roll(raw, 1, axis=0)
    b[:4] = a[:4]
    a[9] = a[9] * np.float32(-3)
    for kind in ("angular", "angular_int"):
        ea, eb = M.element_rows(kind, a), M.element_rows(kind, b)
        want = M.dist_f32(ea, eb) if kind == "angular" else M.dist_i8(ea, eb)
        assert np.array_equal(_bits(granne_b200.api.compute_distances(kind, a, b)), _bits(want)), kind


def test_elements_from_raw_at_its_width_limit():
    # host and device forms accept rows up to 12000 wide and reject 12001
    import torch

    raw = edge_raw_f32(12, 12000, 5)
    for kind in ("angular", "angular_int"):
        want = M.element_rows(kind, raw)
        assert bytes(granne_b200.elements_from_raw(kind, raw)) == _image(want), kind
        got = granne_b200.api.elements_from_raw_device(kind, torch.from_numpy(raw).cuda())
        assert np.array_equal(_host(got).view(np.uint8), want.view(np.uint8)), kind
        with pytest.raises(granne_b200.GranneError):
            granne_b200.elements_from_raw(kind, np.ones((2, 12001), dtype=np.float32))
        with pytest.raises(granne_b200.GranneError):
            granne_b200.api.elements_from_raw_device(kind, torch.ones((2, 12001), device="cuda"))


# ---- SumEmbeddings at the 4096 table limit -------------------------------------------------------------------------------
def _sum_case(oracle, dim=4096, n=150):
    table = random_vectors(300, dim, 11)
    table[7] = edge_raw_f32(12, dim, 2)[4]  # -0.0 and subnormal components
    rng = np.random.default_rng(1)
    terms = [[], [3], [3, 3, 3, 3], [7], list(range(300)), [299, 0, 299]]
    terms += [rng.integers(0, 300, size=int(rng.integers(1, 40))).tolist() for _ in range(n - len(terms))]
    el = oracle.Elements.sum_embeddings(table, terms)
    return table, terms, el.to_bytes(0), el.to_bytes(1)


def test_compute_embeddings_at_the_table_limit(oracle):
    table, terms, eb, mb = _sum_case(oracle)
    sums = np.stack([M.sum_embedding(table, t) for t in terms])
    for kind in ("angular", "angular_int"):
        img = granne_b200.api.compute_embeddings(kind, eb, mb)
        assert bytes(img) == _image(M.element_rows(kind, sums)), kind


def test_embeddings_search_and_rerank_at_the_table_limit(oracle):
    table, terms, eb, mb = _sum_case(oracle)
    n, dim = len(terms), table.shape[1]
    rows = M.sum_elements(table, terms)
    layers = graph(n, 5)
    ib = index_from_lists(oracle, layers)
    raw = random_vectors(12, dim, 3)
    raw[0] = M.sum_embedding(table, terms[4])
    d = M.distances("embeddings", rows, M.element_rows("embeddings", raw))
    p = granne_b200.Granne.from_bytes(ib, "embeddings", eb, mb)
    want = [M.search(layers, d[q], 30, 10) for q in range(len(raw))]
    assert_same(p.search_batch(raw, 30, 10, with_stats=True), ([w[0] for w in want], [w[1] for w in want]), 10,
                "embeddings search")
    want = [M.rank_prefix(d[q], n, 1024) for q in range(len(raw))]
    assert_same(p.exact_search_batch(raw, 1024), want, 1024, "embeddings exact")
    assert_within_f64_bound(rows, M.element_rows("embeddings", raw), p.exact_search_batch(raw, 1024))
    assert np.array_equal(p.get_elements(np.arange(n, dtype=np.uint32)).view(np.uint32), rows.view(np.uint32))
    p.close()

    # two-stage: an angular_int index over the quantised sums, re-ranked by the SumEmbeddings container
    q8 = M.quantize(np.stack([M.sum_embedding(table, t) for t in terms]))
    p = granne_b200.Granne.from_bytes(ib, "angular_int", _image(q8))
    p.set_rerank_embeddings(eb, mb)
    d8 = M.distances("angular_int", q8, M.quantize(raw))
    want = [M.rerank(layers, d8[q], d[q], 40, 25, 10) for q in range(len(raw))]
    assert_same(p.search_batch_rerank(raw, 25, 40, 10, with_stats=True), ([w[0] for w in want], [w[1] for w in want]),
                10, "rerank by SumEmbeddings")
    p.close()


@pytest.mark.parametrize("dim", [33, 4096, 16384])
def test_rerank_over_attached_f32_rows(oracle, dim):
    n = 200
    raw_rows = edge_raw_f32(n, dim, dim)
    f, q8 = M.normalize_f32(raw_rows), M.quantize(raw_rows)
    layers = graph(n, dim + 1)
    p = granne_b200.Granne.from_bytes(index_from_lists(oracle, layers), "angular_int", _image(q8))
    p.set_rerank_elements(_image(f))
    raw = random_vectors(10, dim, 4)
    d8, df = M.distances("angular_int", q8, M.quantize(raw)), M.distances("angular", f, M.normalize_f32(raw))
    for ef, c, k in ((20, 20, 10), (60, 50, 50)):
        want = [M.rerank(layers, d8[q], df[q], ef, c, k) for q in range(len(raw))]
        assert_same(p.search_batch_rerank(raw, c, ef, k, with_stats=True), ([w[0] for w in want], [w[1] for w in want]),
                    k, "rerank ef=%d c=%d" % (ef, c))
    p.close()


# ---- the knn graph, the multi handle, the pass ladder ----------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim", [("angular", 2101), ("angular_int", 1041)])
def test_knn_graph(oracle, kind, dim):
    rows, layers = _case(kind, dim)
    dself = M.distances(kind, rows, rows)
    p = _open(oracle, kind, rows, layers)
    for exact in (True, False):
        want = M.knn_graph(layers, dself, 24, 6, exact=exact)
        assert_same(p.knn_graph(24, 6, exact=exact), want, 6, "knn_graph exact=%s" % exact)
    p.close()


@pytest.mark.parametrize("kind,dim", [("angular", 4096), ("angular_int", 1041)])
def test_multi_handle_one_gpu(oracle, kind, dim):
    rows, layers = _case(kind, dim)
    n = rows.shape[0]
    raw, qe = (f32_queries if kind == "angular" else i8_queries)(dim, 3, rows)
    raw = raw[:10]
    q = M.element_rows(kind, raw)
    ib = index_from_lists(oracle, layers)
    m = granne_b200.MultiGranne.replicated(ib, kind, _image(rows), [0])
    d = M.distances(kind, rows, q)
    want = [M.search(layers, d[i], 20, 10)[0] for i in range(len(q))]
    assert_same(m.search_batch(raw, 20, 10), want, 10, "replicated search", np.uint64)
    want = [M.rank_prefix(d[i], n, 10) for i in range(len(q))]
    assert_same(m.exact_search_batch(raw, 10), want, 10, "replicated exact", np.uint64)
    m.close()

    cut = n // 2 + 3
    parts = [(rows[:cut], graph(cut, 1)), (rows[cut:], graph(n - cut, 2))]
    m = granne_b200.MultiGranne.partitioned([(index_from_lists(oracle, l), _image(r)) for r, l in parts], kind, [0, 0])
    bases = [m.shard_base(s) for s in range(2)]
    assert bases == [0, cut]
    ds = [M.distances(kind, r, q) for r, _ in parts]
    want = [M.merge([M.search(l, dd[i], 20, 10)[0] for (_, l), dd in zip(parts, ds)], bases, 10) for i in range(len(q))]
    assert_same(m.search_batch(raw, 20, 10), want, 10, "partitioned search", np.uint64)
    want = [M.merge([M.rank_prefix(dd[i], len(r), 10) for (r, _), dd in zip(parts, ds)], bases, 10)
            for i in range(len(q))]
    assert_same(m.exact_search_batch(raw, 10), want, 10, "partitioned exact", np.uint64)
    m.close()


def test_every_pass_of_the_ladder_against_the_model(oracle):
    # the mixed fast / retry case of test_parity_regimes_gpu (uniform rows on a fresh handle, max_search 20), then the
    # all-identical plateau that every query leaves to the slow pass
    n, dim = 10_000, 48
    el = oracle.Elements.angular(random_vectors(n, dim, seed=41))
    g = oracle.Granne.from_bytes(oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8).to_bytes(),
                                 el)
    layers = [[g.get_neighbors(i, layer) for i in range(g.layer_len(layer))] for layer in range(g.num_layers())]
    p = granne_b200.Granne.from_bytes(g.to_bytes(), "angular", el.to_bytes())
    raw = random_vectors(1536, dim, seed=42)
    d = M.distances("angular", el.rows(), M.normalize_f32(raw))
    got = p.search_batch(raw, 20, 10, with_stats=True)
    want = [M.search(layers, d[q], 20, 10) for q in range(len(raw))]
    assert_same(got, ([w[0] for w in want], [w[1] for w in want]), 10, "mixed ladder")
    flags = set(np.unique(got[3][:, 3]).tolist())
    p.close()

    n, dim = 400, 8
    rows = M.normalize_f32(np.tile(random_vectors(1, dim, seed=5), (n, 1)))
    layers = [[sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]]
    p = granne_b200.Granne.from_bytes(index_from_lists(oracle, layers), "angular", _image(rows))
    raw = random_vectors(256, dim, seed=6)
    d = M.distances("angular", rows, M.normalize_f32(raw))
    got = p.search_batch(raw, 20, 10, with_stats=True)
    want = [M.search(layers, d[q], 20, 10) for q in range(len(raw))]
    assert_same(got, ([w[0] for w in want], [w[1] for w in want]), 10, "plateau")
    flags |= set(np.unique(got[3][:, 3]).tolist())
    assert flags == {0, 1, 2}, flags
    p.close()


# ---- the builder at the widest accepted width ----------------------------------------------------------------------------
def test_builder_at_the_widest_width(oracle, monkeypatch):
    # insertions one at a time: the build the oracle makes with threads=1 (the default batched build has its own
    # oracle model, test_builder_batched_gpu)
    monkeypatch.setenv("GRANNE_B200_BUILD_MAX_BATCH", "1")
    dim = 16384
    rows = M.normalize_f32(edge_raw_f32(120, dim, 8))
    el = oracle.Elements.angular(rows, as_is=True)
    cfg = dict(num_neighbors=8, max_search=16, layer_multiplier=5.0)
    ref = oracle.GranneBuilder(el, **cfg).build(threads=1)
    b = granne_b200.GranneBuilder("angular", el.to_bytes(0), **cfg)
    b.build()
    image = b.index_bytes().tobytes()
    b.close()
    assert ref.num_layers() >= 2
    assert_same_index(oracle, image, ref, el, "angular dim=%d" % dim)
