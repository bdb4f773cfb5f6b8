"""The diverse search on the GPU, exactly against a composed oracle: the oracle's search_batch(q, ef, ef), the element
itself dropped for QUERY_ID_EXCLUDING, then the oracle's select_neighbors(elements, candidates, k)
(src/index/mod.rs:849-883).  Ids, distance bits, counts and stats[:, :3] are compared on every distance engine and
layout, on edge rows (which pin that the kernel's pair distance d(c, s) has the reference's d(s, c) bits), and at the
shapes of the selection (unpruned short lists, C = k + 1, k = 1, lists of 31 to 1024, more than 32 kept).  The
standalone selection is checked over search_batch and exact_search_batch outputs, with its list errors on host and
device; and the call is tied to its meaning: the row an oracle build gives the element it inserts last."""
import numpy as np
import pytest

import granne_b200
from helpers.data import edge_i8_rows, edge_raw_f32, random_vectors, varied_sum_embeddings
from helpers.fixtures import ExactCase, assert_same, library  # noqa: F401  (autouse)
from oracle import granne_oracle as go

pytestmark = pytest.mark.gpu

UNUSED = 0xFFFFFFFF


class Case:
    """An oracle-built index over `el` (single-threaded build without reinsertion is not needed here: any graph both
    sides search identically serves), the GPU handle over its images and the oracle index."""

    def __init__(self, kind, el, num_neighbors=12, max_search=60):
        self.kind, self.el = kind, el
        self.og = go.GranneBuilder(el, num_neighbors=num_neighbors, max_search=max_search).build(threads=16)
        self.index_bytes = self.og.to_bytes()
        self.eb = el.to_bytes(0)
        self.mb = el.to_bytes(1) if kind == "embeddings" else None
        self.g = granne_b200.Granne.from_bytes(self.index_bytes, kind, self.eb, self.mb)

    def element_rows(self, ids):
        return np.stack([self.el.get(int(i)) for i in ids])


def oracle_select(el, ids, dists, counts, k, exclude=None):
    """select_neighbors(list_q, k) of each list (the first counts[q] entries), without exclude[q] when given."""
    nq = len(counts)
    oi = np.full((nq, k), UNUSED, np.uint32)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for q in range(nq):
        cands = [(int(ids[q, i]), float(dists[q, i])) for i in range(int(counts[q]))
                 if exclude is None or int(ids[q, i]) != int(exclude[q])]
        sel = go.select_neighbors(el, cands, k)
        oc[q] = len(sel)
        for j, (i, d) in enumerate(sel):
            oi[q, j], od[q, j] = i, d
    return oi, od, oc


def oracle_diverse(case, queries, ef, k, already_element=False, exclude=None):
    ids, d, c, st = case.og.search_batch(queries, ef, ef, already_element=already_element, threads=16,
                                         with_stats=True)
    return oracle_select(case.el, ids, d, c, k, exclude) + (st,)


def check_case(case, raw, ef_k=((60, 10), (11, 10), (40, 1), (20, 20), (8, 40))):
    """search_batch_diverse for raw queries, element queries and queries by id (with and without the element
    itself), against the oracle; and the standalone selection over search_batch(q, ef, ef) equal to it."""
    n = len(case.og)
    ids = np.arange(0, n, max(1, n // 24), dtype=np.uint32)[:24]
    rows = case.element_rows(ids)
    for ef, k in ef_k:
        what = "%s ef=%d k=%d" % (case.kind, ef, k)
        want = oracle_diverse(case, raw, ef, k)
        got = case.g.search_batch_diverse(raw, ef, k, with_stats=True)
        assert_same(got, want, what + " raw", stats=True)
        ci, cd, cc = case.g.search_batch(raw, ef, ef)
        assert_same(case.g.select_neighbors(ci, cd, cc, k), want[:3], what + " select over search_batch")
        want = oracle_diverse(case, rows, ef, k, already_element=True)
        assert_same(case.g.search_batch_diverse(rows, ef, k, already_element=True, with_stats=True), want,
                    what + " element", stats=True)
        assert_same(case.g.search_batch_diverse(ids, ef, k, by_id=True, with_stats=True), want, what + " by id",
                    stats=True)
        want = oracle_diverse(case, rows, ef, k, already_element=True, exclude=ids)
        assert_same(case.g.search_batch_diverse(ids, ef, k, exclude_self=True, with_stats=True), want,
                    what + " excluding", stats=True)


F32_DIMS = [32, 64, 96, 128, 192, 256, 160, 300, 2080]   # DistF32<1..8>, generic staged, generic direct


@pytest.mark.parametrize("dim", F32_DIMS)
def test_f32_engines(dim):
    raw = random_vectors(400, dim, dim)
    raw[50:58] = raw[49]  # a block of exact duplicates
    case = Case("angular", go.Elements.angular(raw))
    check_case(case, random_vectors(24, dim, dim + 1))


@pytest.mark.parametrize("dim", [100, 512, 513, 1041])
def test_i8_engine(dim):
    rows = edge_i8_rows(400, dim, dim)
    rows[50:58] = rows[49]
    case = Case("angular_int", go.Elements.angular_int(rows))
    check_case(case, random_vectors(24, dim, dim + 1))


@pytest.mark.parametrize("dim", [129, 300])
def test_embeddings_engine(dim):
    el = varied_sum_embeddings(go, dim, 80, 400, dim)
    case = Case("embeddings", el)
    check_case(case, random_vectors(24, dim, dim + 1), ef_k=((60, 10), (11, 10), (40, 1)))


@pytest.mark.parametrize("dim", [128, 2101])
def test_f32_edge_rows(dim):
    raw = edge_raw_f32(300, dim, 5)
    raw[40:48] = raw[39]
    case = Case("angular", go.Elements.angular(raw))
    n = len(case.og)
    ids = np.arange(0, 48, dtype=np.uint32)
    for ef, k in ((60, 10), (30, 3)):
        want = oracle_diverse(case, case.element_rows(ids), ef, k, already_element=True, exclude=ids)
        assert_same(case.g.search_batch_diverse(ids, ef, k, exclude_self=True, with_stats=True), want,
                    "edge rows excluding", stats=True)
        want = oracle_diverse(case, raw[:48], ef, k)
        assert_same(case.g.search_batch_diverse(raw[:48], ef, k, with_stats=True), want, "edge raw", stats=True)
    # every edge row as a candidate: exact lists over the whole container, selected on both sides
    C = min(n, 200)
    ei, ed, ec = case.g.exact_search_batch(case.element_rows(ids), C, already_element=True)
    assert_same(case.g.select_neighbors(ei, ed, ec, 20), oracle_select(case.el, ei, ed, ec, 20), "edge exact")


def test_i8_edge_rows():
    rows = edge_i8_rows(300, 256, 9)
    case = Case("angular_int", go.Elements.angular_int(rows))
    ids = np.arange(0, 16, dtype=np.uint32)
    for ef, k in ((60, 10), (30, 3)):
        want = oracle_diverse(case, rows[:16], ef, k, already_element=True, exclude=ids)
        assert_same(case.g.search_batch_diverse(ids, ef, k, exclude_self=True, with_stats=True), want,
                    "i8 edge excluding", stats=True)


@pytest.fixture(scope="module")
def wide_lists():
    """An angular 64-wide container of 1100 elements (the exact calls need no graph) and 8 queries near the all-ones
    direction: the nearest 64 elements are near-orthogonal rows close to the 64 axes, which keep one another (a list
    keeps more than a warp's width), and the others lean away from the queries."""
    rng = np.random.default_rng(11)
    raw = random_vectors(1100, 64, 11) - np.float32(0.3)
    raw[:64] = np.eye(64, dtype=np.float32) + np.float32(0.01) * rng.standard_normal((64, 64)).astype(np.float32)
    case = ExactCase(go, "angular", go.Elements.angular(raw).rows())
    q = np.float32(1) + np.float32(0.05) * rng.standard_normal((8, 64)).astype(np.float32)
    return case, q


@pytest.mark.parametrize("C", [31, 32, 33, 1023, 1024])
def test_select_over_exact_lists(wide_lists, C):
    case, q = wide_lists
    el = case.el
    oi, od, oc = case.o.exact_search(q, C)
    ei, ed, ec = case.g.exact_search_batch(q, C)
    assert_same((ei, ed, ec), (oi, od, oc), "exact lists")
    for k in (1, 10, 40, C - 1, C):
        want = oracle_select(el, oi, od, oc, k)
        got = case.g.select_neighbors(ei, ed, ec, k)
        assert_same(got, want, "C=%d k=%d" % (C, k))
        if C >= 1023 and k == 40:
            assert int(got[2].max()) > 32  # more than a warp's width kept


def test_select_device_and_streams(wide_lists):
    import torch

    case, q = wide_lists
    g = case.g
    qd = torch.from_numpy(q).cuda()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for s, C in ((s1, 1024), (s2, 200)):
        with torch.cuda.stream(s):
            ids, d, c = g.exact_search_batch_device(qd, C, stream=s)
            outs.append(g.select_neighbors_device(ids, d, c, 30, stream=s))
    torch.cuda.synchronize()
    g.stream_status()
    for (C, out) in zip((1024, 200), outs):
        want = g.select_neighbors(*g.exact_search_batch(q, C), 30)
        assert_same(tuple(t.cpu().numpy() for t in out), want, "device C=%d" % C)


def test_short_lists():
    # an index of one element: every query's only candidate, unpruned; empty lists give count 0
    raw = random_vectors(3, 16, 3)
    case = ExactCase(go, "angular", go.Elements.angular(raw).rows(), index_len=1)
    ids, d, c = case.g.search_batch_diverse(raw, 10, 5)
    assert list(c) == [1] * 3 and (ids[:, 0] == 0).all()
    assert (ids[:, 1:] == UNUSED).all() and np.isinf(d[:, 1:]).all()
    ids, d, c = case.g.select_neighbors(np.zeros((2, 4), np.uint32), np.zeros((2, 4), np.float32),
                                        np.zeros(2, np.uint32), 3)
    assert list(c) == [0, 0] and (ids == UNUSED).all()
    assert case.g.search_batch_diverse(raw[:0], 10, 5)[0].shape == (0, 5)


def test_max_search_cap(wide_lists):
    case, q = wide_lists
    with pytest.raises(granne_b200.GranneError) as e:
        case.g.search_batch_diverse(q, 1025, 10)
    assert "DIVERSE_MAX_CANDIDATES" in str(e.value)
    assert case.g.search_batch_diverse(q, 1024, 10)[2].max() <= 10


def test_list_errors_host_and_device(wide_lists):
    import torch

    case, q = wide_lists
    g = case.g
    ids, d, c = g.exact_search_batch(q, 50)
    bad_order, bad_id, bad_count = d.copy(), ids.copy(), c.copy()
    bad_order[1, 4] = bad_order[1, 3] - np.float32(0.5)
    bad_id[2, 5] = len(g)
    bad_count[3] = 51
    for args in ((ids, bad_order, c), (bad_id, d, c), (ids, d, bad_count)):
        with pytest.raises(granne_b200.GranneError) as e:
            g.select_neighbors(*args, 10)
        assert e.value.code == -1 and "candidate list" in str(e.value)
    # device: each bad list gets count 0 and padding, the others are answered, and the stream status reports it
    good = g.select_neighbors(ids, d, c, 10)
    cuda = lambda a: torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()  # noqa: E731
    # one fault per list: the order of list 1, an id of list 2, the count of list 3
    oi, od, oc = g.select_neighbors_device(cuda(bad_id), cuda(bad_order), cuda(bad_count), 10)
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status()
    assert e.value.code == -1
    oc, oi = oc.cpu().numpy().view(np.uint32), oi.cpu().numpy().view(np.uint32)
    assert list(oc[1:4]) == [0, 0, 0] and (oi[1:4] == UNUSED).all()
    keep = [0] + list(range(4, len(q)))
    assert np.array_equal(oi[keep], good[0][keep]) and np.array_equal(oc[keep], good[2][keep])


def test_nan_is_reported():
    raw = random_vectors(64, 32, 21)
    rows = go.Elements.angular(raw).rows()
    rows[7] = np.nan
    case = ExactCase(go, "angular", rows)
    ids = np.array([[1, 7, 2, 3]], np.uint32)
    d = np.array([[0.1, 0.2, 0.3, 0.4]], np.float32)
    with pytest.raises(granne_b200.GranneError) as e:
        case.g.select_neighbors(ids, d, np.array([4], np.uint32), 2)
    assert e.value.code == -6
    # the unpruned return computes no pair distance
    assert case.g.select_neighbors(ids, d, np.array([4], np.uint32), 4)[2][0] == 4


def test_handle_sources(tmp_path):
    import torch

    raw = random_vectors(500, 64, 31)
    el = go.Elements.angular(raw)
    case = Case("angular", el)
    q = random_vectors(16, 64, 32)
    want = case.g.search_batch_diverse(q, 50, 10, with_stats=True)
    (tmp_path / "index").write_bytes(case.index_bytes)
    (tmp_path / "el").write_bytes(case.eb)
    handles = [granne_b200.Granne(str(tmp_path / "index"), "angular", str(tmp_path / "el")),
               granne_b200.Granne.from_device_elements(case.index_bytes, "angular",
                                                       torch.from_numpy(el.rows()).cuda())]
    for h in handles:
        assert_same(h.search_batch_diverse(q, 50, 10, with_stats=True), want, "handle source", stats=True)
    b = granne_b200.GranneBuilder("angular", case.eb, num_neighbors=12, max_search=60)
    b.build()
    built = b.get_index()
    ob = go.Granne.from_bytes(built.index_bytes(), el)
    ids, d, c, st = ob.search_batch(q, 50, 50, threads=16, with_stats=True)
    assert_same(built.search_batch_diverse(q, 50, 10, with_stats=True), oracle_select(el, ids, d, c, 10) + (st,),
                "builder get_index", stats=True)


def test_the_row_an_insertion_gets():
    """For an oracle build without reinsertion, element n-1's bottom-layer row after build_partial(n) is the diverse
    search of that element on the image of n-1 elements, with the build's max_search and num_neighbors."""
    M, ef = 10, 40
    raw = random_vectors(700, 24, 41)
    el = go.Elements.angular(raw)
    b = go.GranneBuilder(el, num_neighbors=M, max_search=ef, reinsert_elements=False)
    for n in (300, 451, 700):
        before = b.build_partial(n - 1)
        after = b.build_partial(n)
        # premises: element n-1 joins the bottom layer only, and it is neither zero nor a dead duplicate
        L = after.num_layers()
        assert L == before.num_layers()
        assert [after.layer_len(i) for i in range(L - 1)] == [before.layer_len(i) for i in range(L - 1)]
        assert after.layer_len(L - 1) == n
        row = after.get_neighbors(n - 1, L - 1)
        assert len(row) > 0
        g = granne_b200.Granne.from_bytes(before.to_bytes(), "angular", el.to_bytes(0))
        ids, d, c = g.search_batch_diverse(el.get(n - 1)[None, :], ef, M, already_element=True)
        assert sorted(ids[0, :c[0]].tolist()) == sorted(row)
        assert sorted(g.search_batch_diverse(np.array([n - 1], np.uint32), ef, M, by_id=True)[0][0, :c[0]].tolist()) \
            == sorted(row)
        g.close()


def test_cxx_client(tmp_path):
    from helpers.fixtures import cxx_client

    raw = random_vectors(300, 32, 51)
    el = go.Elements.angular(raw)
    case = Case("angular", el)
    (tmp_path / "index").write_bytes(case.index_bytes)
    (tmp_path / "el").write_bytes(case.eb)
    q = random_vectors(4, 32, 52)
    (tmp_path / "q").write_bytes(q.tobytes())
    r = cxx_client("cxx_diverse_client.cpp", [tmp_path / "index", tmp_path / "el", tmp_path / "q", 4, 40, 8], tmp_path)
    assert r.returncode == 0, r.stderr
    want = case.g.search_batch_diverse(q, 40, 8)
    lines = r.stdout.rstrip("\n").split("\n")
    assert len(lines) == 4, r.stdout  # one line per query, empty for a query without results
    for qi, line in enumerate(lines):
        got = [int(v) for v in line.split()]
        assert got == want[0][qi, :want[2][qi]].tolist()


def _cuda(a):
    import torch

    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).cuda()


def _host(out, stats=None):
    return tuple(t.cpu().numpy() for t in out) + ((stats.cpu().numpy().view(np.uint64),) if stats is not None else ())


def test_device_call_on_streams():
    """search_batch_diverse_device with a stats tensor, raw, by-id and excluding queries on two concurrent streams,
    against the composed oracle; then one out-of-range id: its query gets count 0 and padding, the others are answered,
    and stream_status reports ERR_OUT_OF_RANGE."""
    import torch

    raw = random_vectors(500, 64, 61)
    case = Case("angular", go.Elements.angular(raw))
    q = random_vectors(32, 64, 62)
    ids = np.arange(3, 500, 16, dtype=np.uint32)[:32]
    rows = case.element_rows(ids)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    runs = []
    for s, queries, kw in ((s1, _cuda(q), {}), (s2, _cuda(ids), {"by_id": True}),
                           (s1, _cuda(ids), {"exclude_self": True}), (s2, _cuda(rows), {"already_element": True})):
        stats = torch.zeros((queries.shape[0], 4), dtype=torch.int64, device="cuda")
        with torch.cuda.stream(s):
            out = case.g.search_batch_diverse_device(queries, 60, 10, stats=stats, stream=s, **kw)
        runs.append((out, stats))
    torch.cuda.synchronize()
    case.g.stream_status()
    wants = (oracle_diverse(case, q, 60, 10), oracle_diverse(case, rows, 60, 10, already_element=True),
             oracle_diverse(case, rows, 60, 10, already_element=True, exclude=ids),
             oracle_diverse(case, rows, 60, 10, already_element=True))
    for what, (out, stats), want in zip(("raw", "by id", "excluding", "element"), runs, wants):
        assert_same(_host(out, stats), want, "device " + what, stats=True)
    bad = ids.copy()
    bad[5] = len(case.og.elements)
    for kw in ({"by_id": True}, {"exclude_self": True}):
        out = case.g.search_batch_diverse_device(_cuda(bad), 60, 10, **kw)
        with pytest.raises(granne_b200.GranneError) as e:
            case.g.stream_status()
        assert e.value.code == -8
        oi, od, oc = _host(out)
        good = case.g.search_batch_diverse(ids, 60, 10, **kw)
        assert oc[5] == 0 and (oi[5].view(np.uint32) == UNUSED).all() and np.isinf(od[5]).all()
        keep = [i for i in range(len(ids)) if i != 5]
        assert_same((oi[keep], od[keep], oc[keep]), tuple(x[keep] for x in good), "device bad id " + str(kw))


def test_nan_through_the_search():
    raw = random_vectors(64, 32, 71)
    rows = go.Elements.angular(raw).rows()
    rows[0] = np.nan
    case = ExactCase(go, "angular", rows)
    with pytest.raises(granne_b200.GranneError) as e:
        case.g.search_batch_diverse(raw[:4], 10, 5)
    assert e.value.code == -6
    case.g.search_batch_diverse_device(_cuda(raw[:4]), 10, 5)
    with pytest.raises(granne_b200.GranneError) as e:
        case.g.stream_status()
    assert e.value.code == -6


def _global(ids):
    ids = np.asarray(ids)
    return np.where(ids == UNUSED, np.uint64(2**64 - 1), ids.astype(np.uint64))


def _shards(kind, seed):
    """Two oracle-built shards of `kind` and the global container over both (SumEmbeddings: the shards share one
    table, and the global container holds their materialised rows as angular f32 rows)."""
    rng = np.random.default_rng(seed)
    if kind == "angular":
        raws = [random_vectors(260, 96, seed), random_vectors(240, 96, seed + 1)]
        els = [go.Elements.angular(r) for r in raws]
        glob = go.Elements.angular(np.concatenate(raws))
        mb = None
    elif kind == "angular_int":
        rws = [edge_i8_rows(260, 100, seed), edge_i8_rows(240, 100, seed + 1)]
        els = [go.Elements.angular_int(r) for r in rws]
        glob = go.Elements.angular_int(np.concatenate(rws))
        mb = None
    else:
        table = random_vectors(80, 129, seed)
        lists = [[rng.integers(0, 80, int(rng.integers(0, 40))).tolist() for _ in range(m)] for m in (260, 240)]
        els = [go.Elements.sum_embeddings(table, ls) for ls in lists]
        glob = go.Elements.angular(np.concatenate([np.stack([e.get(i) for i in range(len(e))]) for e in els]),
                                   as_is=True)
        mb = els[0].to_bytes(1)
    cases = [Case(kind, e) for e in els]
    return cases, glob, mb


def oracle_partitioned(cases, glob, queries, ef, k, already_element=False, exclude=None):
    """The shards' oracle search lists merged by (distance, global id), the query's own id dropped, then
    select_neighbors over the global container."""
    res, base = [], 0
    for c in cases:
        i, d, n = c.og.search_batch(queries, ef, ef, already_element=already_element, threads=16)
        res.append((i, d, n, base))
        base += len(c.el)
    nq = len(queries)
    mi = np.full((nq, ef), UNUSED, np.uint32)
    md = np.full((nq, ef), np.inf, np.float32)
    mc = np.zeros(nq, np.uint32)
    for q in range(nq):
        entries = sorted((float(d[q, j]), b + int(i[q, j])) for i, d, n, b in res for j in range(int(n[q])))[:ef]
        mc[q] = len(entries)
        for j, (dd, g) in enumerate(entries):
            mi[q, j], md[q, j] = g, dd
    oi, od, oc = oracle_select(glob, mi, md, mc, k, exclude)
    return _global(oi), od, oc


@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_multi_handle(kind):
    cases, glob, mb = _shards(kind, 81)
    q = random_vectors(16, cases[0].el.dim, 82)
    gids = np.array([0, 7, 259, 260, 261, 400, 499, 130], np.uint64)
    rows = np.stack([glob.get(int(g)) for g in gids])
    # REPLICATED: each device answers its slice as the single handle does
    c0 = cases[0]
    rep = granne_b200.MultiGranne.replicated(c0.index_bytes, kind, c0.eb, [0, 0], embeddings_bytes=mb)
    for ef, k in ((60, 10), (8, 20)):
        oi, od, oc = oracle_diverse(c0, q, ef, k)[:3]
        assert_same(rep.search_batch_diverse(q, ef, k), (_global(oi), od, oc), "replicated raw")
        lid = np.arange(0, 240, 17, dtype=np.uint64)
        oi, od, oc = oracle_diverse(c0, c0.element_rows(lid), ef, k, already_element=True, exclude=lid)[:3]
        assert_same(rep.search_batch_diverse(lid, ef, k, exclude_self=True), (_global(oi), od, oc),
                    "replicated excluding")
    rep.close()
    # RANGE_PARTITIONED: the shards' lists merged, then selected over the global container
    part = granne_b200.MultiGranne.partitioned([(c.index_bytes, c.eb) for c in cases], kind, [0, 0],
                                               embeddings_bytes=mb)
    for ef, k in ((60, 10), (30, 40), (100, 1)):
        want = oracle_partitioned(cases, glob, q, ef, k)
        assert_same(part.search_batch_diverse(q, ef, k), want, "partitioned raw ef=%d k=%d" % (ef, k))
        want = oracle_partitioned(cases, glob, rows, ef, k, already_element=True)
        assert_same(part.search_batch_diverse(gids, ef, k, by_id=True), want, "partitioned by id")
        want = oracle_partitioned(cases, glob, rows, ef, k, already_element=True, exclude=gids)
        assert_same(part.search_batch_diverse(gids, ef, k, exclude_self=True), want, "partitioned excluding")
    part.close()
