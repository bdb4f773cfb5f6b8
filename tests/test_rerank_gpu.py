"""Two-stage search on the GPU (granne_b200_search_rerank_batch*): an angular_int search gives C candidates, their
exact f32 angular distances re-rank them.  Ids, distance bits and counts equal a composed oracle built from the CPU
oracle's own pieces: its angular_int search gives the candidate set S, angular::Vectors::dist_to_element gives each
distance, and (distance, id) order picks the first k.  Also: every f32 engine layout, the edges of C and k, the
rejections, the stage-1 and recall identities, concurrent use, every handle source, the multi handle and a C++ client."""
import ctypes as C
import threading

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.data import clustered_vectors, random_vectors
from helpers.fixtures import assert_same, cxx_client, elements_image
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

INVALID, FORMAT, NOT_FINITE = -1, -2, -6
UNUSED = 0xFFFFFFFF


class Composed:
    """The two-stage result from oracle pieces, over raw f32 rows and one index image."""

    def __init__(self, go, index_bytes, raw):
        self.i8 = go.Elements.angular_int(raw)
        self.f32 = go.Elements.angular(raw)
        self.g = go.Granne.from_bytes(index_bytes, self.i8)
        self.index_bytes = index_bytes

    def candidates(self, q, max_search, c):
        ids, _, cnt = self.g.search_batch(q, max_search, c)
        return [ids[i, :cnt[i]].copy() for i in range(len(q))]

    def rerank(self, q, max_search, c, k):
        nq = len(q)
        ids = np.full((nq, k), UNUSED, np.uint32)
        dists = np.full((nq, k), np.inf, np.float32)
        counts = np.zeros(nq, np.uint32)
        for i, s in enumerate(self.candidates(q, max_search, c)):
            d = np.array([self.f32.dist_to_element(int(j), q[i]) for j in s], np.float32)
            order = np.lexsort((s, d))[:k]
            ids[i, :order.size] = s[order]
            dists[i, :order.size] = d[order]
            counts[i] = order.size
        return ids, dists, counts

    def gpu(self, with_f32=True):
        g = granne_b200.Granne.from_bytes(self.index_bytes, "angular_int", self.i8.to_bytes())
        if with_f32:
            g.set_rerank_elements(self.f32.to_bytes())
        return g


def _oracle_case(go, n, dim, seed, m=10, ef=40):
    raw = random_vectors(n, dim, seed)
    el = go.Elements.angular_int(raw)
    index = go.GranneBuilder(el, num_neighbors=m, max_search=ef).build().to_bytes()
    return Composed(go, index, raw)


# DistF32<FULL> for FULL = 0, 1, 2, 3, 4, 6, 8 (with and without a tail); DistF32Generic with staged rows (160, 300,
# 1000: at most 64 chunks) and with direct loads (2080, 2100: rows too wide for the staging tile)
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 64, 96, 100, 128, 160, 192, 256, 300, 1000, 2080, 2100])
def test_every_f32_engine_layout(oracle, dim):
    c = _oracle_case(oracle, 600, dim, dim)
    g = c.gpu()
    q = random_vectors(24, dim, dim + 7)
    got = g.search_batch_rerank(q, 30, max_search=50, num_elements=10)
    assert_same(got, c.rerank(q, 50, 30, 10))
    # stage 1 is search_batch(q, max_search, C) on the same handle: with k = C the result is that set, re-ordered
    si, _, sc = g.search_batch(q, 50, 30)
    ai, ad, ac = g.search_batch_rerank(q, 30, max_search=50, num_elements=30)
    assert np.array_equal(sc, ac)
    for i in range(len(q)):
        assert set(si[i, :sc[i]].tolist()) == set(ai[i, :ac[i]].tolist())
    # the distances are exact_search_batch's on an angular handle over the same rows
    f = granne_b200.Granne.from_bytes(c.index_bytes, "angular", c.f32.to_bytes())
    ei, ed, _ = f.exact_search_batch(q, 600)
    for i in range(len(q)):
        by_id = dict(zip(ei[i].tolist(), ed[i].view(np.uint32).tolist()))
        assert [by_id[j] for j in ai[i, :ac[i]].tolist()] == ad[i, :ac[i]].view(np.uint32).tolist()


@pytest.mark.parametrize("dim", [100, 128, 300])
def test_gpu_built_index_and_get_index_handle(oracle, dim):
    raw = random_vectors(1500, dim, dim)
    i8_image = oracle.Elements.angular_int(raw).to_bytes()
    b = granne_b200.GranneBuilder("angular_int", i8_image, num_neighbors=12, max_search=40)
    b.build()
    c = Composed(oracle, b.index_bytes().tobytes(), raw)
    q = random_vectors(40, dim, 3)
    want = c.rerank(q, 60, 40, 10)
    assert_same(c.gpu().search_batch_rerank(q, 40, max_search=60), want)
    snap = b.get_index()
    snap.set_rerank_elements(c.f32.to_bytes())
    assert_same(snap.search_batch_rerank(q, 40, max_search=60), want)


@pytest.mark.parametrize("max_search,cands,k", [(50, 1, 1), (50, 10, 10), (50, 50, 10), (20, 100, 10),
                                                (200, 1024, 10), (1200, 1024, 1024), (50, 10, 0)])
def test_candidate_and_neighbour_edges(oracle, max_search, cands, k):
    c = _oracle_case(oracle, 1500, 32, 5, m=16, ef=60)
    g = c.gpu()
    q = random_vectors(12, 32, 6)
    got = g.search_batch_rerank(q, cands, max_search=max_search, num_elements=k)
    want = c.rerank(q, max_search, cands, k)
    assert_same(got, want)
    assert (want[2] <= min(k, cands, max_search)).all()


def test_no_queries(oracle):
    c = _oracle_case(oracle, 200, 16, 1)
    ids, dists, counts = c.gpu().search_batch_rerank(np.zeros((0, 16), np.float32), 10)
    assert ids.shape == (0, 10) and dists.shape == (0, 10) and counts.shape == (0,)


def test_index_shorter_than_its_containers(oracle):
    raw = random_vectors(600, 64, 2)
    el = oracle.Elements.angular_int(raw[:400])
    index = oracle.GranneBuilder(el, num_neighbors=10, max_search=40).build().to_bytes()
    c = Composed(oracle, index, raw)
    q = random_vectors(20, 64, 3)
    g = c.gpu()
    assert len(g) == 400 and g.num_elements() == 600
    got = g.search_batch_rerank(q, 50, max_search=80)
    assert_same(got, c.rerank(q, 80, 50, 10))
    assert (got[0] < 400).all()
    # exactly Index::len f32 rows are enough, one fewer is not
    g2 = c.gpu(with_f32=False)
    g2.set_rerank_elements(elements_image(c.f32.rows()[:400]))
    assert_same(g2.search_batch_rerank(q, 50, max_search=80), got)
    g3 = c.gpu(with_f32=False)
    with pytest.raises(granne_b200.GranneError) as e:
        g3.set_rerank_elements(elements_image(c.f32.rows()[:399]))
    assert e.value.code == INVALID


def test_duplicate_rows_order_ties_by_id(oracle):
    base = random_vectors(50, 48, 4)
    raw = np.concatenate([base, base, base[:10].repeat(6, 0), base]).astype(np.float32)
    c = Composed(oracle, oracle.GranneBuilder(oracle.Elements.angular_int(raw), num_neighbors=12,
                                              max_search=60).build().to_bytes(), raw)
    q = np.concatenate([base[:8], random_vectors(4, 48, 5)])
    got = c.gpu().search_batch_rerank(q, 100, max_search=150, num_elements=40)
    assert_same(got, c.rerank(q, 150, 100, 40))
    d = got[1]
    assert any((d[i, 1:] == d[i, :-1]).any() for i in range(len(q)))  # ties occur, and were ordered by id


def _raw_rerank(g, q, fmt=api.QUERY_RAW_F32, max_search=50, cands=10, k=10):
    q = np.ascontiguousarray(q, dtype=np.float32)
    nq = q.shape[0]
    ids = np.empty((nq, k), np.uint32)
    dists = np.empty((nq, k), np.float32)
    counts = np.empty(nq, np.uint32)
    return api.load_library().granne_b200_search_rerank_batch(g._h, api._ptr(q), nq, fmt, max_search, cands, k,
                                                              api._ptr(ids), api._ptr(dists), api._ptr(counts), None)


def test_rejections(oracle):
    c = _oracle_case(oracle, 300, 32, 7)
    q = random_vectors(3, 32, 8)
    bare = c.gpu(with_f32=False)
    assert _raw_rerank(bare, q) == INVALID  # nothing attached
    for bad in (b"\x20\x00", elements_image(c.f32.rows())[:-3]):
        with pytest.raises(granne_b200.GranneError) as e:
            bare.set_rerank_elements(bad)
        assert e.value.code == FORMAT
    with pytest.raises(granne_b200.GranneError) as e:
        bare.set_rerank_elements(elements_image(random_vectors(300, 33, 1)))
    assert e.value.code == INVALID  # wrong width
    g = c.gpu()
    with pytest.raises(granne_b200.GranneError) as e:
        g.set_rerank_elements(c.f32.to_bytes())
    assert e.value.code == INVALID  # a second attach
    assert _raw_rerank(g, q, cands=1025) == INVALID
    assert _raw_rerank(g, q, cands=0, k=0) == INVALID
    assert _raw_rerank(g, q, cands=5, k=6) == INVALID
    assert _raw_rerank(g, q, fmt=api.QUERY_ELEMENT) == INVALID
    assert _raw_rerank(g, q, max_search=0) == INVALID
    assert _raw_rerank(g, q, cands=1024, k=10) == 0
    f = granne_b200.Granne.from_bytes(c.index_bytes, "angular", c.f32.to_bytes())
    with pytest.raises(granne_b200.GranneError) as e:
        f.set_rerank_elements(c.f32.to_bytes())
    assert e.value.code == INVALID  # not an angular_int index
    assert _raw_rerank(f, q) == INVALID


def test_device_attach_rejections(oracle):
    import torch

    c = _oracle_case(oracle, 300, 32, 9)
    g = c.gpu(with_f32=False)
    rows = torch.from_numpy(c.f32.rows()).cuda()
    lib = api.load_library()
    assert lib.granne_b200_set_rerank_elements_device(g._h, C.c_void_p(rows.data_ptr()), 300, 31) == INVALID
    assert lib.granne_b200_set_rerank_elements_device(g._h, C.c_void_p(rows.data_ptr()), 299, 32) == INVALID
    host = np.ascontiguousarray(c.f32.rows())
    assert lib.granne_b200_set_rerank_elements_device(g._h, api._ptr(host), 300, 32) == INVALID  # not device memory
    g.set_rerank_elements_device(rows)
    with pytest.raises(granne_b200.GranneError) as e:
        g.set_rerank_elements_device(rows)
    assert e.value.code == INVALID


def test_nan_row_is_not_finite(oracle):
    import torch

    c = _oracle_case(oracle, 300, 32, 10)
    q = random_vectors(4, 32, 11)
    cands = c.candidates(q, 50, 10)
    only_late = sorted(set(cands[3].tolist()) - set(cands[0].tolist()) - set(cands[1].tolist()))
    rows = c.f32.rows().copy()
    rows[only_late[0], 5] = np.nan
    g = c.gpu(with_f32=False)
    g.set_rerank_elements(elements_image(rows))
    with pytest.raises(granne_b200.GranneError) as e:
        g.search_batch_rerank(q, 10, max_search=50)
    assert e.value.code == NOT_FINITE
    dq = torch.from_numpy(q).cuda()
    g.search_batch_rerank_device(dq, 10, max_search=50)
    torch.cuda.synchronize()
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status()
    assert e.value.code == NOT_FINITE
    g.search_batch_rerank(q[:2], 10, max_search=50)  # queries whose candidates avoid the row are fine
    g.stream_status()


@pytest.mark.parametrize("cands", [10, 50])
def test_recall_identity(cands):
    n, dim = 20000, 64
    raw = clustered_vectors(n, dim, 3, n_centers=64)
    i8 = granne_b200.elements_from_raw("angular_int", raw).tobytes()
    f32 = granne_b200.elements_from_raw("angular", raw).tobytes()
    b = granne_b200.GranneBuilder("angular_int", i8, num_neighbors=10, max_search=30)
    b.build()
    index = b.index_bytes().tobytes()
    g = granne_b200.Granne.from_bytes(index, "angular_int", i8)
    g.set_rerank_elements(f32)
    f = granne_b200.Granne.from_bytes(index, "angular", f32)
    q = clustered_vectors(500, dim, 4, n_centers=64)
    ti, _, tc = f.exact_search_batch(q, 10)
    si, _, sc = g.search_batch(q, 40, cands)
    ii, _, ic = g.search_batch(q, 40, 10)
    ri, _, rc = g.search_batch_rerank(q, cands, max_search=40, num_elements=10)
    hit_r = hit_i = 0
    for i in range(len(q)):
        t = set(ti[i, :tc[i]].tolist())
        r = set(ri[i, :rc[i]].tolist())
        assert r & t == set(si[i, :sc[i]].tolist()) & t
        hit_r += len(r & t)
        hit_i += len(set(ii[i, :ic[i]].tolist()) & t)
    assert hit_r >= hit_i


def test_device_variant_on_two_streams_and_host_threads(oracle):
    import torch

    c = _oracle_case(oracle, 2000, 64, 12, m=12, ef=50)
    g = c.gpu()
    q = random_vectors(300, 64, 13)
    want = c.rerank(q, 60, 30, 10)
    assert_same(g.search_batch_rerank(q, 30, max_search=60), want)
    dq = torch.from_numpy(q).cuda()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []

    def device(s):
        for _ in range(4):
            with torch.cuda.stream(s):
                r = g.search_batch_rerank_device(dq, 30, max_search=60, stream=s)
                outs.append([t.cpu().numpy() for t in r])

    def host():
        for _ in range(4):
            outs.append(list(g.search_batch_rerank(q, 30, max_search=60)))

    ts = [threading.Thread(target=device, args=(s,)) for s in streams] + [threading.Thread(target=host)
                                                                          for _ in range(3)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    torch.cuda.synchronize()
    g.stream_status()
    assert len(outs) == 20
    for i, d, cnt in outs:
        assert_same((i.view(np.uint32), d, cnt.view(np.uint32)), want)


def test_device_elements_handle_and_device_attach(oracle):
    import torch

    c = _oracle_case(oracle, 800, 96, 14)
    i8 = torch.from_numpy(c.i8.rows()).cuda()
    f32 = torch.from_numpy(c.f32.rows()).cuda()
    g = granne_b200.Granne.from_device_elements(c.index_bytes, "angular_int", i8)
    before = g.device_bytes()
    g.set_rerank_elements_device(f32)
    assert g.device_bytes() >= before + 800 * 96 * 4
    q = random_vectors(30, 96, 15)
    want = c.rerank(q, 50, 40, 10)
    assert_same(g.search_batch_rerank(q, 40, max_search=50), want)
    stats = torch.zeros((30, api.STATS_PER_QUERY), dtype=torch.int64, device="cuda")
    got = g.search_batch_rerank_device(torch.from_numpy(q).cuda(), 40, max_search=50, stats=stats)
    torch.cuda.synchronize()
    g.stream_status()
    assert_same([t.cpu().numpy() for t in got], want)
    _, _, _, s1 = g.search_batch(q, 50, 40, with_stats=True)
    _, _, _, hs = g.search_batch_rerank(q, 40, max_search=50, with_stats=True)
    assert np.array_equal(stats.cpu().numpy().view(np.uint64)[:, :3], s1[:, :3])
    assert np.array_equal(hs[:, :3], s1[:, :3])


def test_multi_replicated_and_partitioned(oracle):
    dim = 40
    c = _oracle_case(oracle, 700, dim, 16)
    q = random_vectors(25, dim, 17)
    want = c.rerank(q, 50, 30, 10)
    r = granne_b200.MultiGranne.replicated(c.index_bytes, "angular_int", c.i8.to_bytes(), [0, 0])
    r.set_rerank_elements(c.f32.to_bytes())
    ri, rd, rc = r.search_batch_rerank(q, 30, max_search=50)
    assert np.array_equal(ri, np.where(want[0] == UNUSED, ~np.uint64(0), want[0].astype(np.uint64)))
    assert np.array_equal(rd.view(np.uint32), want[1].view(np.uint32)) and np.array_equal(rc, want[2])
    r.close()

    shards = [_oracle_case(oracle, s, dim, 20 + i) for i, s in enumerate([300, 1, 450])]
    m = granne_b200.MultiGranne.partitioned([(s.index_bytes, s.i8.to_bytes()) for s in shards], "angular_int", [0])
    m.set_rerank_elements([s.f32.to_bytes() for s in shards])
    k = 15
    mi, md, mc = m.search_batch_rerank(q, 30, max_search=50, num_elements=k)
    base = np.cumsum([0, 300, 1])
    parts = [s.rerank(q, 50, 30, k) for s in shards]
    for i in range(len(q)):
        entries = sorted((float(p[1][i, j]), int(base[s]) + int(p[0][i, j]))
                         for s, p in enumerate(parts) for j in range(p[2][i]))[:k]
        assert mc[i] == len(entries)
        assert mi[i, :mc[i]].tolist() == [e[1] for e in entries]
        assert md[i, :mc[i]].tolist() == [e[0] for e in entries]
        assert (mi[i, mc[i]:] == ~np.uint64(0)).all() and np.isinf(md[i, mc[i]:]).all()
    with pytest.raises(granne_b200.GranneError) as e:
        m.set_rerank_elements([s.f32.to_bytes() for s in shards])
    assert e.value.code == INVALID
    m.close()


def test_cxx_client(tmp_path, oracle):
    c = _oracle_case(oracle, 500, 64, 18)
    idx, i8, f32 = tmp_path / "index.bin", tmp_path / "i8.bin", tmp_path / "f32.bin"
    idx.write_bytes(c.index_bytes)
    i8.write_bytes(c.i8.to_bytes())
    f32.write_bytes(c.f32.to_bytes())
    q = random_vectors(4, 64, 19)
    qf = tmp_path / "q.bin"
    qf.write_bytes(q.tobytes())
    out = cxx_client("cxx_rerank_client.cpp", [idx, i8, f32, qf], tmp_path)
    assert out.returncode == 0, out.stdout + out.stderr
    wi, wd, wc = c.rerank(q, 50, 20, 5)
    lines = out.stdout.split()
    assert [int(x) for x in lines[0::2]] == wi.ravel().tolist()
    assert [np.float32(x).view(np.uint32) for x in lines[1::2]] == wd.ravel().view(np.uint32).tolist()
