"""Two-stage search re-ranked by a SumEmbeddings container (granne_b200_set_rerank_embeddings): an angular_int index
built over compute_embeddings rows gives C candidates, their exact sum-of-embeddings distances re-rank them.  Ids,
distance bits and counts equal a composed oracle built from the CPU oracle's own pieces: the angular_int rows of
compute_embeddings, the oracle's builder and angular_int search for the candidate set S,
SumEmbeddings::dist_to_element for each distance, and (distance, id) order for the first k.  Also: the identities
with the f32 re-rank and the "embeddings" handle, the edges of C and k, NaN tables, the rejections, concurrent use,
device memory, every handle source, the multi handle, string queries and a C++ client."""
import ctypes as C
import json
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers import embeddings_oracle as eo
from helpers.data import random_vectors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, FORMAT, NOT_FINITE = -1, -2, -6
UNUSED = 0xFFFFFFFF
COUNTS = [0, 1, 2, 9, 32, 33, 300]  # term counts that reach every DistSum branch (none, one, 32-term groups)


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _container(n, dim, num_rows, seed, counts=COUNTS):
    """A SumEmbeddings container: a table of num_rows rows and n term lists cycling through `counts`, with repeated
    terms."""
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((num_rows, dim)) * 2).astype(np.float32)
    elements = []
    for i in range(n):
        c = counts[i % len(counts)]
        ids = rng.integers(0, num_rows, c)
        if c > 3:
            ids[c // 2] = ids[0]
        elements.append([int(t) for t in ids])
    return table, elements


class Composed:
    """The two-stage result from oracle pieces, over a SumEmbeddings container and one index image built over its
    angular_int rows."""

    def __init__(self, go, table, elements, index_bytes=None, m=10, ef=40):
        self.table, self.elements = table, elements
        self.ei, self.ti = eo.elements_image(elements), eo.table_image(table)
        self.i8_image = eo.compute_embeddings("angular_int", self.ei, self.ti, threads=8).tobytes()
        self.i8 = go.Elements.from_bytes("angular_int", self.i8_image)
        if index_bytes is None:
            index_bytes = go.GranneBuilder(self.i8, num_neighbors=m, max_search=ef).build().to_bytes()
        self.index_bytes = index_bytes
        self.g = go.Granne.from_bytes(index_bytes, self.i8)
        self.sum = go.Elements.sum_embeddings(table, elements)

    def candidates(self, q, max_search, c):
        ids, _, cnt = self.g.search_batch(q, max_search, c)
        return [ids[i, :cnt[i]].copy() for i in range(len(q))]

    def rerank(self, q, max_search, c, k):
        nq = len(q)
        ids = np.full((nq, k), UNUSED, np.uint32)
        dists = np.full((nq, k), np.inf, np.float32)
        counts = np.zeros(nq, np.uint32)
        for i, s in enumerate(self.candidates(q, max_search, c)):
            d = np.array([self.sum.dist_to_element(int(j), q[i]) for j in s], np.float32)
            order = np.lexsort((s, d))[:k]
            ids[i, :order.size] = s[order]
            dists[i, :order.size] = d[order]
            counts[i] = order.size
        return ids, dists, counts

    def gpu(self, attach=True):
        g = granne_b200.Granne.from_bytes(self.index_bytes, "angular_int", self.i8_image)
        if attach:
            g.set_rerank_embeddings(self.ei, self.ti)
        return g


def _same(got, want):
    gi, gd, gc = got
    wi, wd, wc = want
    assert np.array_equal(np.asarray(gc).view(np.uint32), wc)
    assert np.array_equal(np.asarray(gi).view(np.uint32), wi)
    assert np.array_equal(np.asarray(gd).view(np.uint32), wd.view(np.uint32))


def _queries(nq, dim, seed):
    return (random_vectors(nq, dim, seed) * 3).astype(np.float32)


@pytest.mark.parametrize("dim", [1, 31, 32, 33, 100, 128, 129, 300, 1000, 4096])
def test_composed_oracle_and_identities(oracle, dim):
    n = 350
    c = Composed(oracle, *_container(n, dim, 400, dim))
    g = c.gpu()
    q = _queries(16, dim, dim + 1)
    got = g.search_batch_rerank(q, 30, max_search=50, num_elements=10)
    _same(got, c.rerank(q, 50, 30, 10))

    # the f32 two-stage search over compute_embeddings("angular") rows on a second handle: the same result
    f32_image = granne_b200.compute_embeddings("angular", c.ei, c.ti).tobytes()
    f = c.gpu(attach=False)
    f.set_rerank_elements(f32_image)
    _same(f.search_batch_rerank(q, 30, max_search=50, num_elements=10), got)

    # with k = C the id set is search_batch(q, max_search, C) on the same handle
    si, _, sc = g.search_batch(q, 50, 30)
    ai, ad, ac = g.search_batch_rerank(q, 30, max_search=50, num_elements=30)
    assert np.array_equal(sc, ac)
    for i in range(len(q)):
        assert set(si[i, :sc[i]].tolist()) == set(ai[i, :ac[i]].tolist())

    # the distances are exact_search_batch's on an "embeddings" handle over the same container, and the recall
    # identity holds against its exact top-k
    e = granne_b200.Granne.from_bytes(c.index_bytes, "embeddings", c.ei, c.ti)
    ei, ed, ec = e.exact_search_batch(q, n)
    for i in range(len(q)):
        by_id = dict(zip(ei[i, :ec[i]].tolist(), ed[i, :ec[i]].view(np.uint32).tolist()))
        assert [by_id[j] for j in ai[i, :ac[i]].tolist()] == ad[i, :ac[i]].view(np.uint32).tolist()
    ti, _, tc = e.exact_search_batch(q, 10)
    for i in range(len(q)):
        t = set(ti[i, :tc[i]].tolist())
        assert set(got[0][i, :got[2][i]].tolist()) & t == set(si[i, :sc[i]].tolist()) & t

    # every candidate that is an empty element has distance exactly 1.0; a wide candidate set reaches them
    wi, wd, wc = g.search_batch_rerank(q[:4], 1024, max_search=1024, num_elements=1024)
    _same((wi, wd, wc), c.rerank(q[:4], 1024, 1024, 1024))
    empty = [j for j, el in enumerate(c.elements) if not el]
    seen = 0
    for i in range(4):
        for j, d in zip(wi[i, :wc[i]].tolist(), wd[i, :wc[i]].tolist()):
            if j in empty:
                assert np.float32(d).view(np.uint32) == np.float32(1.0).view(np.uint32)
                seen += 1
    assert seen > 0


@pytest.mark.parametrize("max_search,cands,k", [(50, 1, 0), (50, 1, 1), (50, 10, 1), (50, 10, 10), (20, 100, 10),
                                                (200, 1024, 1), (1200, 1024, 1024), (50, 10, 0)])
def test_candidate_and_neighbour_edges(oracle, max_search, cands, k):
    c = Composed(oracle, *_container(1500, 48, 600, 5), m=16, ef=60)
    g = c.gpu()
    q = _queries(12, 48, 6)
    want = c.rerank(q, max_search, cands, k)
    _same(g.search_batch_rerank(q, cands, max_search=max_search, num_elements=k), want)
    assert (want[2] <= min(k, cands, max_search)).all()


def test_no_queries(oracle):
    c = Composed(oracle, *_container(200, 16, 100, 1))
    ids, dists, counts = c.gpu().search_batch_rerank(np.zeros((0, 16), np.float32), 10)
    assert ids.shape == (0, 10) and dists.shape == (0, 10) and counts.shape == (0,)


def test_nan_table_row_is_not_finite(oracle):
    import torch

    table, elements = _container(300, 32, 200, 10, counts=[1, 2, 3])
    c = Composed(oracle, table, elements)
    q = _queries(4, 32, 11)
    cands = c.candidates(q, 50, 10)
    only_late = sorted(set(cands[3].tolist()) - set(cands[0].tolist()) - set(cands[1].tolist()))
    early = set(cands[0].tolist()) | set(cands[1].tolist())
    # a table row used by a candidate of query 3 only
    row = next(t for j in only_late for t in elements[j]
               if not any(t in elements[e] for e in early))
    bad = table.copy()
    bad[row, 5] = np.nan
    g = c.gpu(attach=False)
    g.set_rerank_embeddings(c.ei, eo.table_image(bad))
    with pytest.raises(granne_b200.GranneError) as e:
        g.search_batch_rerank(q, 10, max_search=50)
    assert e.value.code == NOT_FINITE
    # the device variant on a non-default stream reports it through stream_status and keeps the current device
    prev = torch.cuda.current_device()
    s = torch.cuda.Stream()
    dq = torch.from_numpy(q).cuda()
    g.search_batch_rerank_device(dq, 10, max_search=50, stream=s)
    s.synchronize()
    assert torch.cuda.current_device() == prev
    with pytest.raises(granne_b200.GranneError) as e:
        g.stream_status()
    assert e.value.code == NOT_FINITE
    _same(g.search_batch_rerank(q[:2], 10, max_search=50), c.rerank(q[:2], 50, 10, 10))
    g.stream_status()


def _raw_attach(g, ei, ti):
    eb, mb = np.frombuffer(ei, np.uint8), np.frombuffer(ti, np.uint8)
    return api.load_library().granne_b200_set_rerank_embeddings(g._h, api._ptr(eb), eb.size, api._ptr(mb), mb.size)


def test_rejections(oracle):
    table, elements = _container(300, 32, 100, 7)
    c = Composed(oracle, table, elements)
    q = _queries(3, 32, 8)
    want = c.rerank(q, 50, 10, 10)
    bare = c.gpu(attach=False)
    cases = [
        (eo.elements_image(elements), eo.table_image(table[:, :31]), INVALID),  # width mismatch
        (eo.elements_image(elements[:299]), c.ti, INVALID),  # fewer elements than the index
        (c.ei[:-2], c.ti, FORMAT),  # truncated term lists
        (c.ei, c.ti[:-3], FORMAT),  # truncated table
        (c.ei[:5], c.ti, FORMAT),
        (eo.elements_image(elements[:-1] + [[100]]), c.ti, FORMAT),  # a term id past the table
    ]
    for ei, ti, code in cases:
        assert _raw_attach(bare, ei, ti) == code
        _same(bare.search_batch(q, 50, 10), c.g.search_batch(q, 50, 10))  # the handle still searches
    # a table wider than 4096 (with an index of that width)
    wide_t, wide_e = _container(40, 4100, 20, 9, counts=[1, 2])
    w = Composed(oracle, wide_t, wide_e)
    assert _raw_attach(w.gpu(attach=False), w.ei, w.ti) == INVALID
    # a correct attach still succeeds after every rejection
    bare.set_rerank_embeddings(c.ei, c.ti)
    _same(bare.search_batch_rerank(q, 10, max_search=50), want)
    # second attach of either kind, in both orders
    f32_image = granne_b200.compute_embeddings("angular", c.ei, c.ti).tobytes()
    assert _raw_attach(bare, c.ei, c.ti) == INVALID
    with pytest.raises(granne_b200.GranneError) as e:
        bare.set_rerank_elements(f32_image)
    assert e.value.code == INVALID
    rows_first = c.gpu(attach=False)
    rows_first.set_rerank_elements(f32_image)
    assert _raw_attach(rows_first, c.ei, c.ti) == INVALID
    _same(rows_first.search_batch_rerank(q, 10, max_search=50), want)
    _same(bare.search_batch_rerank(q, 10, max_search=50), want)
    # not an angular_int index
    e_handle = granne_b200.Granne.from_bytes(c.index_bytes, "embeddings", c.ei, c.ti)
    assert _raw_attach(e_handle, c.ei, c.ti) == INVALID
    e_handle.search_batch(q, 50, 10)


def test_concurrent_attaches_and_searches(oracle):
    c = Composed(oracle, *_container(2000, 64, 800, 12), m=12, ef=50)
    g = c.gpu(attach=False)
    codes = []
    ts = [threading.Thread(target=lambda: codes.append(_raw_attach(g, c.ei, c.ti))) for _ in range(6)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert sorted(codes) == [INVALID] * 5 + [0]
    q = _queries(200, 64, 13)
    want = c.rerank(q, 60, 30, 10)
    outs = []

    def host():
        for _ in range(3):
            outs.append(g.search_batch_rerank(q, 30, max_search=60))

    ts = [threading.Thread(target=host) for _ in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert len(outs) == 12
    for o in outs:
        _same(o, want)


def _sum_bytes(c):
    """The device bytes a staged SumEmbeddings container holds: the table (rows padded to 4 floats), the n + 1 u64
    offsets and the u32 term ids, each at least 16 bytes."""
    num_rows, dim = c.table.shape
    terms = sum(len(e) for e in c.elements)
    return (max(num_rows * ((dim + 3) & ~3) * 4, 16) + max((len(c.elements) + 1) * 8, 16) + max(terms * 4, 16))


def test_device_bytes(oracle):
    c = Composed(oracle, *_container(500, 30, 300, 14))
    g = c.gpu(attach=False)
    before = g.device_bytes()
    g.set_rerank_embeddings(c.ei, c.ti)
    assert g.device_bytes() == before + _sum_bytes(c)

    # a second attach of either kind changes nothing
    with pytest.raises(granne_b200.GranneError):
        g.set_rerank_embeddings(c.ei, c.ti)
    assert g.device_bytes() == before + _sum_bytes(c)

    # a multi attach whose last shard is rejected leaves every part without a container: a correct attach then
    # succeeds on every part
    table = c.table
    rng = np.random.default_rng(41)
    shards = [Composed(oracle, table, [[int(t) for t in rng.integers(0, 300, 1 + j % 5)] for j in range(s)])
              for s in (200, 150, 250)]
    m = granne_b200.MultiGranne.partitioned([(s.index_bytes, s.i8_image) for s in shards], "angular_int", [0])
    with pytest.raises(granne_b200.GranneError) as e:
        m.set_rerank_embeddings([shards[0].ei, shards[1].ei, eo.elements_image(shards[2].elements[:10])], c.ti)
    assert e.value.code == INVALID
    m.set_rerank_embeddings([s.ei for s in shards], c.ti)
    q = _queries(5, 30, 42)
    mi, md, mc = m.search_batch_rerank(q, 20, max_search=40, num_elements=5)
    assert (mc == 5).all()
    m.close()


def test_device_elements_handle(oracle):
    import torch

    c = Composed(oracle, *_container(800, 96, 500, 15))
    rows = granne_b200.compute_embeddings_device("angular_int", c.ei, c.ti)
    g = granne_b200.Granne.from_device_elements(c.index_bytes, "angular_int", rows)
    g.set_rerank_embeddings(c.ei, c.ti)
    q = _queries(30, 96, 16)
    want = c.rerank(q, 50, 40, 10)
    _same(g.search_batch_rerank(q, 40, max_search=50), want)
    got = g.search_batch_rerank_device(torch.from_numpy(q).cuda(), 40, max_search=50)
    torch.cuda.synchronize()
    g.stream_status()
    _same([t.cpu().numpy() for t in got], want)


@pytest.mark.parametrize("dim", [100, 300])
def test_gpu_built_index_and_get_index_handle(oracle, dim):
    table, elements = _container(1500, dim, 700, dim)
    i8_image = eo.compute_embeddings("angular_int", eo.elements_image(elements), eo.table_image(table)).tobytes()
    b = granne_b200.GranneBuilder("angular_int", i8_image, num_neighbors=12, max_search=40)
    b.build()
    c = Composed(oracle, table, elements, index_bytes=b.index_bytes().tobytes())
    q = _queries(40, dim, 3)
    want = c.rerank(q, 60, 40, 10)
    _same(c.gpu().search_batch_rerank(q, 40, max_search=60), want)
    snap = b.get_index()
    snap.set_rerank_embeddings(c.ei, c.ti)
    _same(snap.search_batch_rerank(q, 40, max_search=60), want)


def test_multi_replicated_and_partitioned(oracle):
    dim = 40
    table, elements = _container(700, dim, 300, 16)
    c = Composed(oracle, table, elements)
    q = _queries(25, dim, 17)
    want = c.rerank(q, 50, 30, 10)
    r = granne_b200.MultiGranne.replicated(c.index_bytes, "angular_int", c.i8_image, [0, 0])
    r.set_rerank_embeddings(c.ei, c.ti)
    ri, rd, rc = r.search_batch_rerank(q, 30, max_search=50)
    assert np.array_equal(ri, np.where(want[0] == UNUSED, ~np.uint64(0), want[0].astype(np.uint64)))
    assert np.array_equal(rd.view(np.uint32), want[1].view(np.uint32)) and np.array_equal(rc, want[2])
    r.close()

    # three shards over one shared table
    rng = np.random.default_rng(18)
    shard_elements = [[[int(t) for t in rng.integers(0, 300, 1 + j % 7)] for j in range(s)] for s in (300, 1, 450)]
    shards = [Composed(oracle, table, el) for el in shard_elements]
    m = granne_b200.MultiGranne.partitioned([(s.index_bytes, s.i8_image) for s in shards], "angular_int", [0])
    m.set_rerank_embeddings([s.ei for s in shards], c.ti)
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
        m.set_rerank_embeddings([s.ei for s in shards], c.ti)
    assert e.value.code == INVALID
    m.close()


def test_string_queries(oracle, tmp_path):
    dim = 50
    table, elements = _container(900, dim, 200, 19, counts=[1, 2, 3, 4])
    c = Composed(oracle, table, elements)
    words = ["w%d" % i for i in range(len(table))]
    path = tmp_path / "words.json"
    path.write_text("".join(json.dumps(w) + "\n" for w in words), encoding="utf-8")
    g = c.gpu(attach=False)
    g.set_rerank_embeddings(c.ei, c.ti, words_path=str(path))
    from granne_b200 import words as W

    for ids in ([3], [5, 17, 5], [0, 199, 42, 7]):
        got = g.search_rerank(" ".join(words[i] for i in ids), 40, max_search=60, num_elements=8)
        qi, qd, qc = g.search_batch_rerank(W.create_embedding(table, ids)[None, :], 40, max_search=60,
                                           num_elements=8)
        assert got == [(int(qi[0, j]), float(qd[0, j])) for j in range(int(qc[0]))]
        assert len(got) == 8
    with pytest.raises(ValueError):
        c.gpu().search_rerank("w1 w2", 10)


def test_cxx_client(tmp_path, oracle):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    c = Composed(oracle, *_container(500, 64, 300, 20))
    idx, i8, el, emb = (tmp_path / f for f in ("index.bin", "i8.bin", "el.bin", "emb.bin"))
    idx.write_bytes(c.index_bytes)
    i8.write_bytes(c.i8_image)
    el.write_bytes(c.ei)
    emb.write_bytes(c.ti)
    q = _queries(4, 64, 21)
    qf = tmp_path / "q.bin"
    qf.write_bytes(q.tobytes())
    exe = tmp_path / "client"
    libdir = os.path.dirname(granne_b200.library_path())
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", "cxx_rerank_sum_client.cpp"), "-o", str(exe),
                           "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe), str(idx), str(i8), str(el), str(emb), str(qf)], capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    wi, wd, wc = c.rerank(q, 50, 20, 5)
    assert (wc == 5).all()
    lines = out.stdout.split()
    assert [int(x) for x in lines[0::2]] == wi.ravel().tolist()
    assert [np.float32(x).view(np.uint32) for x in lines[1::2]] == wd.ravel().view(np.uint32).tolist()
