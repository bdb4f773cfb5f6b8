"""Exact k nearest neighbours on the GPU (granne_b200_exact_search_batch*): ids, distance bits and counts equal the
CPU oracle's brute force (tests/helpers/composed_oracle.cpp) for every row layout, query format, k, nq and n edge; the
multi handle, the device variant and concurrent use; and, without the oracle, the approximate search with
max_search = n on a strongly connected graph."""
import threading

import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co
from helpers.data import random_vectors
from helpers.fixtures import ExactCase, assert_same, cxx_client, elements_from_raw, elements_image, sum_case
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

NOT_FINITE = -6


def _i8_rows(n, dim, seed):
    return elements_from_raw("angular_int", random_vectors(n, dim, seed))


@pytest.mark.parametrize("dim", [1, 31, 32, 33, 64, 96, 100, 128, 160, 192, 256, 300, 1000])
def test_f32_every_engine_layout(oracle, dim):
    rows = elements_from_raw("angular", random_vectors(700, dim, dim))
    c = ExactCase(oracle, "angular", rows)
    q = random_vectors(70, dim, dim + 1)
    assert_same(c.g.exact_search_batch(q, 10), c.o.exact_search(q, 10))
    qe = rows[[3, 500, 699]]  # ELEMENT queries: distance 0 to themselves
    assert_same(c.g.exact_search_batch(qe, 10, already_element=True), c.o.exact_search(qe, 10, already_element=True))


@pytest.mark.parametrize("dim", [1, 16, 100, 128, 512, 513, 1000])
def test_i8_every_width(oracle, dim):
    rows = elements_from_raw("angular_int", random_vectors(600, dim, dim))
    c = ExactCase(oracle, "angular_int", rows)
    q = random_vectors(70, dim, dim + 1)
    assert_same(c.g.exact_search_batch(q, 10), c.o.exact_search(q, 10))
    qe = rows[[0, 599]]
    assert_same(c.g.exact_search_batch(qe, 10), c.o.exact_search(qe, 10))


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("k", [0, 1, 10, 100, 1024, 1500])
def test_k(oracle, kind, k):
    rows = elements_from_raw(kind, random_vectors(1300, 64, 5))
    c = ExactCase(oracle, kind, rows)
    q = random_vectors(9, 64, 6)
    if k > granne_b200.api.EXACT_MAX_K:
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.exact_search_batch(q, k)
        assert e.value.code == -1
        return
    assert_same(c.g.exact_search_batch(q, k), c.o.exact_search(q, k))


@pytest.mark.parametrize("n", [1, 5, 127, 128, 129, 255, 257])
def test_n_around_the_row_tile_and_k_above_n(oracle, n):
    rows = elements_from_raw("angular", random_vectors(n, 128, n))
    c = ExactCase(oracle, "angular", rows)
    q = random_vectors(3, 128, 1)
    assert_same(c.g.exact_search_batch(q, 200), c.o.exact_search(q, 200))


@pytest.mark.parametrize("nq", [0, 1, 63, 64, 65, 1023, 1024, 1025])
def test_nq_around_the_query_block_and_chunk(oracle, nq):
    rows = elements_from_raw("angular_int", random_vectors(300, 100, 2))
    c = ExactCase(oracle, "angular_int", rows)
    q = random_vectors(nq, 100, 3)
    got = c.g.exact_search_batch(q, 10)
    if nq == 0:
        assert got[0].shape == (0, 10)
        return
    assert_same(got, c.o.exact_search(q, 10))


def test_slab_boundary(oracle):
    # 1024 queries: a slab holds 65536 rows, so this scan has a full slab and a short one
    n = 65536 + 129
    rows = elements_from_raw("angular", random_vectors(n, 32, 8))
    c = ExactCase(oracle, "angular", rows)
    q = random_vectors(1024, 32, 9)
    assert_same(c.g.exact_search_batch(q, 10), c.o.exact_search(q, 10))


def test_index_shorter_than_container_and_empty(oracle):
    rows = elements_from_raw("angular", random_vectors(500, 96, 4))
    q = random_vectors(20, 96, 5)
    for n in (0, 1, 300):
        c = ExactCase(oracle, "angular", rows, index_len=n)
        assert len(c.g) == n and c.g.num_elements() == 500
        got = c.g.exact_search_batch(q, 10)
        assert_same(got, c.o.exact_search(q, 10, index_len=n))
        assert (got[0][:, :min(n, 10)] < n).all() and (got[0][:, min(n, 10):] == 0xFFFFFFFF).all()


def test_ties(oracle):
    base = elements_from_raw("angular", random_vectors(40, 64, 1))
    rows = np.concatenate([base, base, np.zeros((30, 64), np.float32), base[:1].repeat(50, 0), base]).astype(np.float32)
    c = ExactCase(oracle, "angular", rows)
    q = np.concatenate([base[:5], np.zeros((1, 64), np.float32)])
    got = c.g.exact_search_batch(q, 300, already_element=True)
    assert_same(got, c.o.exact_search(q, 300, already_element=True))
    assert (got[1][5][:len(rows)] == 1.0).all()  # the all-zero query: every distance is exactly 1
    rows8 =np.concatenate([_i8_rows(40, 64, 2)] * 3 + [np.zeros((20, 64), np.int8)])
    c = ExactCase(oracle, "angular_int", rows8)
    q8 = np.concatenate([rows8[:4], np.zeros((1, 64), np.int8)])
    got = c.g.exact_search_batch(q8, 150)
    assert_same(got, c.o.exact_search(q8, 150))


def test_nan_element_and_query(oracle):
    rows = elements_from_raw("angular", random_vectors(200, 32, 1)).copy()
    rows[77, 3] = np.nan
    c = ExactCase(oracle, "angular", rows)
    with pytest.raises(co.NotFinite):
        c.o.exact_search(random_vectors(2, 32, 2), 10)
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.exact_search_batch(random_vectors(2, 32, 2), 10)
    assert e.value.code == NOT_FINITE
    c.g.exact_search_batch(random_vectors(2, 32, 2), 0)  # k == 0 reads no element
    rows[77, 3] = 0.0
    g = ExactCase(oracle, "angular", rows).g
    for kind, gg in (("angular", g), ("angular_int", ExactCase(oracle, "angular_int", _i8_rows(50, 32, 3)).g)):
        q = random_vectors(3, 32, 4)
        q[1, 0] = np.nan
        with pytest.raises(granne_b200.GranneError) as e:
            gg.exact_search_batch(q, 10)
        assert e.value.code == NOT_FINITE, kind


@pytest.mark.parametrize("dim,n", [(20, 700), (100, 700), (2048, 20000)])
def test_embeddings(oracle, dim, n):
    c = ExactCase(oracle, "embeddings", index_len=n - 3, images=sum_case(dim, n, dim, repeat_terms=True))
    q = random_vectors(5, dim, 1)
    assert_same(c.g.exact_search_batch(q, 10), c.o.exact_search(q, 10, index_len=c.n))


def test_device_variant_on_a_stream_and_concurrent_with_search(oracle):
    import torch

    el = oracle.Elements.angular(random_vectors(2000, 64, 3))
    gb = oracle.GranneBuilder(el, num_neighbors=10, max_search=50).build()
    g = granne_b200.Granne.from_bytes(gb.to_bytes(), "angular", el.to_bytes(0))
    q = random_vectors(300, 64, 4)
    want_exact = g.exact_search_batch(q, 10)
    want_search = g.search_batch(q, 50, 10)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    dq = torch.from_numpy(q).cuda()
    outs = []

    def run_exact():
        for _ in range(5):
            with torch.cuda.stream(s1):
                outs.append(("e", [t.cpu().numpy() for t in g.exact_search_batch_device(dq, 10, stream=s1.cuda_stream)]))

    def run_search():
        for _ in range(5):
            with torch.cuda.stream(s2):
                outs.append(("s", [t.cpu().numpy() for t in g.search_batch_device(dq, 50, 10, stream=s2.cuda_stream)]))

    ts = [threading.Thread(target=run_exact), threading.Thread(target=run_search)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    torch.cuda.synchronize()
    g.stream_status()
    assert len(outs) == 10
    for tag, (i, d, c) in outs:
        want = want_exact if tag == "e" else want_search
        assert_same((i.view(np.uint32), d, c.view(np.uint32)), want)


def test_multi_partitioned_and_replicated(oracle):
    sizes = [300, 1, 450]
    parts = [elements_from_raw("angular", random_vectors(s, 48, 10 + i)) for i, s in enumerate(sizes)]
    shards = [(co.single_layer_index(oracle, s), elements_image(p)) for s, p in zip(sizes, parts)]
    q = random_vectors(30, 48, 2)
    m = granne_b200.MultiGranne.partitioned(shards, "angular", [0])
    ids, d, cnt = m.exact_search_batch(q, 20)
    allrows = np.concatenate(parts)
    c = ExactCase(oracle, "angular", allrows)
    wi, wd, wc = c.o.exact_search(q, 20)
    assert np.array_equal(ids, wi.astype(np.uint64)) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(cnt, wc)
    r = granne_b200.MultiGranne.replicated(c.index_bytes, "angular", c.eb, [0, 0])
    ri, rd, rc = r.exact_search_batch(q, 20)
    gi, gd, gc = c.g.exact_search_batch(q, 20)
    assert np.array_equal(ri, gi.astype(np.uint64)) and np.array_equal(rd, gd) and np.array_equal(rc, gc)
    m.close()
    r.close()


def _strongly_connected(g):
    n = len(g)
    adj = [g.get_neighbors(i) for i in range(n)]
    radj = [[] for _ in range(n)]
    for i, ns in enumerate(adj):
        for j in ns:
            radj[j].append(i)

    def reach(a):
        seen, st = {0}, [0]
        while st:
            for j in a[st.pop()]:
                if j not in seen:
                    seen.add(j)
                    st.append(j)
        return len(seen) == n

    return reach(adj) and reach(radj)


@pytest.mark.parametrize("kind,dim,n", [("angular", 32, 1500), ("angular", 100, 800), ("angular_int", 100, 2000)])
def test_search_with_max_search_n_equals_exact(kind, dim, n):
    b = granne_b200.GranneBuilder(kind, granne_b200.elements_from_raw(kind, random_vectors(n, dim, n)).tobytes(),
                                  num_neighbors=20, max_search=100)
    b.build()
    g = b.get_index()
    assert _strongly_connected(g)
    q = random_vectors(40, dim, 7)
    assert_same(g.search_batch(q, n, 50), g.exact_search_batch(q, 50))


def test_at_size_f32_1m():
    import torch

    n, dim = 1_000_000, 128
    rows = torch.from_numpy(random_vectors(n, dim, 11)).cuda()
    el = granne_b200.elements_from_raw_device("angular", rows)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(co.single_layer_index(go, n), "angular", el)
    host = el.cpu().numpy()
    c = co.Container("angular", elements_image(host))
    q = random_vectors(64, dim, 12)
    assert_same(g.exact_search_batch(q, 10), c.exact_search(q, 10, threads=32))


def test_at_size_i8_10m():
    import torch

    n, dim = 10_000_000, 100
    rng = np.random.default_rng(5)
    host = rng.integers(-128, 128, (n, dim), dtype=np.int8)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(co.single_layer_index(go, n), "angular_int",
                                                torch.from_numpy(host).cuda())
    c = co.Container("angular_int", elements_image(host))
    q = random_vectors(32, dim, 13)
    assert_same(g.exact_search_batch(q, 10), c.exact_search(q, 10, threads=32))


def test_cxx_client(tmp_path, oracle):
    rows = elements_from_raw("angular", random_vectors(500, 64, 1))
    c = ExactCase(oracle, "angular", rows)
    idx = tmp_path / "index.bin"
    els = tmp_path / "elements.bin"
    idx.write_bytes(c.index_bytes)
    els.write_bytes(c.eb)
    out = cxx_client("cxx_exact_client.cpp", [idx, els], tmp_path)
    assert out.returncode == 0, out.stdout + out.stderr
    q = rows[:4]
    wi, wd, wc = c.o.exact_search(q, 5, already_element=True)
    lines = out.stdout.split()
    assert [int(x) for x in lines] == wi.ravel().tolist()
