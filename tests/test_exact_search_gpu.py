"""Exact k nearest neighbours on the GPU (granne_b200_exact_search_batch*): ids, distance bits and counts equal the
CPU oracle's brute force (tests/helpers/exact_oracle.cpp) for every row layout, query format, k, nq and n edge; the
multi handle, the device variant and concurrent use; and, without the oracle, the approximate search with
max_search = n on a strongly connected graph."""
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

import granne_b200
from helpers import embeddings_oracle as eo
from helpers import exact_oracle as xo
from helpers.data import random_vectors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_FINITE = -6


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _same(got, want):
    gi, gd, gc = got
    wi, wd, wc = want
    assert np.array_equal(np.asarray(gc), wc)
    assert np.array_equal(np.asarray(gi).view(np.uint32), wi)
    assert np.array_equal(np.asarray(gd).view(np.uint32), wd.view(np.uint32))


def _dense(go, kind, rows, index_len=None):
    """(GPU handle, oracle container) over the given element rows; the index covers index_len of them."""
    rows = np.ascontiguousarray(rows)
    eb = np.uint64(rows.shape[1]).tobytes() + rows.tobytes()
    n = rows.shape[0] if index_len is None else index_len
    g = granne_b200.Granne.from_bytes(xo.single_layer_index(go, n), kind, eb)
    return g, xo.Container(kind, eb)


def _i8_rows(n, dim, seed):
    return elements_from_raw_rows("angular_int", random_vectors(n, dim, seed))


def _rows(image, dt):
    dim = int(np.frombuffer(bytes(image[:8]), dtype=np.uint64)[0])
    return np.frombuffer(bytes(image[8:]), dtype=dt).reshape(-1, dim)


def elements_from_raw_rows(kind, raw):
    return _rows(granne_b200.elements_from_raw(kind, raw), np.float32 if kind == "angular" else np.int8)


@pytest.mark.parametrize("dim", [1, 31, 32, 33, 64, 96, 100, 128, 160, 192, 256, 300, 1000])
def test_f32_every_engine_layout(oracle, dim):
    rows = elements_from_raw_rows("angular", random_vectors(700, dim, dim))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(70, dim, dim + 1)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10))
    qe = rows[[3, 500, 699]]  # ELEMENT queries: distance 0 to themselves
    _same(g.exact_search_batch(qe, 10, already_element=True), c.exact_search(qe, 10, already_element=True))


@pytest.mark.parametrize("dim", [1, 16, 100, 128, 512, 513, 1000])
def test_i8_every_width(oracle, dim):
    rows = elements_from_raw_rows("angular_int", random_vectors(600, dim, dim))
    g, c = _dense(oracle, "angular_int", rows)
    q = random_vectors(70, dim, dim + 1)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10))
    qe = rows[[0, 599]]
    _same(g.exact_search_batch(qe, 10), c.exact_search(qe, 10))


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("k", [0, 1, 10, 100, 1024, 1500])
def test_k(oracle, kind, k):
    rows = elements_from_raw_rows(kind, random_vectors(1300, 64, 5))
    g, c = _dense(oracle, kind, rows)
    q = random_vectors(9, 64, 6)
    if k > granne_b200.api.EXACT_MAX_K:
        with pytest.raises(granne_b200.GranneError) as e:
            g.exact_search_batch(q, k)
        assert e.value.code == -1
        return
    _same(g.exact_search_batch(q, k), c.exact_search(q, k))


@pytest.mark.parametrize("n", [1, 5, 127, 128, 129, 255, 257])
def test_n_around_the_row_tile_and_k_above_n(oracle, n):
    rows = elements_from_raw_rows("angular", random_vectors(n, 128, n))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(3, 128, 1)
    _same(g.exact_search_batch(q, 200), c.exact_search(q, 200))


@pytest.mark.parametrize("nq", [0, 1, 63, 64, 65, 1023, 1024, 1025])
def test_nq_around_the_query_block_and_chunk(oracle, nq):
    rows = elements_from_raw_rows("angular_int", random_vectors(300, 100, 2))
    g, c = _dense(oracle, "angular_int", rows)
    q = random_vectors(nq, 100, 3)
    got = g.exact_search_batch(q, 10)
    if nq == 0:
        assert got[0].shape == (0, 10)
        return
    _same(got, c.exact_search(q, 10))


def test_slab_boundary(oracle):
    # 1024 queries: a slab holds 65536 rows, so this scan has a full slab and a short one
    n = 65536 + 129
    rows = elements_from_raw_rows("angular", random_vectors(n, 32, 8))
    g, c = _dense(oracle, "angular", rows)
    q = random_vectors(1024, 32, 9)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10))


def test_index_shorter_than_container_and_empty(oracle):
    rows = elements_from_raw_rows("angular", random_vectors(500, 96, 4))
    q = random_vectors(20, 96, 5)
    for n in (0, 1, 300):
        g, c = _dense(oracle, "angular", rows, index_len=n)
        assert len(g) == n and g.num_elements() == 500
        got = g.exact_search_batch(q, 10)
        _same(got, c.exact_search(q, 10, index_len=n))
        assert (got[0][:, :min(n, 10)] < n).all() and (got[0][:, min(n, 10):] == 0xFFFFFFFF).all()


def test_ties(oracle):
    base = elements_from_raw_rows("angular", random_vectors(40, 64, 1))
    rows = np.concatenate([base, base, np.zeros((30, 64), np.float32), base[:1].repeat(50, 0), base]).astype(np.float32)
    g, c = _dense(oracle, "angular", rows)
    q = np.concatenate([base[:5], np.zeros((1, 64), np.float32)])
    got = g.exact_search_batch(q, 300, already_element=True)
    _same(got, c.exact_search(q, 300, already_element=True))
    assert (got[1][5][:len(rows)] == 1.0).all()  # the all-zero query: every distance is exactly 1
    rows8 =np.concatenate([_i8_rows(40, 64, 2)] * 3 + [np.zeros((20, 64), np.int8)])
    g, c = _dense(oracle, "angular_int", rows8)
    q8 = np.concatenate([rows8[:4], np.zeros((1, 64), np.int8)])
    got = g.exact_search_batch(q8, 150)
    _same(got, c.exact_search(q8, 150))


def test_nan_element_and_query(oracle):
    rows = elements_from_raw_rows("angular", random_vectors(200, 32, 1)).copy()
    rows[77, 3] = np.nan
    g, c = _dense(oracle, "angular", rows)
    with pytest.raises(xo.NotFinite):
        c.exact_search(random_vectors(2, 32, 2), 10)
    with pytest.raises(granne_b200.GranneError) as e:
        g.exact_search_batch(random_vectors(2, 32, 2), 10)
    assert e.value.code == NOT_FINITE
    g.exact_search_batch(random_vectors(2, 32, 2), 0)  # k == 0 reads no element
    rows[77, 3] = 0.0
    g, _ = _dense(oracle, "angular", rows)
    for kind, gg in (("angular", g), ("angular_int", _dense(oracle, "angular_int", _i8_rows(50, 32, 3))[0])):
        q = random_vectors(3, 32, 4)
        q[1, 0] = np.nan
        with pytest.raises(granne_b200.GranneError) as e:
            gg.exact_search_batch(q, 10)
        assert e.value.code == NOT_FINITE, kind


def _sum_case(dim, n, seed, num_rows=300):
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((num_rows, dim))).astype(np.float32)
    counts = [0, 1, 2, 7, 33, 40]
    elements = []
    for i in range(n):
        ids = rng.integers(0, num_rows, counts[i % len(counts)])
        if ids.size > 3:
            ids[2] = ids[0]  # repeated terms
        elements.append([int(t) for t in ids])
    return eo.table_image(table), eo.elements_image(elements)


@pytest.mark.parametrize("dim,n", [(20, 700), (100, 700), (2048, 20000)])
def test_embeddings(oracle, dim, n):
    ti, ei = _sum_case(dim, n, dim)
    m = n - 3
    g = granne_b200.Granne.from_bytes(xo.single_layer_index(oracle, m), "embeddings", ei, ti)
    c = xo.Container("embeddings", ei, ti)
    q = random_vectors(5, dim, 1)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10, index_len=m))


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
        _same((i.view(np.uint32), d, c.view(np.uint32)), want)


def test_multi_partitioned_and_replicated(oracle):
    sizes = [300, 1, 450]
    parts = [elements_from_raw_rows("angular", random_vectors(s, 48, 10 + i)) for i, s in enumerate(sizes)]
    shards = [(xo.single_layer_index(oracle, s), np.uint64(48).tobytes() + p.tobytes()) for s, p in zip(sizes, parts)]
    q = random_vectors(30, 48, 2)
    m = granne_b200.MultiGranne.partitioned(shards, "angular", [0])
    ids, d, cnt = m.exact_search_batch(q, 20)
    allrows = np.concatenate(parts)
    g, c = _dense(oracle, "angular", allrows)
    wi, wd, wc = c.exact_search(q, 20)
    assert np.array_equal(ids, wi.astype(np.uint64)) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(cnt, wc)
    r = granne_b200.MultiGranne.replicated(xo.single_layer_index(oracle, 751), "angular",
                                           np.uint64(48).tobytes() + allrows.tobytes(), [0, 0])
    ri, rd, rc = r.exact_search_batch(q, 20)
    gi, gd, gc = g.exact_search_batch(q, 20)
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
    _same(g.search_batch(q, n, 50), g.exact_search_batch(q, 50))


def test_at_size_f32_1m():
    import torch

    n, dim = 1_000_000, 128
    rows = torch.from_numpy(random_vectors(n, dim, 11)).cuda()
    el = granne_b200.elements_from_raw_device("angular", rows)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(xo.single_layer_index(go, n), "angular", el)
    host = el.cpu().numpy()
    c = xo.Container("angular", np.uint64(dim).tobytes() + host.tobytes())
    q = random_vectors(64, dim, 12)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10, threads=32))


def test_at_size_i8_10m():
    import torch

    n, dim = 10_000_000, 100
    rng = np.random.default_rng(5)
    host = rng.integers(-128, 128, (n, dim), dtype=np.int8)
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_device_elements(xo.single_layer_index(go, n), "angular_int",
                                                torch.from_numpy(host).cuda())
    c = xo.Container("angular_int", np.uint64(dim).tobytes() + host.tobytes())
    q = random_vectors(32, dim, 13)
    _same(g.exact_search_batch(q, 10), c.exact_search(q, 10, threads=32))


def test_cxx_client(tmp_path, oracle):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    rows = elements_from_raw_rows("angular", random_vectors(500, 64, 1))
    idx = tmp_path / "index.bin"
    els = tmp_path / "elements.bin"
    idx.write_bytes(xo.single_layer_index(oracle, 500))
    els.write_bytes(np.uint64(64).tobytes() + rows.tobytes())
    exe = tmp_path / "client"
    libdir = os.path.dirname(granne_b200.library_path())
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", "cxx_exact_client.cpp"), "-o", str(exe),
                           "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe), str(idx), str(els)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    g, c = _dense(oracle, "angular", rows)
    q = rows[:4]
    wi, wd, wc = c.exact_search(q, 5, already_element=True)
    lines = out.stdout.split()
    assert [int(x) for x in lines] == wi.ravel().tolist()
