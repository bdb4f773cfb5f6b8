"""Exact search within caller-given candidate lists on the GPU (granne_b200_exact_search_within_batch*).  Ids,
distance bits and counts equal an oracle composed from the CPU oracle's own pieces: Elements.dist_to_element gives
each listed element's distance, the unique ids sorted by (distance, id) give the first k.  Also: every engine, list
shapes around the segment, k and nq edges, the identities with exact and graph search, ties and NaN, the rejections,
the device variant under concurrency, every handle source, the multi handle and a C++ client."""
import os
import shutil
import subprocess
import threading

import numpy as np
import pytest

import granne_b200
from helpers import exact_oracle as xo
from helpers.data import clustered_vectors, random_sum_embeddings, random_vectors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, NOT_FINITE = -1, -6
UNUSED = 0xFFFFFFFF


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _image(rows):
    rows = np.ascontiguousarray(rows)
    return np.uint64(rows.shape[1]).tobytes() + rows.tobytes()


def _rows(image, dt):
    dim = int(np.frombuffer(bytes(image[:8]), dtype=np.uint64)[0])
    return np.frombuffer(bytes(image[8:]), dtype=dt).reshape(-1, dim)


def _elements(kind, raw):
    return _rows(granne_b200.elements_from_raw(kind, raw), np.float32 if kind == "angular" else np.int8)


class Case:
    """A GPU handle and the oracle container over the same elements; the index covers index_len of them."""

    def __init__(self, go, kind, rows=None, index_len=None, sum_el=None):
        if sum_el is not None:
            self.el = sum_el
            eb, mb = sum_el.to_bytes(0), sum_el.to_bytes(1)
        else:
            eb, mb = _image(rows), None
            self.el = go.Elements.from_bytes(kind, eb)
        self.n = len(self.el) if index_len is None else index_len
        self.index_bytes = xo.single_layer_index(go, self.n)
        self.kind, self.eb, self.mb = kind, eb, mb
        self.g = granne_b200.Granne.from_bytes(self.index_bytes, kind, eb, mb)

    def want(self, q, lists, k, already_element=False):
        nq = len(q)
        ids = np.full((nq, k), UNUSED, np.uint32)
        dists = np.full((nq, k), np.inf, np.float32)
        counts = np.zeros(nq, np.uint32)
        for i, lst in enumerate(lists):
            s = np.unique(np.asarray(lst, np.int64)).astype(np.uint32)
            d = np.array([self.el.dist_to_element(int(j), q[i], already_element) for j in s], np.float32)
            order = np.lexsort((s, d))[:k]
            ids[i, :order.size] = s[order]
            dists[i, :order.size] = d[order]
            counts[i] = order.size
        return ids, dists, counts


def _same(got, want):
    gi, gd, gc = (np.asarray(x) for x in got)
    wi, wd, wc = want
    assert np.array_equal(gc.view(np.uint32), wc)
    assert np.array_equal(gi.view(np.uint32), wi)
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))


def _lists(rng, n, lengths):
    return [rng.integers(0, n, size=L).astype(np.uint32) for L in lengths]


# DistF32<FULL> for FULL = 0, 1, 2, 3, 4, 6, 8; DistF32Generic with staged rows and with direct loads
@pytest.mark.parametrize("dim", [1, 31, 32, 33, 64, 96, 100, 128, 160, 192, 256, 300, 1000, 2080, 2100])
def test_every_f32_engine_layout(oracle, dim):
    rows = _elements("angular", random_vectors(1500, dim, dim))
    c = Case(oracle, "angular", rows)
    rng = np.random.default_rng(dim)
    q = random_vectors(6, dim, dim + 1)
    lists = _lists(rng, 1500, [0, 1, 9, 40, 1024, 1300])
    _same(c.g.exact_search_within(q, lists, 10), c.want(q, lists, 10))
    qe = rows[[3, 700]]
    le = lists[2:4]
    _same(c.g.exact_search_within(qe, le, 10, already_element=True), c.want(qe, le, 10, True))


# DistI8 over rows of 16 bytes up to beyond its 512-byte sub-warp path
@pytest.mark.parametrize("dim", [1, 16, 100, 128, 512, 513, 1000])
def test_i8_every_width(oracle, dim):
    rows = _elements("angular_int", random_vectors(1500, dim, dim))
    c = Case(oracle, "angular_int", rows)
    rng = np.random.default_rng(dim)
    q = random_vectors(5, dim, dim + 1)
    lists = _lists(rng, 1500, [1, 31, 33, 1025, 2100])
    _same(c.g.exact_search_within(q, lists, 10), c.want(q, lists, 10))
    qe = rows[[0, 1499]]
    _same(c.g.exact_search_within(qe, lists[:2], 10), c.want(qe.astype(np.float32), lists[:2], 10, True))


@pytest.mark.parametrize("dim, num_embeddings", [(20, 300), (128, 50), (1000, 40), (4096, 8)])
def test_sum_embeddings(oracle, dim, num_embeddings):
    el = random_sum_embeddings(oracle, dim, num_embeddings, 1200, dim)
    c = Case(oracle, "embeddings", sum_el=el)
    rng = np.random.default_rng(dim)
    q = random_vectors(4, dim, dim + 1)
    lists = _lists(rng, 1200, [1, 50, 1024, 1100])
    _same(c.g.exact_search_within(q, lists, 10), c.want(q, lists, 10))


def test_sum_embeddings_term_edges(oracle):
    # 0 terms, more than 32 terms, repeated terms
    emb = random_vectors(64, 48, 1)
    terms = [[], list(range(40)), [5, 5, 5, 9], [63] * 70, [1, 2]] * 30
    el = oracle.Elements.sum_embeddings(emb, terms)
    c = Case(oracle, "embeddings", sum_el=el)
    q = random_vectors(3, 48, 2)
    lists = [np.arange(150), np.arange(0, 150, 5), np.array([1, 3, 1, 3])]
    _same(c.g.exact_search_within(q, lists, 20), c.want(q, lists, 20))


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_list_lengths_around_the_segment(oracle, kind):
    rows = _elements(kind, random_vectors(6000, 64, 3))
    c = Case(oracle, kind, rows)
    rng = np.random.default_rng(4)
    k = 10
    lengths = [0, 1, k - 1, k, k + 1, 1023, 1024, 1025, 2048, 5000]
    q = random_vectors(len(lengths), 64, 5)
    lists = _lists(rng, 6000, lengths)  # mixed lengths in one launch
    _same(c.g.exact_search_within(q, lists, k), c.want(q, lists, k))
    # one query at a time: the same rows
    for i in (0, 4, 7, 9):
        _same(c.g.exact_search_within(q[i:i + 1], lists[i:i + 1], k), c.want(q[i:i + 1], lists[i:i + 1], k))


def test_empty_lists(oracle):
    rows = _elements("angular", random_vectors(100, 32, 1))
    c = Case(oracle, "angular", rows)
    q = random_vectors(5, 32, 2)
    got = c.g.exact_search_within(q, [np.zeros(0, np.uint32)] * 5, 10)
    _same(got, c.want(q, [[]] * 5, 10))
    assert (got[2] == 0).all() and (got[0] == UNUSED).all() and np.isinf(got[1]).all()
    lists = [[], [4], [], [5, 6], []]
    _same(c.g.exact_search_within(q, lists, 10), c.want(q, lists, 10))


def test_one_long_list(oracle):
    rows = _elements("angular", random_vectors(250_000, 32, 6))
    c = Case(oracle, "angular", rows)
    rng = np.random.default_rng(7)
    q = random_vectors(1, 32, 8)
    lst = rng.permutation(250_000)[:200_000].astype(np.uint32)
    got = c.g.exact_search_within(q, [lst], 100)
    # its answer is exact search's over the listed rows: a handle over just those rows, in listed order
    sub = np.sort(lst)
    sc = Case(oracle, "angular", rows[sub])
    ei, ed, ec = sc.g.exact_search_batch(q, 100)
    assert np.array_equal(got[2], ec)
    assert np.array_equal(got[0], sub[ei])  # sub is increasing, so (distance, id) order is kept
    assert np.array_equal(got[1].view(np.uint32), ed.view(np.uint32))


def test_order_and_multiplicity_do_not_matter(oracle):
    rows = _elements("angular", random_vectors(3000, 96, 9))
    c = Case(oracle, "angular", rows)
    rng = np.random.default_rng(10)
    q = random_vectors(3, 96, 11)
    base = rng.permutation(3000)[:2500].astype(np.uint32)
    want = c.g.exact_search_within(q, [np.sort(base)] * 3, 50)
    _same(c.g.exact_search_within(q, [rng.permutation(base) for _ in range(3)], 50), want)
    # an id repeated across segments, 3000 times, counts once; so do doubled lists
    rep = np.concatenate([np.repeat(base[:1], 3000), base])
    _same(c.g.exact_search_within(q, [rep, np.concatenate([base, base]), rng.permutation(rep)], 50), want)
    _same(want, c.want(q, [base] * 3, 50))
    # the segments of a long list finish in any order: repeated calls give the same answer
    for _ in range(3):
        _same(c.g.exact_search_within(q, [rng.permutation(rep) for _ in range(3)], 50), want)


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("k", [0, 1, 10, 1024, 1025])
def test_k(oracle, kind, k):
    rows = _elements(kind, random_vectors(5000, 64, 12))
    c = Case(oracle, kind, rows)
    rng = np.random.default_rng(13)
    q = random_vectors(4, 64, 14)
    lists = _lists(rng, 5000, [3, 1000, 1500, 4000])
    if k > granne_b200.api.EXACT_MAX_K:
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.exact_search_within(q, lists, k)
        assert e.value.code == INVALID
        return
    _same(c.g.exact_search_within(q, lists, k), c.want(q, lists, k))


@pytest.mark.parametrize("nq", [0, 1, 1023, 1024, 1025, 2100])
def test_nq_and_query_chunks(oracle, nq):
    rows = _elements("angular_int", random_vectors(400, 100, 15))
    c = Case(oracle, "angular_int", rows)
    rng = np.random.default_rng(nq)
    q = random_vectors(nq, 100, 16)
    lists = _lists(rng, 400, rng.integers(0, 1500, size=nq))
    got = c.g.exact_search_within(q, lists, 10)
    if nq == 0:
        assert got[0].shape == (0, 10)
        return
    _same(got, c.want(q, lists, 10))


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_all_ids_is_exact_search(kind):
    n, dim = 300_000, 64
    rows = _elements(kind, clustered_vectors(n, dim, 17))
    from oracle import granne_oracle as go

    g = granne_b200.Granne.from_bytes(xo.single_layer_index(go, n), kind, _image(rows))
    q = clustered_vectors(40, dim, 18)
    want = g.exact_search_batch(q, 100)
    got = g.exact_search_within(q, [np.arange(n, dtype=np.uint32)] * len(q), 100)
    _same(got, want)
    # shuffled: the same
    rng = np.random.default_rng(19)
    _same(g.exact_search_within(q[:4], [rng.permutation(n).astype(np.uint32) for _ in range(4)], 100),
          tuple(x[:4] for x in want))


def test_search_result_set_is_search():
    n, dim, ef = 1_000_000, 32, 120
    raw = clustered_vectors(n, dim, 20)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw), num_neighbors=16,
                                  max_search=60)
    b.build()
    g = b.get_index()
    q = clustered_vectors(500, dim, 21)
    si, sd, sc = g.search_batch(q, ef, ef)
    lists = [si[i, :sc[i]] for i in range(len(q))]
    for k in (1, 10, ef):
        ki, kd, kc = g.search_batch(q, ef, k)
        _same(g.exact_search_within(q, lists, k), (ki, kd, kc))


def test_ties_and_zero_distances(oracle):
    base = _elements("angular", random_vectors(40, 64, 1))
    rows = np.concatenate([base, base, np.zeros((30, 64), np.float32), base[:1].repeat(50, 0), -base, base])
    c = Case(oracle, "angular", rows.astype(np.float32))
    q = np.concatenate([base[:5], np.zeros((1, 64), np.float32), -base[:1]])
    lists = [np.arange(len(rows))[::-1].copy()] * len(q)
    got = c.g.exact_search_within(q, lists, 300, already_element=True)
    _same(got, c.want(q, lists, 300, True))
    assert (got[1][5][:len(rows)] == 1.0).all()  # the all-zero query: every distance is exactly 1
    # i8 element queries: rows of quantised elements, which the oracle's quantisation leaves as they are
    rows8 = np.concatenate([_elements("angular_int", random_vectors(40, 64, 2))] * 3 + [np.zeros((20, 64), np.int8)])
    c8 = Case(oracle, "angular_int", rows8)
    q8 = rows8[:4]
    lists8 = [np.arange(len(rows8))] * len(q8)
    _same(c8.g.exact_search_within(q8, lists8, 150), c8.want(q8.astype(np.float32), lists8, 150, True))


def test_nan(oracle):
    rows = _elements("angular", random_vectors(2000, 32, 22)).copy()
    rows[777] = np.nan
    c = Case(oracle, "angular", rows)
    q = random_vectors(3, 32, 23)
    # a NaN element no list names: the call succeeds
    lists = [np.arange(0, 700), np.arange(800, 2000), np.array([5, 6])]
    _same(c.g.exact_search_within(q, lists, 10), c.want(q, lists, 10))
    # a listed NaN element, in a list of one segment and in a list of several
    for lst in (np.array([1, 777, 3]), np.arange(2000)):
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.exact_search_within(q[:1], [lst], 10)
        assert e.value.code == NOT_FINITE
    # a NaN query
    qn = q.copy()
    qn[1, 4] = np.nan
    with pytest.raises(granne_b200.GranneError) as e:
        c.g.exact_search_within(qn, lists, 10)
    assert e.value.code == NOT_FINITE
    c8 = Case(oracle, "angular_int", _elements("angular_int", random_vectors(100, 32, 24)))
    with pytest.raises(granne_b200.GranneError) as e:
        c8.g.exact_search_within(qn[1:2], [np.array([1, 2])], 10)
    assert e.value.code == NOT_FINITE


def test_host_rejections(oracle):
    rows = _elements("angular", random_vectors(500, 32, 25))
    c = Case(oracle, "angular", rows, index_len=300)  # a container larger than its index
    q = random_vectors(2, 32, 26)
    launches = c.g.launch_count()
    for bad in ([np.array([1, 300])], [np.array([499])], [np.array([2**32 - 1])]):
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.exact_search_within(q[:1], bad, 10)
        assert e.value.code == INVALID and "Index::len" in str(e.value)
    for offsets in ([1, 1, 2], [0, 2, 1]):
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.exact_search_within(q, granne_b200.CsrLists(np.array(offsets), np.array([1, 2], np.uint32)), 10)
        assert e.value.code == INVALID
    # offsets past the end of the ids given: rejected before the library reads the buffer
    with pytest.raises(ValueError, match="exceeds"):
        c.g.exact_search_within(q, granne_b200.CsrLists(np.array([0, 1, 9]), np.array([1, 2], np.uint32)), 10)
    assert c.g.launch_count() == launches  # rejected before any device call
    _same(c.g.exact_search_within(q, [[299], [0, 299]], 10), c.want(q, [[299], [0, 299]], 10))


def _device_lists(lists, dev):
    import torch

    offsets = np.zeros(len(lists) + 1, np.int64)
    np.cumsum([len(x) for x in lists], out=offsets[1:])
    ids = np.concatenate([np.asarray(x, np.uint32) for x in lists]) if lists else np.zeros(0, np.uint32)
    return (torch.from_numpy(offsets).to(dev), torch.from_numpy(ids.view(np.int32)).to(dev))


def test_device_rejections(oracle):
    import torch

    rows = _elements("angular", random_vectors(500, 32, 27))
    c = Case(oracle, "angular", rows, index_len=300)
    dev = torch.device("cuda", 0)
    q = torch.from_numpy(random_vectors(3, 32, 28)).to(dev)
    good = [np.array([1, 2]), np.arange(3000) % 300, np.array([7])]
    for lists in ([good[0], np.array([5, 300]), good[2]],
                  [good[0], np.concatenate([np.arange(2000) % 300, [450]]), good[2]]):
        offsets, ids = _device_lists(lists, dev)
        ri, rd, rc = c.g.exact_search_within_device(q, offsets, ids, 10)
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.stream_status()
        assert e.value.code == INVALID
        want = c.want(q.cpu().numpy(), good, 10)
        # the query with the bad list writes count 0 and padding; the others are answered
        assert rc.cpu().numpy()[1] == 0 and (ri.cpu().numpy()[1].view(np.uint32) == UNUSED).all()
        for i in (0, 2):
            assert np.array_equal(ri.cpu().numpy()[i].view(np.uint32), want[0][i])
    offsets, ids = _device_lists(good, dev)
    for bad in ([0, 2, 1, 3003], [1, 2, 3002, 3003]):
        ri, rd, rc = c.g.exact_search_within_device(q, torch.tensor(bad, dtype=torch.int64, device=dev), ids, 10)
        with pytest.raises(granne_b200.GranneError) as e:
            c.g.stream_status()
        assert e.value.code == INVALID
    ri, rd, rc = c.g.exact_search_within_device(q, offsets, ids, 10)
    c.g.stream_status()
    _same((ri.cpu(), rd.cpu(), rc.cpu()), c.want(q.cpu().numpy(), good, 10))


def test_device_variant_streams_and_threads(oracle):
    import torch

    rows = _elements("angular_int", random_vectors(20000, 100, 29))
    c = Case(oracle, "angular_int", rows)
    rng = np.random.default_rng(30)
    dev = torch.device("cuda", 0)
    batches = []
    for s in range(6):
        q = random_vectors(300, 100, 100 + s)
        lists = _lists(rng, 20000, rng.integers(0, 3000, size=300))
        batches.append((q, lists, c.g.exact_search_within(q, lists, 20)))
    _same(batches[0][2], c.want(batches[0][0], batches[0][1], 20))
    streams = [torch.cuda.Stream(dev) for _ in range(3)]
    outs = []
    for i, (q, lists, _) in enumerate(batches):
        with torch.cuda.stream(streams[i % 3]):
            qd = torch.from_numpy(q).to(dev)
            offsets, ids = _device_lists(lists, dev)
            outs.append((qd, offsets, ids, c.g.exact_search_within_device(qd, offsets, ids, 20,
                                                                          stream=streams[i % 3])))
    torch.cuda.synchronize(dev)
    c.g.stream_status()
    for (q, lists, want), (_, _, _, got) in zip(batches, outs):
        _same(tuple(t.cpu() for t in got), want)
    errors = []

    def worker(i):
        try:
            q, lists, want = batches[i]
            for _ in range(3):
                _same(c.g.exact_search_within(q, lists, 20), want)
        except Exception as e:  # noqa: BLE001 — reported below
            errors.append(e)

    th = [threading.Thread(target=worker, args=(i,)) for i in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    for s in streams:
        c.g.release_stream(s)


def test_handle_sources(oracle):
    import torch

    raw = random_vectors(3000, 128, 31)
    rows = _elements("angular", raw)
    c = Case(oracle, "angular", rows)
    rng = np.random.default_rng(32)
    q = random_vectors(8, 128, 33)
    lists = _lists(rng, 3000, [5, 100, 1024, 1025, 2900, 0, 1, 3000])
    want = c.want(q, lists, 10)
    _same(c.g.exact_search_within(q, lists, 10), want)
    d = granne_b200.Granne.from_device_elements(c.index_bytes, "angular",
                                                torch.from_numpy(rows.copy()).to(torch.device("cuda", 0)))
    _same(d.exact_search_within(q, lists, 10), want)
    # a builder's get_index after append: the appended rows are listed too
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw[:2000]), num_neighbors=10,
                                  max_search=40)
    b.build()
    for v in raw[2000:]:
        b.append(v)
    b.build()
    snap = b.get_index()
    assert len(snap) == 3000
    _same(snap.exact_search_within(q, lists, 10), want)


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_multi_handle(oracle, mode):
    dim = 64
    raw = random_vectors(3000, dim, 34)
    rows = _elements("angular", raw)
    rng = np.random.default_rng(35)
    q = random_vectors(7, dim, 36)
    lists = _lists(rng, 3000, [0, 1, 50, 1024, 1500, 2999, 3000])
    full = Case(oracle, "angular", rows)
    want = full.want(q, lists, 10)
    if mode == "replicated":
        m = granne_b200.MultiGranne.replicated(full.index_bytes, "angular", full.eb, [0, 0])
    else:
        cuts = [0, 1000, 2200, 3000]
        shards = [(xo.single_layer_index(oracle, b - a), _image(rows[a:b])) for a, b in zip(cuts, cuts[1:])]
        m = granne_b200.MultiGranne.partitioned(shards, "angular", [0, 0])
    gi, gd, gc = m.exact_search_within(q, [x.astype(np.uint64) for x in lists], 10)
    wi = np.where(want[0] == UNUSED, np.iinfo(np.uint64).max, want[0].astype(np.uint64))
    assert np.array_equal(gc, want[2])
    assert np.array_equal(gi, wi)
    assert np.array_equal(gd.view(np.uint32), want[1].view(np.uint32))
    with pytest.raises(granne_b200.GranneError) as e:
        m.exact_search_within(q[:1], [np.array([3000], np.uint64)], 10)
    assert e.value.code == INVALID


def test_cxx_client(oracle, tmp_path):
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    rows = _elements("angular", random_vectors(2000, 64, 37))
    c = Case(oracle, "angular", rows)
    idx, el = tmp_path / "index.bin", tmp_path / "elements.bin"
    idx.write_bytes(c.index_bytes)
    el.write_bytes(c.eb)
    exe = tmp_path / "client"
    libdir = os.path.dirname(granne_b200.library_path())
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", "cxx_within_client.cpp"), "-o", str(exe),
                           "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe), str(idx), str(el)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    wi, wd, wc = c.want(rows[7:8], [np.concatenate([np.arange(100), np.arange(50, 150)])], 5, already_element=True)
    lines = out.stdout.split()
    assert [int(x) for x in lines[0::2]] == wi.ravel().tolist()
    assert [np.float32(x).view(np.uint32) for x in lines[1::2]] == wd.ravel().view(np.uint32).tolist()
