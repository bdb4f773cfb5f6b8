"""GPU GranneBuilder (SURVEY.md §8f-1/2): built like the reference's own build tests check it
(src/index/tests.rs:41-132: self-recall > 0.95; :305-335 layer sizes; :337-451 write/load round trip), plus: an index
written by the GPU builder is a valid granne file (the CPU oracle loads it) and searching it on the GPU is
bit-identical to the oracle searching the same file."""
import numpy as np
import pytest

import granne_b200
from helpers.data import clustered_vectors, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


def test_elements_from_raw_matches_vector_from(oracle):
    raw = random_vectors(300, 100, seed=1)
    raw[7] = 0.0  # the zero vector stays zero (norm == 0, math.rs:141)
    eb = granne_b200.elements_from_raw("angular", raw).tobytes()
    assert eb == oracle.Elements.angular(raw).to_bytes()
    ib = granne_b200.elements_from_raw("angular_int", raw).tobytes()
    assert ib == oracle.Elements.angular_int(raw).to_bytes()
    for dim in [3, 28, 32, 33, 128]:
        r = random_vectors(50, dim, seed=dim)
        assert granne_b200.elements_from_raw("angular", r).tobytes() == oracle.Elements.angular(r).to_bytes()


def _self_recall(index, rows, max_search):
    ids, dists, counts = index.search_batch(rows, max_search, 1, already_element=True)
    return float((ids[:, 0] == np.arange(rows.shape[0])).mean())


@pytest.mark.parametrize("kind,n,dim,m", [("angular", 1500, 28, 20), ("angular_int", 500, 32, 20),
                                          ("angular", 3000, 128, 20), ("angular", 2500, 32, 48),
                                          ("angular_int", 1200, 40, 70)])
def test_build_and_search_like_the_reference(oracle, kind, n, dim, m):
    # build_and_search_float / build_and_search_int8 (src/index/tests.rs:41-62,114-132): M=20, max_search=20,
    # then every element must find itself with max_search = 10.  BuildConfig has no cap on num_neighbors
    # (src/index/mod.rs:198-291): rows wider than a warp (48, 70) go through the same kernels 32 slots at a time.
    raw = random_vectors(n, dim, seed=n)
    eb = granne_b200.elements_from_raw(kind, raw).tobytes()
    b = granne_b200.GranneBuilder(kind, eb, num_neighbors=m, max_search=max(20, m))
    b.build()
    assert len(b) == n
    expect_layers = []
    l = 0
    while not expect_layers or expect_layers[-1] < n:  # compute_num_elements_in_layer (:634-643)
        expect_layers.append(oracle.num_elements_in_layer(n, 15.0, l))
        l += 1
    assert [b.layer_len(i) for i in range(b.num_layers())] == expect_layers
    index = b.get_index()
    el = oracle.Elements.from_bytes(kind, eb)
    rows = el.rows()
    assert _self_recall(index, rows, 10) > 0.95
    # degrees respect num_neighbors (and num_neighbors / 2 on upper layers, :665-668)
    for layer in range(index.num_layers()):
        limit = m if layer == index.num_layers() - 1 else m // 2
        for i in range(0, index.layer_len(layer), 37):
            nb = index.get_neighbors(i, layer)
            assert len(nb) <= limit and len(set(nb)) == len(nb) and i not in nb
    # the written index is a valid granne file: the oracle loads it, and both sides search it identically
    image = b.index_bytes().tobytes()
    g = oracle.Granne.from_bytes(image, el)
    assert [g.layer_len(i) for i in range(g.num_layers())] == expect_layers
    for layer in range(g.num_layers()):
        for i in range(0, g.layer_len(layer), 53):
            assert g.get_neighbors(i, layer) == sorted(index.get_neighbors(i, layer))
    p = granne_b200.Granne.from_bytes(image, kind, eb)
    q = random_vectors(100, dim, seed=5)
    ref = g.search_batch(q, 50, 10, with_stats=True)
    got = p.search_batch(q, 50, 10, with_stats=True)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1].view(np.uint32), got[1].view(np.uint32))
    assert np.array_equal(ref[3][:, :3], got[3][:, :3])
    p.close()
    index.close()
    b.close()


def test_incremental_build_and_snapshots(oracle):
    # incremental_build_* (src/index/tests.rs:134-242): build_partial in steps; earlier snapshots stay valid
    raw = random_vectors(1200, 25, seed=9)
    eb = granne_b200.elements_from_raw("angular", raw).tobytes()
    b = granne_b200.GranneBuilder("angular", eb, num_neighbors=20, max_search=20, expected_num_elements=1200)
    b.build(0 + 300)
    snap = b.get_index()
    assert len(b) == 300 and len(snap) == 300
    b.build(900)
    b.build()
    assert len(b) == 1200 and len(snap) == 300
    rows = oracle.Elements.from_bytes("angular", eb).rows()
    assert _self_recall(snap, rows[:300], 40) > 0.95
    full = b.get_index()
    assert _self_recall(full, rows, 40) > 0.95
    with pytest.raises(granne_b200.GranneError):
        b.build(100)  # "Cannot index fewer elements than already in index." (:379-382)
    snap.close()
    full.close()
    b.close()


def test_recall_against_brute_force():
    import torch

    n, dim = 50_000, 64
    raw = clustered_vectors(n, dim, seed=3)
    eb = granne_b200.elements_from_raw("angular", raw).tobytes()
    b = granne_b200.GranneBuilder("angular", eb, num_neighbors=30, max_search=200)
    b.build()
    index = b.get_index()
    q = clustered_vectors(512, dim, seed=4)
    ids, d, c = index.search_batch(q, 200, 10)
    rows = torch.from_numpy(np.frombuffer(eb, dtype=np.float32, offset=8).reshape(n, dim).copy()).cuda()
    qn = torch.nn.functional.normalize(torch.from_numpy(q).cuda(), dim=1)
    gt = torch.topk(qn @ rows.T, 10, dim=1).indices.cpu().numpy()
    recall = np.mean([len(set(gt[i]) & set(ids[i].tolist())) / 10 for i in range(512)])
    assert recall > 0.95, recall
    index.close()
    b.close()


def test_builder_queries_that_overflow_the_fast_path():
    # Uniform random vectors have little neighbourhood overlap, so a search visits almost max_search x degree nodes and
    # regularly exceeds the per-warp visited table: those insertions / queries take the slow pass while the index under
    # construction keeps growing (regression: the slow-path buffers must follow the index size, not the size at the
    # time the builder's workspace was created).
    raw = random_vectors(30_000, 64, seed=11)
    eb = granne_b200.elements_from_raw("angular", raw).tobytes()
    b = granne_b200.GranneBuilder("angular", eb, num_neighbors=31, max_search=40)
    b.build()
    index = b.get_index()
    ids, d, c, st = index.search_batch(random_vectors(2000, 64, seed=12), 40, 10, with_stats=True)
    assert (c == 10).all()
    assert int((st[:, 3] != 0).sum()) > 0  # passes beyond the fast one really are exercised with these parameters
    rows = np.frombuffer(eb, dtype=np.float32, offset=8).reshape(30_000, 64)
    assert _self_recall(index, rows[:3000], 40) > 0.9
    index.close()
    b.close()


def test_python_class_surface_save_and_reload(tmp_path, oracle):
    # py/src/lib.rs:325-343 (Granne.save_index / save_elements), :504-579 (GranneBuilder.save_index / save_elements /
    # get_neighbors / num_elements): the files written are granne files — the oracle's loader reads them back
    raw = random_vectors(900, 16, seed=21)
    eb = granne_b200.elements_from_raw("angular", raw).tobytes()
    b = granne_b200.GranneBuilder("angular", eb, num_neighbors=12, max_search=30)
    b.build(500)
    assert len(b) == 500 and b.num_elements() == 900
    b.build()
    ip, ep = str(tmp_path / "index.granne"), str(tmp_path / "elements.bin")
    b.save_index(ip)
    b.save_elements(ep)
    index = granne_b200.Granne(ip, "angular", ep)
    assert len(index) == 900 and index.num_elements() == 900
    last = index.num_layers() - 1
    for node in (0, 1, 17, 899):
        # builder rows are in insertion order (FixedWidthSliceVector), file rows are sorted (set_vector.rs:117-148)
        assert sorted(b.get_neighbors(node)) == index.get_neighbors(node) == index.get_neighbors(node, last)
    assert sorted(b.get_neighbors(0, 0)) == index.get_neighbors(0, 0)
    ip2, ep2 = str(tmp_path / "index2.granne"), str(tmp_path / "elements2.bin")
    index.save_index(ip2)
    index.save_elements(ep2)
    assert open(ip2, "rb").read() == open(ip, "rb").read() and open(ep2, "rb").read() == eb
    snap = b.get_index()
    snap.save_index(ip2)
    assert open(ip2, "rb").read() == open(ip, "rb").read()
    ref = oracle.Granne.from_bytes(open(ip, "rb").read(), oracle.Elements.from_bytes("angular", open(ep, "rb").read()))
    q = random_vectors(64, 16, seed=22)
    want = ref.search_batch(q, 30, 5)
    got = index.search_batch(q, 30, 5)
    assert np.array_equal(want[0], got[0]) and np.array_equal(want[1].view(np.uint32), got[1].view(np.uint32))
    for h in (snap, index, b):
        h.close()


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_append_then_build_incrementally(oracle, kind):
    # GranneBuilder.append (py/src/lib.rs:474-476 -> GranneBuilder::push, src/index/mod.rs:512-531): pushed elements are
    # `Vector::from(raw)` and get indexed by the next build(); earlier snapshots keep their container
    raw = random_vectors(1000, 24, seed=31)
    whole = granne_b200.elements_from_raw(kind, raw).tobytes()
    first = granne_b200.elements_from_raw(kind, raw[:600]).tobytes()
    b = granne_b200.GranneBuilder(kind, first, num_neighbors=20, max_search=30)
    b.build()
    snap = b.get_index()
    assert len(b) == 600 and b.num_elements() == 600
    for row in raw[600:]:
        b.append(row.tolist())
    assert b.num_elements() == 1000 and len(b) == 600            # pushed, not yet indexed
    b.build(800)
    assert len(b) == 800
    b.build()
    assert len(b) == 1000 and len(snap) == 600 and snap.num_elements() == 600
    index = b.get_index()
    rows = oracle.Elements.from_bytes(kind, whole).rows()
    for i in (0, 599, 600, 777, 999):
        assert np.array_equal(index.get_element(i), rows[i])
    assert _self_recall(index, rows, 30) > 0.95
    assert _self_recall(snap, rows[:600], 30) > 0.95
    assert bytes(index.elements_bytes()) == whole
    # the index over the appended container is a valid granne index: the oracle searches it identically
    g = oracle.Granne.from_bytes(index.index_bytes(), oracle.Elements.from_bytes(kind, whole))
    q = random_vectors(64, 24, seed=32)
    ref = g.search_batch(q, 40, 10, with_stats=True)
    got = index.search_batch(q, 40, 10, with_stats=True)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1].view(np.uint32), got[1].view(np.uint32))
    with pytest.raises(granne_b200.GranneError):
        b._pending.append(np.zeros(7, dtype=np.float32))           # wrong width is rejected by the library
        b._flush()
    for h in (snap, index, b):
        h.close()


def test_append_to_an_embeddings_builder(oracle):
    """ExtendableElementContainer for SumEmbeddings (src/elements/embeddings/mod.rs:97-100,177-189): elements (lists of
    embedding ids) pushed after a first build are indexed by the next one; the container then equals the one built in
    one go, and the oracle searches the resulting index identically."""
    from granne_b200 import words as W
    from helpers.data import random_sum_embeddings

    dim, n_emb, n = 24, 120, 700
    el = random_sum_embeddings(oracle, dim, n_emb, n, seed=8)
    whole, emb = el.to_bytes(0), el.to_bytes(1)
    lists = W.read_sum_terms(whole)
    assert W.write_sum_terms(lists) == whole                      # the writer is the exact inverse of the reader
    first = W.write_sum_terms(lists[:400])
    b = granne_b200.GranneBuilder("embeddings", first, emb, num_neighbors=16, max_search=30)
    b.build()
    snap = b.get_index()
    assert len(b) == 400
    for l in lists[400:]:
        b.append(l)
    assert b.num_elements() == n and len(b) == 400                # pushed, not yet indexed
    b.build()
    assert len(b) == n and len(snap) == 400
    index = b.get_index()
    for i in (0, 399, 400, 555, n - 1):
        assert np.array_equal(index.get_element(i), el.get(i))
    assert bytes(index.elements_bytes()) == whole
    g = oracle.Granne.from_bytes(index.index_bytes(), el)
    q = random_vectors(64, dim, seed=9)
    ref = g.search_batch(q, 40, 10, with_stats=True)
    got = index.search_batch(q, 40, 10, with_stats=True)
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1].view(np.uint32), got[1].view(np.uint32))
    assert np.array_equal(ref[3][:, :3], got[3][:, :3])
    with pytest.raises(granne_b200.GranneError):
        b.append([n_emb + 5])                                      # a missing embedding id is rejected by the library
        b._flush()
    for h in (snap, index, b):
        h.close()
