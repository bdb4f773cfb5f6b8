"""The GPU GranneBuilder's default batched build (builder_index_elements in granne_b200.cu, build_link_kernel in
build_kernels.cuh) against the oracle's model of the same batch schedule (oracle GranneBuilder.build_batched): every
member of a batch searches one snapshot of the layer, then the members are linked in.

A. With GRANNE_B200_BUILD_LINK_WARPS=1 one warp links a batch's members in batch order, which is exactly the model's
   schedule: the index image must equal the model's byte for byte.  This checks the batch sizes, the id order of both
   passes, the by-id search of a whole batch and its result tiles.
B. At the default link grid the members of a batch are linked concurrently under per-node spin locks.  When no
   connect_nodes overflows and no select_neighbors has more candidates than its limit, every row ends as the SET of the
   links made into it whatever the interleaving (search results depend only on row contents), and the written index
   stores sorted lists: the image must still equal the model's.  A lost or duplicated link under contention breaks it.
C. Concurrent builds with overflow depend on the interleaving; every row of every layer is checked for the invariants
   the final prune guarantees, and recall must match the serialized-link build of the same data."""
import os

import numpy as np
import pytest

import granne_b200
from helpers.data import clustered_vectors, random_sum_embeddings, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)
from helpers.index_image import assert_same_index

pytestmark = pytest.mark.gpu

DEFAULT_MAX_BATCH = 4096  # the builder's largest insertion batch when GRANNE_B200_BUILD_MAX_BATCH is unset
THREADS = max(1, min(16, os.cpu_count() or 1))  # the model's searches of one batch; its image does not depend on it


@pytest.fixture(autouse=True)
def _default_knobs(monkeypatch):
    # both knobs are read by the library on every build call
    monkeypatch.delenv("GRANNE_B200_BUILD_MAX_BATCH", raising=False)
    monkeypatch.delenv("GRANNE_B200_BUILD_LINK_WARPS", raising=False)


def _set_knobs(monkeypatch, max_batch=None, link_warps=None):
    if max_batch is not None:
        monkeypatch.setenv("GRANNE_B200_BUILD_MAX_BATCH", str(max_batch))
    if link_warps is not None:
        monkeypatch.setenv("GRANNE_B200_BUILD_LINK_WARPS", str(link_warps))


def _elements(oracle, kind, raw=None, n=0, dim=0, seed=0):
    if kind == "embeddings":
        el = random_sum_embeddings(oracle, dim, 200, n, seed)
        return el, el.to_bytes(1)
    raw = random_vectors(n, dim, seed) if raw is None else raw
    return (oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)), None


def gpu_build(kind, el, emb, **cfg):
    b = granne_b200.GranneBuilder(kind, el.to_bytes(0), emb, **cfg)
    b.build()
    return b


def model_build(oracle, el, max_batch, **cfg):
    rb = oracle.GranneBuilder(el, **cfg)
    ref = rb.build_batched(max_batch, threads=THREADS)
    return ref, rb.counters()


def gpu_image(kind, el, emb, **cfg):
    b = gpu_build(kind, el, emb, **cfg)
    image = b.index_bytes().tobytes()
    b.close()
    return image


# ---- A. serialized links: the model's schedule exactly ----------------------------------------------------------
@pytest.mark.parametrize("n,dim,max_batch,largest", [
    (20_000, 24, None, 1250),               # batches grow to present / 16
    (70_000, 16, None, DEFAULT_MAX_BATCH),  # batches of the full 4096
])
def test_serialized_links_equal_the_model(oracle, monkeypatch, n, dim, max_batch, largest):
    _set_knobs(monkeypatch, max_batch, link_warps=1)
    el, emb = _elements(oracle, "angular", n=n, dim=dim, seed=n + dim)
    cfg = dict(num_neighbors=20, max_search=40)
    ref, ctr = model_build(oracle, el, max_batch or DEFAULT_MAX_BATCH, **cfg)
    assert ctr["max_batch"] == largest and ctr["connect_overflow"] > 0, ctr
    assert_same_index(oracle, gpu_image("angular", el, emb, **cfg), ref, el, "n=%d dim=%d" % (n, dim))


@pytest.mark.parametrize("max_batch", [2, 7, 64])
@pytest.mark.parametrize("kind,dim,m", [
    ("angular", 100, 20),
    ("angular_int", 100, 20),
    ("angular_int", 300, 20),
    ("embeddings", 50, 20),
    ("angular", 32, 48),  # rows wider than a warp
])
def test_serialized_links_with_small_batches(oracle, monkeypatch, kind, dim, m, max_batch):
    _set_knobs(monkeypatch, max_batch, link_warps=1)
    n = 2000
    el, emb = _elements(oracle, kind, n=n, dim=dim, seed=dim + m + max_batch)
    cfg = dict(num_neighbors=m, max_search=40)
    ref, ctr = model_build(oracle, el, max_batch, **cfg)
    assert ctr["max_batch"] == max_batch and ctr["connect_overflow"] > 0, ctr
    assert_same_index(oracle, gpu_image(kind, el, emb, **cfg), ref, el,
                      "%s dim=%d M=%d max_batch=%d" % (kind, dim, m, max_batch))


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_serialized_links_zero_rows_and_duplicates_in_one_batch(oracle, monkeypatch, kind):
    # With the default schedule the last layer's insertion batch that starts at node 1266 holds 79 members, so row 1299
    # and its 35 copies at 1300..1334 are inserted together: none sees the others in the snapshot, and the
    # dead-duplicate rule (:826-832) acts differently than in the sequential build, where the later copies see the
    # earlier ones and stay unconnected.
    _set_knobs(monkeypatch, link_warps=1)
    n, m = 3000, 20
    raw = random_vectors(n, 24, seed=17)
    zeros = [100, 777, 1500]
    raw[zeros] = 0.0
    dups = np.arange(1300, 1335)
    raw[dups] = raw[1299]
    el, _ = _elements(oracle, kind, raw=raw)
    cfg = dict(num_neighbors=m, max_search=40)
    ref, ctr = model_build(oracle, el, DEFAULT_MAX_BATCH, **cfg)
    seq = oracle.GranneBuilder(el, **cfg).build(threads=1)
    last = ref.num_layers() - 1
    assert all(ref.get_neighbors(i, last) == [] for i in zeros)
    dead = lambda g: [int(i) for i in dups if g.get_neighbors(int(i), last) == []]
    assert len(dead(seq)) > 0 and dead(ref) != dead(seq), (dead(seq), dead(ref))
    assert_same_index(oracle, gpu_image(kind, el, None, **cfg), ref, el, "%s zero / duplicate rows" % kind)


def test_serialized_links_incremental_build_with_append(oracle, monkeypatch):
    _set_knobs(monkeypatch, 64, link_warps=1)
    n0, n = 1500, 2000
    raw = random_vectors(n, 24, seed=8)
    el = oracle.Elements.angular(raw[:n0])
    cfg = dict(num_neighbors=20, max_search=40, expected_num_elements=n0)
    rb = oracle.GranneBuilder(el, **cfg)
    b = granne_b200.GranneBuilder("angular", el.to_bytes(), **cfg)
    for step in (1, 40, 700, n0):
        ref = rb.build_partial(step, threads=THREADS, max_batch=64)
        b.build(step)
        assert len(b) == step
        assert_same_index(oracle, b.index_bytes().tobytes(), ref, el, "build_partial(%d)" % step)
    el.push(raw[n0:])
    for row in raw[n0:]:
        b.append(row.tolist())
    ref = rb.build_partial(n, threads=THREADS, max_batch=64)
    b.build()
    assert len(b) == n
    ctr = rb.counters()
    assert ctr["max_batch"] == 64 and ctr["connect_overflow"] > 0, ctr
    assert_same_index(oracle, b.index_bytes().tobytes(), ref, el, "append + build")
    b.close()


# ---- B. concurrent links where the result does not depend on their order -----------------------------------------
@pytest.mark.parametrize("kind,n,dim,ef", [
    ("angular", 70_000, 16, 12),
    ("angular_int", 30_000, 12, 10),
    ("embeddings", 20_000, 16, 10),
])
def test_concurrent_links_equal_the_model_without_overflow(oracle, kind, n, dim, ef):
    # M = 255 and a small max_search: no row fills up and every selection keeps all of its candidates, so a row is
    # the set of links made into it.  The precondition is checked on the model, not assumed.
    el, emb = _elements(oracle, kind, n=n, dim=dim, seed=n + dim)
    cfg = dict(num_neighbors=255, max_search=ef)
    ref, ctr = model_build(oracle, el, DEFAULT_MAX_BATCH, **cfg)
    assert ctr["connect_overflow"] == 0 and ctr["nontrivial_selects"] == 0, ctr
    # contention: links already present are re-found, batches are large, hub rows take many links per batch
    assert ctr["connect_present"] > 0 and ctr["max_batch"] >= 1250 and ctr["max_batch_in_links"] >= 6, ctr
    assert_same_index(oracle, gpu_image(kind, el, emb, **cfg), ref, el, "%s concurrent, M=255" % kind)


# ---- C. concurrent links with overflow: invariants of every row --------------------------------------------------
def check_rows(b, el, m, zeros):
    """Every row of every layer: no duplicates, no self-links, ids inside the layer, at most M (max(1, M / 2) on upper
    layers) neighbours, zero elements unconnected, and ascending by distance to the node (the final prune writes every
    row sorted)."""
    nl = b.num_layers()
    for layer in range(nl):
        n = b.layer_len(layer)
        limit = m if layer == nl - 1 else max(1, m // 2)
        for i in range(n):
            nb = b.get_neighbors(i, layer)
            where = "layer %d node %d: %s" % (layer, i, nb)
            assert len(nb) <= limit and len(set(nb)) == len(nb) and i not in nb, where
            assert all(j < n for j in nb), where
            if i in zeros:
                assert nb == [], where
            d = el.dists(i, nb)
            assert np.all(d[:-1] <= d[1:]), "%s not ascending: %s" % (where, d)


def element_recall(b, el, sample, ef):
    """Mean fraction of each sampled element's 10 nearest elements (oracle distances) that a search finds."""
    index = b.get_index()
    q = np.stack([el.get(int(i)) for i in sample])
    ids, _, _ = index.search_batch(q, ef, 10, already_element=True)
    index.close()
    n = len(el)
    hits = 0
    for row, i in zip(ids, sample):
        d = el.dists(int(i), np.arange(n))
        exact = set(np.lexsort((np.arange(n), d))[:10].tolist())
        hits += len(exact & set(row.tolist()))
    return hits / (10.0 * len(sample))


@pytest.mark.parametrize("case", ["angular", "angular_int", "embeddings", "clustered"])
def test_concurrent_build_with_overflow_keeps_row_invariants(oracle, monkeypatch, case):
    zeros = []
    if case == "angular":
        kind, n, m, ef = "angular", 12_000, 20, 40
        el, emb = _elements(oracle, kind, n=n, dim=24, seed=41)
    elif case == "angular_int":
        kind, n, m, ef = "angular_int", 6_000, 30, 200
        el, emb = _elements(oracle, kind, n=n, dim=32, seed=42)
    elif case == "embeddings":
        kind, n, m, ef = "embeddings", 6_000, 30, 40
        el, emb = _elements(oracle, kind, n=n, dim=50, seed=43)
    else:
        # tight clusters: their central nodes are hubs that many members of one batch link to at once
        kind, n, m, ef = "angular", 20_000, 20, 40
        raw = clustered_vectors(n, 32, seed=44, n_centers=16, sub_dim=8, spread=0.05)
        zeros = [5, 4321, 15000]
        raw[zeros] = 0.0
        el, emb = _elements(oracle, kind, raw=raw)
    cfg = dict(num_neighbors=m, max_search=ef)
    b = gpu_build(kind, el, emb, **cfg)
    check_rows(b, el, m, set(zeros))
    sample = [i for i in np.random.default_rng(n).choice(n, 200, replace=False) if i not in zeros]
    recall = element_recall(b, el, sample, 40)
    b.close()
    _set_knobs(monkeypatch, link_warps=1)
    s = gpu_build(kind, el, emb, **cfg)
    serial = element_recall(s, el, sample, 40)
    s.close()
    assert recall >= serial - 0.01, (recall, serial)
