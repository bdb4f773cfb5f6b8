"""GranneBuilder::from_bytes on the GPU (granne_b200_builder_from_index): a builder that continues from an index image.
Every resumed build is held to the oracle's GranneBuilder.from_index (the reference's from_bytes, src/index/mod.rs:
428-461) fed the same image and elements, byte for byte through assert_same_index:

1. Sequential insertion (GRANNE_B200_BUILD_MAX_BATCH=1) against the oracle's threads=1 resume, then build_partial steps:
   num_neighbors reduced (rows cut to their lowest ids) and widened, reinsertion off, expected_num_elements set, and a
   layer_multiplier change under which the loaded last layer is already full and a new layer is cloned from it.
2. Serialized links (GRANNE_B200_BUILD_LINK_WARPS=1) against the oracle's model of the batch schedule.
3. The checkpoint workflow inside the product: build_partial -> index_bytes -> resume, with and without appended
   elements.
4. Loading alone: the image is written back unchanged, searched like Granne.from_bytes, cut like the reference.
5. Device-resident elements give the same builder as an elements image.
6. The default concurrent link phase on a resumed builder: row invariants and recall.
7. Bad input gives statuses and leaves the device usable."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import granne_b200
from helpers.data import random_sum_embeddings, random_vectors
from helpers.fixtures import compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)
from helpers.index_image import assert_same_index

pytestmark = pytest.mark.gpu

THREADS = max(1, min(16, os.cpu_count() or 1))  # the oracle's searches of one batch; its image does not depend on it
INVALID, FORMAT = -1, -2


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


def _elements(oracle, kind, n, dim, seed, raw=None):
    if kind == "embeddings":
        el = random_sum_embeddings(oracle, dim, 200, n, seed)
        return el, el.to_bytes(1)
    raw = random_vectors(n, dim, seed) if raw is None else raw
    return (oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)), None


def oracle_image(oracle, el, n1, **cfg):
    """The oracle's sequential build_partial(n1): the image a resume starts from."""
    return oracle.GranneBuilder(el, **cfg).build_partial(n1, threads=1).to_bytes()


def oracle_resume(oracle, image, el, **cfg):
    return oracle.GranneBuilder.from_index(oracle.Granne.from_bytes(image, el), el, **cfg)


def resume(kind, el, emb, image, **cfg):
    return granne_b200.GranneBuilder(kind, el.to_bytes(0), emb, index_bytes=image, **cfg)


def layer_size(total, multiplier, layer):
    """compute_num_elements_in_layer (src/index/mod.rs:634-643)."""
    e = math.floor(math.log(total) / math.log(multiplier)) - layer
    return min(math.ceil(total / multiplier ** e), total)


def image_of(b):
    return b.index_bytes().tobytes()


# ---- 1. sequential insertion: the reference's resume exactly ------------------------------------------------------
SCENARIOS = {
    # name: (phase-1 config, resumed config, phase-1 length as a function of n)
    "reduce": (dict(num_neighbors=20, max_search=40), dict(num_neighbors=5, max_search=40), lambda n: n // 2),
    "widen": (dict(num_neighbors=10, max_search=40), dict(num_neighbors=30, max_search=40), lambda n: n // 2),
    "no_reinsert": (dict(num_neighbors=20, max_search=40), dict(num_neighbors=12, max_search=30,
                                                                reinsert_elements=False), lambda n: n // 2),
    "expected": (dict(num_neighbors=20, max_search=40, expected_num_elements=6000),
                 dict(num_neighbors=20, max_search=40, expected_num_elements=6000), lambda n: n // 2),
    # layers 9 and 134 loaded; at multiplier 40 their ideal sizes are 2 and 50, so layer 2 is cloned from layer 1
    "multiplier": (dict(num_neighbors=20, max_search=40), dict(num_neighbors=20, max_search=40, layer_multiplier=40.0),
                   lambda n: math.ceil(n / 15)),
}


@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
@pytest.mark.parametrize("kind,dim", [("angular", 24), ("angular", 100), ("angular_int", 100), ("angular_int", 300),
                                      ("embeddings", 50)])
def test_sequential_resume_equals_the_oracle(oracle, monkeypatch, kind, dim, scenario):
    _set_knobs(monkeypatch, max_batch=1)
    n = 2000
    first, second, n1_of = SCENARIOS[scenario]
    n1 = n1_of(n)
    el, emb = _elements(oracle, kind, n, dim, seed=dim + len(scenario))
    image = oracle_image(oracle, el, n1, **first)
    loaded = oracle.Granne.from_bytes(image, el)
    if scenario == "reduce":
        assert max(len(loaded.get_neighbors(i)) for i in range(n1)) > 5
    if scenario == "multiplier":
        last = loaded.num_layers() - 1
        assert loaded.layer_len(last) == n1 and layer_size(n, 40.0, last) <= n1  # already full under the new config
    rb = oracle_resume(oracle, image, el, **second)
    b = resume(kind, el, emb, image, **second)
    assert len(b) == n1 and b.num_layers() == loaded.num_layers()
    what = "%s dim=%d %s" % (kind, dim, scenario)
    for step in (n1 + (n - n1) // 3, n):
        ref = rb.build_partial(step, threads=1)
        b.build(step)
        assert len(b) == step
        assert_same_index(oracle, image_of(b), ref, el, "%s build_partial(%d)" % (what, step))
    if scenario == "multiplier":
        assert ref.num_layers() == loaded.num_layers() + 1
        assert ref.layer_len(loaded.num_layers() - 1) == n1  # left alone
    if scenario == "reduce":
        assert all(len(ref.get_neighbors(i, layer)) <= 5 for layer in range(ref.num_layers())
                   for i in range(ref.layer_len(layer)))
    b.close()


# ---- 2. serialized links: the batch schedule's model exactly ----------------------------------------------------
@pytest.mark.parametrize("kind,dim,n,max_batch", [
    ("angular", 24, 2000, 64),
    ("angular_int", 100, 2000, 64),
    ("embeddings", 50, 2000, 64),
    ("angular", 24, 16_000, None),  # the default schedule: batches grow to present / 16
])
def test_serialized_links_resume_equals_the_model(oracle, monkeypatch, kind, dim, n, max_batch):
    _set_knobs(monkeypatch, max_batch, link_warps=1)
    el, emb = _elements(oracle, kind, n, dim, seed=n + dim)
    image = oracle_image(oracle, el, n // 2, num_neighbors=20, max_search=40)
    cfg = dict(num_neighbors=16, max_search=40)
    rb = oracle_resume(oracle, image, el, **cfg)
    ref = rb.build_partial(n, threads=THREADS, max_batch=max_batch or 4096)
    ctr = rb.counters()
    assert ctr["connect_overflow"] > 0, ctr
    b = resume(kind, el, emb, image, **cfg)
    b.build()
    assert_same_index(oracle, image_of(b), ref, el, "%s n=%d max_batch=%s" % (kind, n, max_batch))
    b.close()


# ---- 3. checkpoint and resume inside the product ----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_checkpoint_and_resume(oracle, monkeypatch, kind):
    _set_knobs(monkeypatch, max_batch=1)
    n, n1 = 2000, 1100
    el, emb = _elements(oracle, kind, n, 32, seed=61)
    cfg = dict(num_neighbors=20, max_search=40)
    first = granne_b200.GranneBuilder(kind, el.to_bytes(0), emb, **cfg)
    first.build(n1)
    checkpoint = image_of(first)
    first.close()
    b = resume(kind, el, emb, checkpoint, **cfg)
    b.build()
    ref = oracle_resume(oracle, checkpoint, el, **cfg).build_partial(n, threads=1)
    assert_same_index(oracle, image_of(b), ref, el, "%s checkpoint at %d" % (kind, n1))
    b.close()


@pytest.mark.parametrize("kind", ["angular", "embeddings"])
def test_resume_then_append(oracle, monkeypatch, kind):
    from granne_b200 import words as W

    _set_knobs(monkeypatch, max_batch=1)
    n0, n = 1500, 2000
    cfg = dict(num_neighbors=20, max_search=40)
    if kind == "angular":
        raw = random_vectors(n, 24, seed=62)
        el, emb = _elements(oracle, kind, n0, 24, seed=0, raw=raw[:n0])
        first_bytes = el.to_bytes(0)
    else:
        el, emb = _elements(oracle, kind, n, 24, seed=62)
        lists = W.read_sum_terms(el.to_bytes(0))
        first_bytes = W.write_sum_terms(lists[:n0])
    first = granne_b200.GranneBuilder(kind, first_bytes, emb, **cfg)
    first.build()
    checkpoint = image_of(first)
    first.close()
    b = granne_b200.GranneBuilder(kind, first_bytes, emb, index_bytes=checkpoint, **cfg)
    assert len(b) == n0
    if kind == "angular":
        rb = oracle_resume(oracle, checkpoint, el, **cfg)
        el.push(raw[n0:])
        for row in raw[n0:]:
            b.append(row.tolist())
    else:
        # the oracle's container already holds the appended term lists: from_index does not look at the element
        # count, so this is the same as pushing them after the resume
        rb = oracle_resume(oracle, checkpoint, el, **cfg)
        for terms in lists[n0:]:
            b.append(terms)
    assert b.num_elements() == n and len(b) == n0
    ref = rb.build_partial(n, threads=1)
    b.build()
    assert len(b) == n
    assert_same_index(oracle, image_of(b), ref, el, "%s resume + append" % kind)
    index = b.get_index()
    assert bytes(index.elements_bytes()) == el.to_bytes(0)
    index.close()
    b.close()


# ---- 4. loading alone -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_loading_writes_the_image_back_and_searches_like_granne(oracle, kind):
    n, dim = 3000, 40
    el, emb = _elements(oracle, kind, n, dim, seed=71)
    image = oracle.GranneBuilder(el, num_neighbors=20, max_search=40).build(threads=THREADS).to_bytes()
    ref = oracle.Granne.from_bytes(image, el)
    widest = max(len(ref.get_neighbors(i)) for i in range(n))
    for m in (widest, 20, 64):
        b = resume(kind, el, emb, image, num_neighbors=m, max_search=40)
        assert image_of(b) == image, "num_neighbors=%d" % m
        if m == widest:
            snap = b.get_index()
        b.close()
    direct = granne_b200.Granne.from_bytes(image, kind, el.to_bytes(0), emb)
    q = random_vectors(256, dim, seed=72)
    want = ref.search_batch(q, 60, 10, with_stats=True)
    for g in (snap, direct):
        got = g.search_batch(q, 60, 10, with_stats=True)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
        assert np.array_equal(got[2], want[2]) and np.array_equal(got[3][:, :3], want[3][:, :3])
    snap.close()
    direct.close()


@pytest.mark.parametrize("m", [1, 5, 11])
def test_loading_with_fewer_neighbours_cuts_rows_like_the_reference(oracle, m):
    n = 3000
    el, _ = _elements(oracle, "angular", n, 24, seed=73)
    image = oracle.GranneBuilder(el, num_neighbors=20, max_search=40).build(threads=THREADS).to_bytes()
    b = resume("angular", el, None, image, num_neighbors=m, max_search=40)
    rb = oracle_resume(oracle, image, el, num_neighbors=m, max_search=40)
    ref = rb.build_partial(n, threads=1)  # everything is indexed: nothing is rebuilt, the rows are only cut
    assert_same_index(oracle, image_of(b), ref, el, "num_neighbors=%d" % m)
    loaded = oracle.Granne.from_bytes(image, el)
    last = loaded.num_layers() - 1
    for i in range(0, n, 97):
        assert b.get_neighbors(i) == loaded.get_neighbors(i, last)[:m]  # the lowest ids, not the nearest
    b.close()


def test_an_image_without_layers_gives_a_new_builder(oracle, monkeypatch):
    _set_knobs(monkeypatch, max_batch=1)
    el, _ = _elements(oracle, "angular", 1500, 24, seed=74)
    empty = granne_b200.GranneBuilder("angular", el.to_bytes(0)).index_bytes().tobytes()
    b = resume("angular", el, None, empty, num_neighbors=20, max_search=40)
    assert len(b) == 0 and b.num_layers() == 0
    b.build()
    ref = oracle.GranneBuilder(el, num_neighbors=20, max_search=40).build(threads=1)
    assert_same_index(oracle, image_of(b), ref, el, "resumed from an empty image")
    b.close()


# ---- 5. device-resident elements ----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_device_elements_resume_like_an_image(oracle, monkeypatch, kind):
    import torch

    _set_knobs(monkeypatch, max_batch=1)
    n = 2000
    el, _ = _elements(oracle, kind, n, 48, seed=75)
    image = oracle_image(oracle, el, 900, num_neighbors=20, max_search=40)
    cfg = dict(num_neighbors=12, max_search=40)
    rows = torch.from_numpy(el.rows()).cuda()
    d = granne_b200.GranneBuilder.from_device_elements(kind, rows, index_bytes=image, **cfg)
    h = resume(kind, el, None, image, **cfg)
    assert image_of(d) == image_of(h)
    d.build()
    h.build()
    assert image_of(d) == image_of(h)
    ref = oracle_resume(oracle, image, el, **cfg).build_partial(n, threads=1)
    assert_same_index(oracle, image_of(d), ref, el, "%s device elements" % kind)
    d.close()
    h.close()


# ---- 6. the default concurrent link phase -------------------------------------------------------------------------
def check_rows(b, el, m, zeros, loaded):
    """Every row of every layer: no duplicates, no self-links, ids inside the layer, at most M (max(1, M / 2) on upper
    layers) neighbours, zero elements unconnected.  A layer that grew was pruned at the end of its build, which writes
    every row ascending by distance to the node; a loaded layer that did not grow keeps its loaded rows."""
    nl = b.num_layers()
    for layer in range(nl):
        n = b.layer_len(layer)
        limit = m if layer == nl - 1 else max(1, m // 2)
        kept = layer < loaded.num_layers() and loaded.layer_len(layer) == n
        for i in range(n):
            nb = b.get_neighbors(i, layer)
            where = "layer %d node %d: %s" % (layer, i, nb)
            if kept:
                assert nb == loaded.get_neighbors(i, layer), where
                continue
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


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_concurrent_resume_keeps_row_invariants(oracle, monkeypatch, kind):
    n, n1, m, ef = 12_000, 6_000, 20, 40
    raw = random_vectors(n, 24, seed=76)
    zeros = [7, 5000, 9000]
    raw[zeros] = 0.0
    el, _ = _elements(oracle, kind, n, 24, seed=0, raw=raw)
    cfg = dict(num_neighbors=m, max_search=ef)
    image = oracle_image(oracle, el, n1, **cfg)
    loaded = oracle.Granne.from_bytes(image, el)
    b = resume(kind, el, None, image, **cfg)
    b.build()
    check_rows(b, el, m, set(zeros), loaded)
    sample = [i for i in np.random.default_rng(n).choice(n, 200, replace=False) if i not in zeros]
    recall = element_recall(b, el, sample, 40)
    b.close()
    _set_knobs(monkeypatch, link_warps=1)
    s = resume(kind, el, None, image, **cfg)
    s.build()
    serial = element_recall(s, el, sample, 40)
    s.close()
    assert recall >= serial - 0.01, (recall, serial)


# ---- 7. errors ----------------------------------------------------------------------------------------------------
def test_errors_are_statuses_and_leave_the_device_usable(oracle):
    import torch

    n = 2000
    el, _ = _elements(oracle, "angular", n, 24, seed=77)
    image = oracle_image(oracle, el, n, num_neighbors=20, max_search=40)
    other = granne_b200.Granne.from_bytes(image, "angular", el.to_bytes(0))
    q = random_vectors(64, 24, seed=78)
    before = other.search_batch(q, 40, 10)

    def status(fn):
        with pytest.raises(granne_b200.GranneError) as ei:
            fn()
        return ei.value.code

    # an index over more elements than the container
    fewer = oracle.Elements.angular(random_vectors(n - 1, 24, seed=77))
    assert status(lambda: resume("angular", fewer, None, image)) == FORMAT
    rows = torch.from_numpy(fewer.rows()).cuda()
    assert status(lambda: granne_b200.GranneBuilder.from_device_elements("angular", rows, index_bytes=image)) == FORMAT
    # a wrong element kind or width
    assert status(lambda: granne_b200.GranneBuilder(99, el.to_bytes(0), index_bytes=image)) == INVALID
    assert status(lambda: granne_b200.GranneBuilder("embeddings", el.to_bytes(0), index_bytes=image)) == INVALID
    i8 = oracle.Elements.angular_int(random_vectors(n, 24, seed=77))
    assert status(lambda: granne_b200.GranneBuilder("angular", i8.to_bytes(0), index_bytes=image)) == FORMAT
    lib = granne_b200.load_library()
    cfg = granne_b200.api._build_config(20, 40, 15.0, True, None)
    ib = np.frombuffer(image, dtype=np.uint8)
    h = C.c_void_p()
    rc = lib.granne_b200_builder_from_index_device_elements(C.byref(cfg), granne_b200.api._ptr(ib), ib.size, 2,
                                                            C.c_void_p(rows.data_ptr()), n - 1, 24, 0, C.byref(h))
    assert rc == INVALID and not h.value
    # build(k) below the loaded length
    b = resume("angular", el, None, image, num_neighbors=20, max_search=40)
    assert status(lambda: b.build(n - 1)) == INVALID
    b.build()
    assert len(b) == n and image_of(b) == image
    b.close()
    after = other.search_batch(q, 40, 10)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1].view(np.uint32), after[1].view(np.uint32))
    other.close()


# ---- the C++ mirror: read_index_reduce_num_neighbors (tests.rs:243-290) ------------------------------------------
def test_cxx_read_index_reduce_num_neighbors(oracle, tmp_path):
    exe = compile_cxx_client("cxx_resume_client.cpp", tmp_path)
    el = oracle.Elements.angular(random_vectors(1000, 5, seed=11))
    (tmp_path / "elements").write_bytes(el.to_bytes(0))
    env = dict(os.environ, GRANNE_B200_BUILD_MAX_BATCH="1")
    r = subprocess.run([exe, "gpu", str(tmp_path)], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and "gpu ok" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    half = oracle.GranneBuilder(el, num_neighbors=20, max_search=10).build_partial(500, threads=1)
    assert_same_index(oracle, (tmp_path / "half.index").read_bytes(), half, el, "build_partial(500)")
    ref = oracle_resume(oracle, half.to_bytes(), el, num_neighbors=5, max_search=10).build_partial(1000, threads=1)
    assert_same_index(oracle, (tmp_path / "resumed.index").read_bytes(), ref, el, "resumed with num_neighbors 5")
