"""The GPU GranneBuilder on every distance engine, byte for byte against the oracle.

build_link_kernel<Dist> and build_prune_kernel<Dist> (build_kernels.cuh) are compiled once per engine that DistDispatch
(granne_b200.cu) can pick, each with its own shared-memory layout (the engine's tiles, then LinkLayout's link scratch)
and its own `dists` under select_neighbors, add_and_limit, the zero-element rule (dist(idx, idx) > 100 eps) and the
dead-duplicate rule.  The search half of a build is the search kernel, checked on every engine elsewhere; this file
holds the link half of every engine to the oracle:

1. Sequential insertion (GRANNE_B200_BUILD_MAX_BATCH=1) against the oracle's threads=1 build, on every engine and at
   each side of its bounds (SEQUENTIAL; test_builder_engines_cpu reads the engine choice from the sources and checks
   that this list reaches all of it): DistF32<FULL> for every compiled FULL, DistF32Generic on staged rows and on direct
   loads, DistI8 on sub-warp groups and on rows wider than 512 bytes (with i32 sums past 2^24), DistSum over several
   128-float passes with elements of 0, 1, 33 and 70 terms.
2. Edge rows (zero, subnormal, norm-underflow and norm-overflow f32 rows; saturated and zero i8 rows; a block of
   duplicates) in the sequential build.  Which rows the zero rule and the dead-duplicate rule leave unconnected is
   asserted on the oracle's index first, so each case is known to take both rules.
3. Serialized links (GRANNE_B200_BUILD_LINK_WARPS=1) against the oracle's model of the batch schedule.
4. The concurrent link phase at the default grid where no row overflows (M = 255): the model's image again.
5. Resume (GranneBuilder.from_bytes) with a num_neighbors that cuts or pads the loaded rows."""
import os

import numpy as np
import pytest

import granne_b200
from helpers.data import (clustered_vectors, edge_i8_rows, edge_raw_f32, random_vectors, varied_sum_embeddings)
from helpers.index_image import assert_same_index

pytestmark = pytest.mark.gpu

DEFAULT_MAX_BATCH = 4096  # the builder's largest insertion batch when GRANNE_B200_BUILD_MAX_BATCH is unset
THREADS = max(1, min(16, os.cpu_count() or 1))  # the model's searches of one batch; its image does not depend on it
HUNDRED_EPS = np.float32(100.0) * np.float32(1.1920929e-07)  # the zero-element and dead-duplicate bound

# 3 layers at n = 1500.  Wide rows: fewer elements, 4 layers at n = 300 (5 at 1200) with halved M above the last.
NARROW = dict(num_neighbors=20, max_search=40)
WIDE = dict(num_neighbors=10, max_search=24, layer_multiplier=5.0)

# kind, dim, n, config, and the engine and layout that serve the rows, as test_builder_engines_cpu derives them from
# the sources: it fails if one of these dims reaches another engine, or if an engine or one side of a bound between two
# layouts has no case here.
SEQUENTIAL = [
    ("angular", 24, 1500, NARROW, ("DistF32<0>", "tail")),
    ("angular", 32, 1500, NARROW, ("DistF32<1>", "no tail")),
    ("angular", 64, 1500, NARROW, ("DistF32<2>", "no tail")),   # lane-permuted rows from here on
    ("angular", 96, 1500, NARROW, ("DistF32<3>", "no tail")),
    ("angular", 128, 1500, NARROW, ("DistF32<4>", "no tail")),  # the production width
    ("angular", 192, 1500, NARROW, ("DistF32<6>", "no tail")),
    ("angular", 256, 1500, NARROW, ("DistF32<8>", "no tail")),
    ("angular", 160, 1500, NARROW, ("DistF32Generic", "staged")),
    ("angular", 175, 1500, NARROW, ("DistF32Generic", "staged")),   # and a tail of 15
    ("angular", 2079, 300, WIDE, ("DistF32Generic", "staged")),     # 64 chunks: the widest staged rows
    ("angular", 2080, 300, WIDE, ("DistF32Generic", "direct")),
    ("angular", 2101, 300, WIDE, ("DistF32Generic", "direct")),     # and a tail
    ("angular_int", 512, 1500, NARROW, ("DistI8", "sub-warp groups")),    # C = 32, one row per warp pass
    ("angular_int", 513, 1500, NARROW, ("DistI8", "one row at a time")),  # C == 0, lanes stride over 32-bit words
    ("angular_int", 1041, 300, WIDE, ("DistI8", "one row at a time")),    # saturated rows' r and dx past 2^24
    ("angular_int", 4096, 300, WIDE, ("DistI8", "one row at a time")),
    ("embeddings", 129, 1000, NARROW, ("DistSum", "several passes")),
    ("embeddings", 300, 1000, NARROW, ("DistSum", "several passes")),
    ("embeddings", 4096, 300, WIDE, ("DistSum", "several passes")),       # 32 passes of 128 floats
]


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


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
    """(oracle elements, embeddings image or None); embeddings have the term lists of varied_sum_embeddings."""
    if kind == "embeddings":
        el = varied_sum_embeddings(oracle, dim, 200, n, seed)
        return el, el.to_bytes(1)
    raw = random_vectors(n, dim, seed) if raw is None else raw
    return (oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)), None


def gpu_image(kind, el, emb, index_bytes=None, **cfg):
    b = granne_b200.GranneBuilder(kind, el.to_bytes(0), emb, index_bytes=index_bytes, **cfg)
    b.build()
    image = b.index_bytes().tobytes()
    b.close()
    return image


def model_build(oracle, el, max_batch, **cfg):
    rb = oracle.GranneBuilder(el, **cfg)
    ref = rb.build_batched(max_batch, threads=THREADS)
    return ref, rb.counters()


def unconnected(ref, i):
    """Node i has no neighbours in any layer that holds it."""
    return all(ref.get_neighbors(i, layer) == [] for layer in range(ref.num_layers()) if i < ref.layer_len(layer))


def zero_rule_rows(el):
    """The elements the builder does not index: dist(idx, idx) > 100 eps (the oracle's distance)."""
    return [i for i in range(len(el)) if el.dists(i, [i])[0] > HUNDRED_EPS]


# ---- 1. sequential insertion on every engine ----------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim,n,cfg,engine", SEQUENTIAL, ids=["%s-%d" % c[:2] for c in SEQUENTIAL])
def test_sequential_build_on_every_engine(oracle, monkeypatch, kind, dim, n, cfg, engine):
    _set_knobs(monkeypatch, max_batch=1)
    el, emb = _elements(oracle, kind, n, dim, seed=dim + n)
    ref = oracle.GranneBuilder(el, **cfg).build(threads=1)
    assert ref.num_layers() >= 2
    if kind == "embeddings":
        lists = [el.terms(i) for i in range(n)]
        # elements without terms are zero vectors the builder skips; the longest term lists are linked
        assert all(unconnected(ref, i) for i in range(n) if not lists[i])
        assert zero_rule_rows(el) == [i for i in range(n) if not lists[i]]
        assert any(len(lists[i]) > 64 and ref.get_neighbors(i) for i in range(n))
        assert any(len(set(l)) < len(l) for l in lists)  # repeated terms
    assert_same_index(oracle, gpu_image(kind, el, emb, **cfg), ref, el, "%s dim=%d (%s, %s)" % ((kind, dim) + engine))


# ---- 2. edge rows -------------------------------------------------------------------------------------------------
def edge_case(kind, n, dim, seed, copies):
    """Random rows with the rows of edge_raw_f32 / edge_i8_rows spread over the first half (the first of them on an
    upper layer) and `copies` duplicates of one random row behind it.  Returns (rows, edge positions, duplicates)."""
    if kind == "angular":
        raw = random_vectors(n, dim, seed)
        edge = edge_raw_f32(12, dim, seed + 1)
    else:
        raw = np.random.default_rng(seed).integers(-127, 128, size=(n, dim)).astype(np.int8)
        edge = edge_i8_rows(8, dim, seed + 1)
    step = (4 * n // 10) // len(edge)
    pos = [n // 20 + k * step for k in range(len(edge))]
    raw[pos] = edge
    d0 = 7 * n // 10
    dups = list(range(d0 + 1, d0 + 1 + copies))
    raw[dups] = raw[d0]
    return raw, pos, dups


@pytest.mark.parametrize("kind,dim,n,cfg,copies", [
    ("angular", 128, 1500, NARROW, 30),
    ("angular", 2101, 300, WIDE, 15),
    ("angular_int", 1041, 300, WIDE, 15),
    ("angular_int", 4096, 300, WIDE, 15),
])
def test_sequential_build_with_edge_rows(oracle, monkeypatch, kind, dim, n, cfg, copies):
    _set_knobs(monkeypatch, max_batch=1)
    raw, pos, dups = edge_case(kind, n, dim, dim, copies)
    el, _ = _elements(oracle, kind, n, dim, 0, raw=raw)  # int8 rows are stored as they are
    ref = oracle.GranneBuilder(el, **cfg).build(threads=1)
    assert ref.num_layers() >= 2 and pos[0] < ref.layer_len(ref.num_layers() - 2)
    if kind == "angular":
        # zero rows, squared norms that underflow (left as they are) or overflow (normalised to +-0), subnormal rows
        zero = [pos[k] for k in (0, 5, 6, 7, 9, 11)]
    else:
        zero = [pos[0], pos[7]]
        # saturated rows are linked; their exact r and dx pass 2^24 and round on the way to f32
        assert 127 * 127 * dim > 2 ** 24 and not any(unconnected(ref, pos[k]) for k in range(1, 7))
    assert zero_rule_rows(el) == zero
    assert all(unconnected(ref, i) for i in zero)
    dead = [i for i in dups if unconnected(ref, i)]
    assert 0 < len(dead) < len(dups), dead  # the first copies are linked, later ones are dead duplicates
    assert_same_index(oracle, gpu_image(kind, el, None, **cfg), ref, el, "%s dim=%d edge rows" % (kind, dim))


# ---- 3. serialized links: the model's batch schedule --------------------------------------------------------------
@pytest.mark.parametrize("max_batch", [7, 64])
@pytest.mark.parametrize("kind,dim,n,cfg", [
    ("angular", 128, 1500, NARROW),
    ("angular", 2101, 1200, WIDE),
    ("angular_int", 513, 1500, NARROW),
    ("angular_int", 1041, 1200, WIDE),
    ("embeddings", 300, 1500, NARROW),
])
def test_serialized_links_on_wide_engines(oracle, monkeypatch, kind, dim, n, cfg, max_batch):
    _set_knobs(monkeypatch, max_batch, link_warps=1)
    el, emb = _elements(oracle, kind, n, dim, seed=dim + max_batch)
    ref, ctr = model_build(oracle, el, max_batch, **cfg)
    assert ref.num_layers() >= 2
    assert ctr["max_batch"] == max_batch and ctr["connect_overflow"] > 0, ctr
    assert_same_index(oracle, gpu_image(kind, el, emb, **cfg), ref, el,
                      "%s dim=%d max_batch=%d" % (kind, dim, max_batch))


# ---- 4. concurrent links without overflow -------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim,ef", [("angular", 128, 12), ("angular_int", 513, 10)])
def test_concurrent_links_on_wide_engines_without_overflow(oracle, kind, dim, ef):
    # M = 255 and a small max_search: no row fills up and every selection keeps all of its candidates, so a row is the
    # set of links made into it whatever the order.  Random i8 rows of 513 dims make hubs that overflow; rows on a
    # 16-dimensional subspace do not.
    n = 20_000
    raw = random_vectors(n, dim, n + dim) if kind == "angular" else \
        clustered_vectors(n, dim, seed=5, n_centers=8, sub_dim=16, spread=1.0)
    el, _ = _elements(oracle, kind, n, dim, 0, raw=raw)
    cfg = dict(num_neighbors=255, max_search=ef)
    ref, ctr = model_build(oracle, el, DEFAULT_MAX_BATCH, **cfg)
    assert ctr["connect_overflow"] == 0 and ctr["nontrivial_selects"] == 0, ctr
    # contention: links already present are re-found, batches are large, hub rows take many links per batch
    assert ctr["connect_present"] > 0 and ctr["max_batch"] >= 1250 and ctr["max_batch_in_links"] >= 6, ctr
    assert_same_index(oracle, gpu_image(kind, el, None, **cfg), ref, el, "%s dim=%d concurrent, M=255" % (kind, dim))


# ---- 5. resume ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first,second", [(20, 8), (10, 24)], ids=["cut", "pad"])
@pytest.mark.parametrize("kind,dim", [("angular", 128), ("angular_int", 513), ("embeddings", 300)])
def test_sequential_resume_on_wide_engines(oracle, monkeypatch, kind, dim, first, second):
    _set_knobs(monkeypatch, max_batch=1)
    n, n1 = 1500, 700
    el, emb = _elements(oracle, kind, n, dim, seed=dim + first)
    image = oracle.GranneBuilder(el, num_neighbors=first, max_search=40).build_partial(n1, threads=1).to_bytes()
    loaded = oracle.Granne.from_bytes(image, el)
    assert loaded.num_layers() >= 2
    widest = max(len(loaded.get_neighbors(i)) for i in range(n1))
    assert widest > second if second < first else widest == first  # rows are cut, or padded with free slots
    cfg = dict(num_neighbors=second, max_search=40)
    rb = oracle.GranneBuilder.from_index(loaded, el, **cfg)
    b = granne_b200.GranneBuilder(kind, el.to_bytes(0), emb, index_bytes=image, **cfg)
    assert len(b) == n1
    for step in (n1 + (n - n1) // 3, n):
        ref = rb.build_partial(step, threads=1)
        b.build(step)
        assert len(b) == step
        assert_same_index(oracle, b.index_bytes().tobytes(), ref, el,
                          "%s dim=%d M %d -> %d, build_partial(%d)" % (kind, dim, first, second, step))
    b.close()
