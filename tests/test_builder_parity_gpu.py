"""GPU GranneBuilder under sequential insertion (GRANNE_B200_BUILD_MAX_BATCH=1): every insertion sees all earlier
links, so the build is the reference's `singlethreaded` one (src/index/mod.rs:645-960) and its index image must equal
the oracle's threads=1 build byte for byte.  This checks select_neighbors, initialize_node, connect_nodes,
add_and_limit_neighbors, the final prune pass, the zero-element skip (:813), the dead duplicate rule (:826-832), half M
on upper layers (:665-668) and half max_search when reinserting (:698-699) exactly, not through recall.

The default batched build is checked against the oracle's model of the batch schedule in test_builder_batched_gpu.py."""
import numpy as np
import pytest

import granne_b200
from helpers.data import random_sum_embeddings, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)
from helpers.index_image import assert_same_index

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _sequential(monkeypatch):
    monkeypatch.setenv("GRANNE_B200_BUILD_MAX_BATCH", "1")  # read by the library on every build call


def build_both(oracle, kind, el, emb_bytes=None, **cfg):
    ref = oracle.GranneBuilder(el, **cfg).build(threads=1)
    b = granne_b200.GranneBuilder(kind, el.to_bytes(0), emb_bytes, **cfg)
    b.build()
    image = b.index_bytes().tobytes()
    b.close()
    return image, ref


def _elements(oracle, kind, n, dim, seed):
    if kind == "embeddings":
        el = random_sum_embeddings(oracle, dim, 200, n, seed)
        return el, el.to_bytes(1)
    raw = random_vectors(n, dim, seed)
    return (oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)), None


@pytest.mark.parametrize("kind,dim,n", [
    ("angular", 24, 2000),       # DistF32<0> (tail only)
    ("angular", 100, 1500),      # DistF32<3> + tail of 4
    ("angular", 300, 1500),      # DistF32Generic, staged rows
    ("angular_int", 100, 2000),
    ("angular_int", 300, 1500),  # i8 rows of 257..512 bytes
    ("embeddings", 50, 2000),
])
def test_sequential_build_equals_the_oracle(oracle, kind, dim, n):
    el, emb = _elements(oracle, kind, n, dim, seed=dim + n)
    image, ref = build_both(oracle, kind, el, emb, num_neighbors=20, max_search=40)
    assert ref.num_layers() > 2
    assert_same_index(oracle, image, ref, el, "%s dim=%d" % (kind, dim))


@pytest.mark.parametrize("m,n", [(48, 2500), (1, 1500), (3, 1500)])
def test_sequential_build_neighbour_counts(oracle, m, n):
    # M=48: rows wider than a warp (24 on upper layers); M=1 and 3: max(1, M / 2) on upper layers
    el = oracle.Elements.angular(random_vectors(n, 32, seed=m))
    image, ref = build_both(oracle, "angular", el, num_neighbors=m, max_search=40)
    assert ref.num_layers() > 2
    if m == 48:
        assert max(len(ref.get_neighbors(i)) for i in range(n)) > 32
    assert_same_index(oracle, image, ref, el, "M=%d" % m)


def test_sequential_build_without_reinsertion(oracle):
    el = oracle.Elements.angular(random_vectors(2000, 24, seed=5))
    image, ref = build_both(oracle, "angular", el, num_neighbors=20, max_search=40, reinsert_elements=False)
    assert ref.num_layers() > 2
    assert_same_index(oracle, image, ref, el, "no reinsertion")


def test_sequential_build_with_many_layers(oracle):
    el = oracle.Elements.angular(random_vectors(2500, 24, seed=6))
    image, ref = build_both(oracle, "angular", el, num_neighbors=20, max_search=40, layer_multiplier=4.0)
    assert ref.num_layers() > 4
    assert_same_index(oracle, image, ref, el, "layer_multiplier=4")


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_sequential_build_skips_zero_and_dead_elements(oracle, kind):
    # zero elements are not indexed (dist(idx, idx) > 100 eps, :812-815); an element that is a duplicate of more than
    # M / 2 of its selected neighbours stays unconnected (:826-832).  Both leave an empty neighbour list.
    n, m = 2000, 20
    raw = random_vectors(n, 24, seed=7)
    zeros = [100, 777, 1500]
    raw[zeros] = 0.0
    dups = np.arange(300, 335)  # 35 copies of one row, more than M / 2 + 1
    raw[dups] = raw[299]
    el = oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)
    image, ref = build_both(oracle, kind, el, num_neighbors=m, max_search=40)
    assert ref.num_layers() > 2
    last = ref.num_layers() - 1
    assert all(ref.get_neighbors(i, last) == [] for i in zeros)
    dead = [int(i) for i in dups if ref.get_neighbors(int(i), last) == []]
    assert len(dead) > 0 and len(dead) < dups.size  # the first copies are connected, the later ones are dead
    assert_same_index(oracle, image, ref, el, "%s zero / duplicate rows" % kind)


def test_sequential_incremental_build_with_append(oracle):
    # build_partial steps with expected_num_elements (:374-402), then elements pushed and indexed by a later build
    n0, n = 1500, 2000
    raw = random_vectors(n, 24, seed=8)
    el = oracle.Elements.angular(raw[:n0])
    cfg = dict(num_neighbors=20, max_search=40, expected_num_elements=n0)
    rb = oracle.GranneBuilder(el, **cfg)
    b = granne_b200.GranneBuilder("angular", el.to_bytes(), **cfg)
    for step in (1, 40, 700, n0):
        ref = rb.build_partial(step, threads=1)
        b.build(step)
        assert len(b) == step
        assert_same_index(oracle, b.index_bytes().tobytes(), ref, el, "build_partial(%d)" % step)
    assert ref.num_layers() > 2
    el.push(raw[n0:])
    for row in raw[n0:]:
        b.append(row.tolist())
    ref = rb.build_partial(n, threads=1)
    b.build()
    assert len(b) == n
    assert_same_index(oracle, b.index_bytes().tobytes(), ref, el, "append + build")
    b.close()
