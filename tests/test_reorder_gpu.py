"""Granne::reorder / reorder_by_keys through the C ABI on the GPU (src/index/reorder.rs): the order is computed by the
search kernel (one max_search = 1 single-layer search per trail layer) and must equal the oracle's order exactly."""
import numpy as np
import pytest

import granne_b200
from helpers.data import build_fixture, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


def _assert_same_results(ref, got):
    assert np.array_equal(ref[2], got[2]) and np.array_equal(ref[0], got[0])
    assert np.array_equal(ref[1].view(np.uint32), got[1].view(np.uint32))
    assert np.array_equal(ref[3][:, :3], got[3][:, :3])


@pytest.mark.parametrize("kind,n,dim,mult", [("angular", 5000, 5, 5.0), ("angular", 4000, 128, 15.0),
                                             ("angular_int", 3000, 20, 8.0), ("embeddings", 1500, 12, 6.0)])
def test_compute_order_matches_the_oracle(oracle, kind, n, dim, mult):
    el, g, ib, eb, mb = build_fixture(oracle, kind, n, dim, seed=n + 7, num_neighbors=12, max_search=5 if dim == 5 else 20,
                                      layer_multiplier=mult)
    p = granne_b200.Granne.from_bytes(ib, kind, eb, mb)
    launches = p.launch_count()
    order = p.compute_order()
    assert p.launch_count() > launches                                       # the trails came from the search kernel
    assert np.array_equal(order, g.compute_order(threads=4))
    # the handle still searches the original graph afterwards
    q = random_vectors(50, dim, seed=3)
    _assert_same_results(g.search_batch(q, 20, 5, with_stats=True), p.search_batch(q, 20, 5, with_stats=True))
    p.close()


def test_reorder_index_like_the_reference(oracle):
    # reorder_index (reorder.rs:298-323): 5000 x 5, max_search 5, layer_multiplier 5; results map through the order
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 5000, 5, seed=1, num_neighbors=30, max_search=5,
                                     layer_multiplier=5.0)
    index = granne_b200.Granne.from_bytes(ib, "angular", eb)
    reordered = granne_b200.Granne.from_bytes(ib, "angular", eb)
    permutation = np.array(reordered.reorder(False))
    assert sorted(permutation.tolist()) == list(range(5000))
    for idx in (0, 10, 123, 99, 499):
        element = index.get_element(idx)
        exp = index.search_batch(element[None, :], 10, 10, already_element=True)
        res = reordered.search_batch(element[None, :], 10, 10, already_element=True)
        c = int(exp[2][0])
        assert c == int(res[2][0]) == 10
        assert np.array_equal(exp[0][0, :c], permutation[res[0][0, :c]])
        assert np.array_equal(exp[1].view(np.uint32), res[1].view(np.uint32))
    # the reordered product index is the oracle's reordered index, bit for bit in every search
    ref = oracle.Granne.from_bytes(ib, oracle.Elements.from_bytes("angular", eb))
    assert np.array_equal(ref.reorder(), permutation)
    q = random_vectors(200, 5, seed=8)
    _assert_same_results(ref.search_batch(q, 30, 10, with_stats=True), reordered.search_batch(q, 30, 10, with_stats=True))
    for i in (0, 77, 4999):
        assert np.array_equal(reordered.get_element(i), index.get_element(int(permutation[i])))
        assert reordered.get_neighbors(i) == ref.get_neighbors(i)
    index.close()
    reordered.close()


def test_reorder_by_keys_sum_embeddings(oracle, tmp_path):
    # reorder_sum_embeddings (embeddings/reorder.rs:79-102), through files like the Python class
    el, g, ib, eb, mb = build_fixture(oracle, "embeddings", 500, 5, seed=6, num_neighbors=30, max_search=5,
                                      layer_multiplier=5.0, num_embeddings=277)
    paths = [str(tmp_path / name) for name in ("index.granne", "elements.bin", "embeddings.bin")]
    for path, data in zip(paths, (ib, eb, mb)):
        with open(path, "wb") as f:
            f.write(data)
    reordered = granne_b200.Granne(paths[0], "embeddings", paths[1], paths[2])
    keys = granne_b200.compute_keys_for_reordering(eb, mb)
    permutation = np.array(reordered.reorder_by_keys(keys))
    ref = oracle.Granne.from_bytes(ib, oracle.Elements.from_bytes("embeddings", eb, mb))
    assert np.array_equal(ref.reorder_by_keys(keys), permutation)
    queries = np.stack([el.get(i) for i in (0, 10, 123, 99, 499)])
    exp = g.search_batch(queries, 10, 10, already_element=True, with_stats=True)
    res = reordered.search_batch(queries, 10, 10, already_element=True, with_stats=True)
    for qi in range(5):
        assert np.array_equal(exp[0][qi], permutation[res[0][qi]])
    _assert_same_results(ref.search_batch(queries, 10, 10, already_element=True, with_stats=True), res)
    out = str(tmp_path / "reordered.granne")
    reordered.save_index(out)
    assert open(out, "rb").read() == ref.to_bytes()
    reordered.close()
