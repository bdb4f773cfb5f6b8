"""compute_distance (py/src/lib.rs:71-89) through the C ABI: Vector::from(a).dist(&Vector::from(b)) for raw f32
vectors, bit-identical to the oracle's angular (angular.rs:55-74) and angular_int (angular_int.rs:19-59) distances."""
import numpy as np
import pytest

import granne_b200
from helpers.data import random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


def _oracle_pairs(oracle, kind, a, b):
    out = np.empty(a.shape[0], dtype=np.float32)
    for i in range(a.shape[0]):
        if kind == "angular":
            out[i] = oracle.dist_f32(oracle.normalize_f32(a[i]), oracle.normalize_f32(b[i]))
        else:
            out[i] = oracle.dist_i8(oracle.quantize_i8(a[i]), oracle.quantize_i8(b[i]))
    return out


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
@pytest.mark.parametrize("dim", [1, 3, 25, 32, 33, 64, 100, 128, 160, 200, 256, 300, 1000])
def test_pairwise_distances_are_bit_identical(oracle, kind, dim):
    n = 200
    a, b = random_vectors(n, dim, seed=dim), random_vectors(n, dim, seed=dim + 1)
    a[0], b[0] = 0.0, b[1]                   # zero vector: normalise leaves zeros / i8 norm 0 -> NaN -> r = 0
    a[1] = b[1]                              # identical
    a[2] = -b[2]                             # opposite
    a[3] = b[3] * 1e-3                       # same direction, different scale
    got = granne_b200.compute_distances(kind, a, b)
    want = _oracle_pairs(oracle, kind, a, b)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert abs(float(got[1])) < 1e-5 and abs(float(got[2]) - 2.0) < 1e-5     # angular.rs:112-126
    assert granne_b200.compute_distance(kind, a[5], b[5]) == float(want[5])


def test_nan_is_an_error_like_the_reference_panic():
    a, b = random_vectors(4, 16, seed=1), random_vectors(4, 16, seed=2)
    a[2, 3] = np.nan
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.compute_distances("angular", a, b)
    assert ei.value.code == -6                                               # NotNan panic, angular.rs:70
    with pytest.raises(ValueError):
        granne_b200.compute_distance("embeddings", a[0], b[0])               # "Unsupported element type"


def test_embeddings_class_distances(oracle, tmp_path):
    # Embeddings.dist / dists (py/src/embeddings.rs:78-95): angular distance of the normalised sums
    emb = random_vectors(60, 20, seed=9)
    e = granne_b200.Embeddings()
    for i, row in enumerate(emb):
        e.append(row.tolist(), "w%d" % i)

    def want(l, r):
        a = oracle.normalize_f32(np.asarray(e.get_embedding(l), dtype=np.float32))
        b = oracle.normalize_f32(np.asarray(e.get_embedding(r), dtype=np.float32))
        return float(oracle.dist_f32(a, b))

    assert e.dist("w1 w2 w3", [4, 5]) == want("w1 w2 w3", [4, 5])
    rights = ["w7", [8, 9, 10], 11, "w1 w2 w3"]
    assert e.dists("w1 w2 w3", rights) == [want("w1 w2 w3", r) for r in rights]
    assert abs(e.dist(3, 3)) < 1e-5 and e.dists(0, []) == []


def test_string_queries_on_an_embeddings_index(oracle, tmp_path):
    # WordEmbeddingsGranne (py/src/variants/index.rs:41-139): str query -> word ids -> create_embedding -> search
    from helpers.data import build_fixture

    el, g, ib, eb, mb = build_fixture(oracle, "embeddings", 400, 16, seed=12, num_neighbors=10, max_search=30,
                                      num_embeddings=90)
    paths = {k: str(tmp_path / k) for k in ("index", "elements", "embeddings", "words")}
    for k, data in (("index", ib), ("elements", eb), ("embeddings", mb)):
        with open(paths[k], "wb") as f:
            f.write(data)
    d = granne_b200.WordDict()
    for i in range(90):
        d.push("tok%d" % i)
    d.write(paths["words"])
    index = granne_b200.Granne(paths["index"], "embeddings", paths["elements"], paths["embeddings"], paths["words"])
    assert index.get_internal_element(5) == " ".join("tok%d" % t for t in el.terms(5))
    query = "tok3 tok4 missing tok5"
    vec = np.asarray(granne_b200.Embeddings(paths["embeddings"], paths["words"]).get_embedding(query), dtype=np.float32)
    got = index.search(query, 30, 8)
    assert got == index.search(vec, 30, 8)
    ref = g.search_batch(vec[None, :], 30, 8)
    assert [i for i, _ in got] == ref[0][0, :len(got)].tolist()
    assert np.array_equal(np.array([x for _, x in got], dtype=np.float32).view(np.uint32), ref[1][0, :len(got)].view(np.uint32))
    # element 3 = ids 3..7 (test_helper::random_sum_embeddings): its own words find it at distance ~0
    own = index.search(index.get_internal_element(3), 30, 1)
    assert own[0][0] == 3 and own[0][1] < 1e-5
    # reorder for this type = reorder_by_keys(compute_keys_for_reordering) (py/src/variants/index.rs:70-75)
    order = np.array(index.reorder())
    keys = el.reorder_keys()
    assert np.array_equal(order, g.order_by_keys(keys))
    again = index.search(query, 30, 8)
    assert [int(order[i]) for i, _ in again] == [i for i, _ in got]
    assert index.get_internal_element(0) == " ".join("tok%d" % t for t in el.terms(int(order[0])))
    index.close()
