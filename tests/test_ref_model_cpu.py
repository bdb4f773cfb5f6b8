"""The NumPy model of the reference (tests/helpers/ref_model.py) against the CPU oracle, bit for bit, and against
float64, within a derived error bound: element arithmetic at its edges, exact ranking, and the search loop with its
counters on the golden fixtures, oracle-built indexes of each kind and several-layer indexes from explicit lists.

The model and the oracle were written separately from the reference; where they disagree the reference decides."""
import os
from fractions import Fraction

import numpy as np
import pytest

from helpers import composed_oracle as co
from helpers import ref_model as M
from helpers.data import edge_i8_rows, edge_raw_f32, index_from_lists, random_sum_embeddings, random_vectors
from helpers.fixtures import elements_image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U32 = np.uint32


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(U32)


# ---- the exact FMA ---------------------------------------------------------------------------------------------------
def _f32_round(fr):
    """Fraction -> float32, round to nearest, ties to even, by comparing the candidates around float(fr); +-inf stands
    for +-2^128, where IEEE rounding puts it."""
    with np.errstate(over="ignore"):
        c = np.float32(float(fr))
        cands = {c, np.nextafter(c, np.float32(np.inf)), np.nextafter(c, np.float32(-np.inf))}

    def value(x):
        return Fraction(float(x)) if np.isfinite(x) else Fraction(2 ** 128) * (1 if x > 0 else -1)

    best = min(abs(value(x) - fr) for x in cands)
    near = [x for x in cands if abs(value(x) - fr) == best]
    return min(near, key=lambda x: int(np.float32(x).view(U32)) & 1)  # a tie: the even significand


P = lambda e: np.float32(2.0 ** e)  # noqa: E731

# (a, b, c) whose float64 sum a*b + c lands exactly on a float32 rounding midpoint while the true sum does not: a
# plain float64 multiply-add rounds these to the wrong neighbour
DOUBLE_ROUNDING = [
    (1 + P(-12), 1 + P(-12), P(-80)),              # 1 + 2^-11 + 2^-24 + 2^-80: up, not to the even 1 + 2^-11
    (-(1 + P(-12)), 1 + P(-12), -P(-80)),          # the same, negative
    (P(-75) * (1 + P(-23)), P(-75) * (1 - P(-23)), P(-127) + P(-149)),  # subnormal: just below a midpoint, down to
]                                                                         # the odd 2^-127 + 2^-149
# near midpoints, at the top of the range and among subnormals, and exactly on them (ties to even)
NEAR_MIDPOINTS = [
    (1 + P(-12), 1 + P(-12), -P(-80)),
    (P(-75) * (1 + P(-23)), P(-75) * (1 + P(-23)), P(-127)),
    (np.float32(3.4028235e38), np.float32(1.0), P(103) * (1 - P(-24))),  # just below FLT_MAX + half an ulp: finite
    (np.float32(3.4028235e38), np.float32(1.0), P(103) * (1 + P(-23))),  # just above: +inf
    (P(0), P(0), P(-24)),
    (P(-149), P(-1), P(-149)),                      # 1.5 * 2^-149: ties to even (2^-148)
]


def _fma_exact(a, b, c):
    return _f32_round(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


@pytest.mark.parametrize("a,b,c", DOUBLE_ROUNDING + NEAR_MIDPOINTS)
def test_fma_at_rounding_midpoints(a, b, c):
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    assert _bits(M.fma_f32(a, b, c)) == _bits(_fma_exact(a, b, c))


@pytest.mark.parametrize("a,b,c", DOUBLE_ROUNDING)
def test_fma_cases_that_defeat_double_rounding(a, b, c):
    # these test the fix-up, not luck: a float64 multiply-add rounded to float32 gets them wrong
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    naive = np.float32(np.float64(a) * np.float64(b) + np.float64(c))
    assert _bits(naive) != _bits(_fma_exact(a, b, c))


def test_fma_random_against_fractions():
    rng = np.random.default_rng(7)
    n = 3000
    scale = lambda: np.float32(2.0) ** rng.integers(-140, 60, n).astype(np.float32)  # noqa: E731
    a = (rng.standard_normal(n).astype(np.float32) * scale()).astype(np.float32)
    b = (rng.standard_normal(n).astype(np.float32) * scale()).astype(np.float32)
    c = np.where(rng.random(n) < 0.5, -(a * b), rng.standard_normal(n) * scale()).astype(np.float32)
    c = np.nextafter(c, rng.choice([-np.inf, np.inf], n).astype(np.float32))  # near-cancellation
    got = M.fma_f32(a, b, c)
    for i in range(n):
        fr = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        if abs(fr) >= Fraction(2) ** 128:
            continue
        assert _bits(got[i]) == _bits(_f32_round(fr)), (a[i], b[i], c[i])


# ---- element arithmetic against the oracle ---------------------------------------------------------------------------
WIDTHS = [1, 31, 32, 33, 64, 100, 1041, 2101]


@pytest.mark.parametrize("dim", WIDTHS)
def test_dot_normalize_quantize(oracle, dim):
    raw = edge_raw_f32(24, dim, dim)
    nrm, q = M.normalize_f32(raw), M.quantize(raw)
    for i in range(raw.shape[0]):
        assert _bits(M.dot_f32(raw[i], raw[(i + 1) % 24])) == _bits(oracle.dot_product_f32(raw[i], raw[(i + 1) % 24]))
        assert np.array_equal(_bits(nrm[i]), _bits(oracle.normalize_f32(raw[i]))), "row %d" % i
        assert np.array_equal(q[i], oracle.quantize_i8(raw[i])), "row %d" % i


@pytest.mark.parametrize("dim", WIDTHS + [4096])
def test_f32_distance_including_unnormalised_rows(oracle, dim):
    x = M.normalize_f32(edge_raw_f32(16, dim, dim + 3))
    y = np.concatenate([x[:8], (x[8:] * np.float32(1.5)).astype(np.float32)])  # r > 1 clamps at 0
    d = M.dist_f32(x[:, None, :], y[None, :, :])
    for i in range(16):
        for j in range(16):
            assert _bits(d[i, j]) == _bits(oracle.dist_f32(x[i], y[j])), (i, j)


@pytest.mark.parametrize("dim", [1, 33, 1040, 1041, 4096, 16384])
def test_i8_sums_and_distance_past_2_24(oracle, dim):
    x = edge_i8_rows(10, dim, dim)
    d = M.distances("angular_int", x, x)
    for i in range(10):
        for j in range(10):
            r = M.r_dx_dy_i8(x[i], x[j])
            assert tuple(int(v) for v in r) == oracle.dot_i8(x[i], x[j])
            assert _bits(d[j, i]) == _bits(oracle.dist_i8(x[i], x[j])), (i, j)
    if dim > 1040:
        assert int(M.r_dx_dy_i8(x[1], x[1])[0]) > 2 ** 24


def test_sum_embeddings_rows(oracle):
    table = edge_raw_f32(40, 50, 3)
    table[6] = 0  # keep the sums finite
    terms = [[], [5], [5, 5, 5], [1, 2], list(range(40)) * 3, [3, 4, 7], [0, 0], [8, 9, 10, 11]]
    el = oracle.Elements.sum_embeddings(table, terms)
    want = np.stack([el.get(i) for i in range(len(terms))])
    assert np.array_equal(_bits(M.sum_elements(table, terms)), _bits(want))
    for t in terms[1:]:
        x = table[t[0]].copy()
        for u in t[1:]:
            x = oracle.sum_into_f32(x, table[u])
        assert np.array_equal(_bits(M.sum_embedding(table, t)), _bits(x))


# ---- float64 bound ---------------------------------------------------------------------------------------------------
def f32_distance_bound(x, y):
    """|model - true| for dist_f32(x, y): each of the dim//32 + 32 + dim%32 roundings of the dot product contributes
    at most 2^-24 of sum |x_i y_i| (one per step of the longest chain, (dim + 64) bounds them all), plus one rounding of
    1 - r.  Returns (true distance in float64, bound)."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    dim = x.shape[-1]
    exact = np.maximum(0.0, 1.0 - (x * y).sum(-1))
    return exact, (dim + 64) * 2.0 ** -24 * np.abs(x * y).sum(-1) + 2.0 ** -24


@pytest.mark.parametrize("dim", [1, 33, 2101, 16384])
def test_f32_distance_within_float64_bound(dim):
    x = M.normalize_f32(random_vectors(40, dim, dim))
    d = M.dist_f32(x[:, None, :], x[None, :, :]).astype(np.float64)
    exact, bound = f32_distance_bound(x[:, None, :], x[None, :, :])
    assert (np.abs(d - exact) <= bound).all()


# ---- exact ranking ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_exact_ranking(kind):
    raw = edge_raw_f32(300, 33, 5)
    rows = M.element_rows(kind, raw)
    rows[40:60] = rows[10]  # ties broken by id
    q = M.element_rows(kind, random_vectors(12, 33, 6))
    q[0] = rows[10]
    c = co.Container(kind, elements_image(rows))
    d = M.distances(kind, rows, q)
    for k in (1, 10, 64, 400):
        want = c.exact_search(q, k, already_element=True)
        got = M.as_arrays([M.rank_prefix(d[i], len(rows), k) for i in range(len(q))], k)
        assert np.array_equal(got[0], want[0]) and np.array_equal(_bits(got[1]), _bits(want[1]))
        assert np.array_equal(got[2], want[2])


# ---- search ----------------------------------------------------------------------------------------------------------
def adjacency(g):
    """Neighbour lists of every layer of an oracle index, top layer first: the arguments of the model's search."""
    return [[g.get_neighbors(i, layer) for i in range(g.layer_len(layer))] for layer in range(g.num_layers())]


def model_rows(kind, el, n):
    """The model's element rows for an oracle container: the stored rows, or the normalised sums of SumEmbeddings."""
    if kind == "embeddings":
        return M.sum_elements(el.rows(), [el.terms(i) for i in range(n)])
    return el.rows()[:n]


def model_search(layers, d, max_search, k):
    out = [M.search(layers, d[i], max_search, k) for i in range(d.shape[0])]
    ids, dists, counts = M.as_arrays([o[0] for o in out], k)
    return ids, dists, counts, np.array([o[1] for o in out], dtype=np.uint64).reshape(-1, 3)


def assert_same_search(got, want, what=""):
    assert np.array_equal(got[2], want[2]), what + ": counts"
    for q in range(len(got[2])):
        c = int(got[2][q])
        assert got[0][q, :c].tolist() == want[0][q, :c].tolist(), "%s: query %d ids" % (what, q)
        assert _bits(got[1][q, :c]).tolist() == _bits(want[1][q, :c]).tolist(), "%s: query %d dists" % (what, q)
    assert np.array_equal(np.asarray(got[3])[:, :3], np.asarray(want[3])[:, :3]), what + ": stats"


@pytest.mark.parametrize("name", ["angular_2000x32_m10", "angular_int_800x100_m20", "embeddings_600x20_m16"])
def test_search_reproduces_golden(oracle, name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    kind = str(z["kind"])
    el = oracle.Elements.from_bytes(kind, z["elements"].tobytes(), z["embeddings"].tobytes() if kind == "embeddings"
                                    else None)
    g = oracle.Granne.from_bytes(z["index"].tobytes(), el)
    layers = adjacency(g)
    d = M.distances(kind, model_rows(kind, el, len(layers[-1])), M.element_rows(kind, z["queries"]))
    got = model_search(layers, d, int(z["max_search"]), int(z["k"]))
    assert_same_search(got, (z["ids"], z["dists"], z["counts"], z["stats"]), name)


@pytest.mark.parametrize("kind,dim", [("angular", 33), ("angular", 100), ("angular_int", 40), ("embeddings", 24)])
def test_search_on_oracle_built_indexes(oracle, kind, dim):
    from helpers.data import build_fixture

    el, g, ib, eb, mb = build_fixture(oracle, kind, 700, dim, seed=dim, num_neighbors=12, max_search=30,
                                      layer_multiplier=6.0)
    layers = adjacency(g)
    assert len(layers) >= 3
    raw = random_vectors(40, dim, dim + 1)
    d = M.distances(kind, model_rows(kind, el, len(layers[-1])), M.element_rows(kind, raw))
    for ef, k in ((1, 1), (8, 5), (30, 10), (200, 50)):
        want = g.search_batch(raw, ef, k, with_stats=True)
        assert_same_search(model_search(layers, d, ef, k), want, "%s ef=%d k=%d" % (kind, ef, k))


def _lists_index(n, seed, degree, layer_lens):
    rng = np.random.default_rng(seed)
    layers = []
    for m in layer_lens:
        layers.append([sorted(set(rng.integers(0, m, size=min(degree, m)).tolist()) - {i}) or [(i + 1) % m]
                       for i in range(m)])
    return layers


@pytest.mark.parametrize("kind", ["angular", "angular_int"])
def test_search_on_several_layer_lists_with_ties(oracle, kind):
    n, dim = 500, 33
    raw = edge_raw_f32(n, dim, 9)
    raw[100:200] = raw[50]  # a plateau of equal distances: the (dist, id) orders decide
    el = oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw[:, :])
    layers = _lists_index(n, 3, 9, [3, 25, 140, n])
    g = oracle.Granne.from_bytes(index_from_lists(oracle, layers), el)
    assert adjacency(g) == [[sorted(l) for l in layer] for layer in layers]
    q = np.concatenate([random_vectors(20, dim, 4), raw[[50, 0, 5]]])
    d = M.distances(kind, el.rows(), M.element_rows(kind, q))
    for ef, k in ((1, 1), (10, 10), (64, 20), (600, 600)):
        want = g.search_batch(q, ef, k, with_stats=True)
        assert_same_search(model_search(layers, d, ef, k), want, "%s ef=%d k=%d" % (kind, ef, k))


def test_embeddings_queries_are_normalised_angular_rows(oracle):
    el = random_sum_embeddings(oracle, 20, 60, 200, 2)
    q = random_vectors(5, 20, 3)
    rows = model_rows("embeddings", el, 200)
    d = M.distances("embeddings", rows, M.element_rows("embeddings", q))
    for i in range(5):
        for j in (0, 17, 199):
            assert _bits(d[i, j]) == _bits(el.dist_to_element(j, q[i]))
