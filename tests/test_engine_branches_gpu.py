"""Search parity for the distance-engine branches and query edges that the shape sweeps of test_parity_gpu.py do not
reach (GPU).  Each case runs raw queries and `already_element` queries through search_kernel and compares them with
the oracle: same ids, bit-identical distances, same counts and counters.

Engine selection (granne_b200.cu, DistDispatch / engine_tiles): f32 rows use DistF32<FULL> (FULL = dim / 32 in
{0..4, 6, 8} with 4-float groups), else DistF32Generic, which stages rows of up to 64 32-float chunks (dim < 2080) and
loads wider rows directly; i8 rows use DistI8 (lanes per row by row bytes, a separate path beyond 512 bytes); sums of
embeddings use DistSum (128 floats per pass, 32 terms per id load)."""
import numpy as np
import pytest

from helpers.data import random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)
from test_parity_gpu import assert_parity, open_product, run_both

pytestmark = pytest.mark.gpu

GENERIC_STAGED_MAX_CHUNKS = 64  # DistF32Generic stages rows of <= 64 32-float chunks; wider rows load directly


def _index(oracle, el, m=20, ef=30):
    ib = oracle.GranneBuilder(el, num_neighbors=m, max_search=ef).build(threads=8).to_bytes()
    return ib, oracle.Granne.from_bytes(ib, el)


def _edge_queries(dim, seed):
    """Raw queries at the edges: zero (every distance is 1 and ties everywhere), tiny magnitudes whose squares are
    subnormal (1e-20) or underflow to zero (1e-25) — a build with flush-to-zero or fast-math would differ here."""
    base = random_vectors(40, dim, seed)
    return np.concatenate([np.zeros((2, dim), np.float32), base[:20] * np.float32(1e-20), base[20:] * np.float32(1e-25)])


def _f32_cases(p, g, el, dim, what):
    n = len(el)
    assert_parity(*run_both(g, p, random_vectors(150, dim, seed=dim + 7), 40, 10), what=what + " raw")
    rows = el.rows()[:: max(1, n // 100)]
    assert_parity(*run_both(g, p, rows, 20, 10, already_element=True), what=what + " element")
    # elements that are not unit length: r > 1 clamps to distance 0 (many exact ties), r < 1 does not
    assert_parity(*run_both(g, p, rows[:50] * np.float32(3.0), 20, 10, already_element=True), what=what + " r > 1")
    assert_parity(*run_both(g, p, rows[50:] * np.float32(0.5), 20, 10, already_element=True), what=what + " r < 1")
    tiny = rows[:40] * np.float32(1e-20)
    assert_parity(*run_both(g, p, tiny, 20, 10, already_element=True), what=what + " tiny element")
    ref, got = run_both(g, p, _edge_queries(dim, dim), 20, 10)
    assert_parity(ref, got, what + " zero / tiny raw")
    assert (ref[1][:2, :ref[2][0]] == 1.0).all()  # a zero query is at distance 1 from everything


# ---- f32: FULL with a tail, generic staged, generic direct --------------------------------------------------------
@pytest.mark.parametrize("dim", [33, 65, 129, 287, 512, 1024, 2100])
def test_f32_engine_branches(oracle, dim):
    if dim == 2100:
        assert dim // 32 > GENERIC_STAGED_MAX_CHUNKS  # really the direct-load branch (stg_rows == 0)
    n = 1000 if dim <= 300 else 600
    el = oracle.Elements.angular(random_vectors(n, dim, seed=dim))
    ib, g = _index(oracle, el)
    p = open_product(ib, "angular", el.to_bytes())
    _f32_cases(p, g, el, dim, "f32 dim=%d" % dim)
    p.close()


# ---- i8: 32 lanes per row (257..512 bytes) and the wide-row path (> 512 bytes) -----------------------------------
@pytest.mark.parametrize("dim", [300, 512, 600, 1000])
def test_i8_engine_branches(oracle, dim):
    el = oracle.Elements.angular_int(random_vectors(800, dim, seed=dim))
    ib, g = _index(oracle, el)
    p = open_product(ib, "angular_int", el.to_bytes())
    assert_parity(*run_both(g, p, random_vectors(150, dim, seed=dim + 1), 40, 10), what="i8 dim=%d raw" % dim)
    assert_parity(*run_both(g, p, el.rows()[::8], 20, 10), what="i8 dim=%d element" % dim)
    assert_parity(*run_both(g, p, _edge_queries(dim, dim), 20, 10), what="i8 dim=%d zero / tiny raw" % dim)
    p.close()


# ---- SumEmbeddings: wide rows, many terms, empty and repeated terms -----------------------------------------------
def _sum_elements(n, n_emb, seed, min_terms, max_terms):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, n_emb, size=int(rng.integers(min_terms, max_terms + 1))).tolist() for _ in range(n)]


def _sum_case(oracle, dim, lists, n_emb, seed, what):
    el = oracle.Elements.sum_embeddings(random_vectors(n_emb, dim, seed=seed), lists)
    ib, g = _index(oracle, el, m=16)
    p = open_product(ib, "embeddings", el.to_bytes(0), el.to_bytes(1))
    n = len(lists)
    for i in (0, 1, n // 2, n - 1):
        assert np.array_equal(p.get_element(i), el.get(i))
    assert_parity(*run_both(g, p, random_vectors(150, dim, seed=seed + 1), 40, 10), what=what + " raw")
    elems = np.stack([el.get(i) for i in range(0, n, max(1, n // 100))])
    assert_parity(*run_both(g, p, elems, 20, 10, already_element=True), what=what + " element")
    assert_parity(*run_both(g, p, elems[:40] * np.float32(2.0), 20, 10, already_element=True), what=what + " r > 1")
    assert_parity(*run_both(g, p, _edge_queries(dim, seed), 20, 10), what=what + " zero / tiny raw")
    p.close()
    return el


@pytest.mark.parametrize("dim", [129, 300])
def test_sum_embeddings_wide_rows(oracle, dim):
    _sum_case(oracle, dim, _sum_elements(700, 300, dim, 1, 8), 300, dim, "sum dim=%d" % dim)


@pytest.mark.parametrize("terms", [33, 70])
def test_sum_embeddings_many_terms(oracle, terms):
    lists = _sum_elements(600, 400, terms, terms - 3, terms + 3)
    assert max(len(l) for l in lists) > 32
    _sum_case(oracle, 50, lists, 400, terms, "sum %d terms" % terms)


def test_sum_embeddings_empty_and_repeated_terms(oracle):
    # an element without terms is the zero vector (embeddings/mod.rs:125-131): never indexed by the builder, at
    # distance 1 from every query; repeated terms are summed as often as they occur
    lists = _sum_elements(700, 150, 9, 1, 6)
    for i in (3, 50, 400, 699):
        lists[i] = []
    for i in range(100, 160):
        t = lists[i][0]
        lists[i] = [t] * (2 + i % 5) + lists[i][1:] + [t]
    el = _sum_case(oracle, 40, lists, 150, 9, "sum empty / repeated")
    assert not el.get(3).any()
