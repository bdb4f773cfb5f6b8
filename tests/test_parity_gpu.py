"""Parity tests proper (GPU): the CUDA search path, called through the C ABI, against the CPU oracle on the same
seeded inputs.  Bar: identical id lists, bit-identical f32 distances, identical result counts and identical
n_dist / n_expand / n_neighbors counters (the traversal itself is identical, not just its answer).

Reference behaviour under test: Granne::search (src/index/mod.rs:140-150, 962-1037) for the three element kinds
(src/elements/angular.rs, angular_int.rs, embeddings/mod.rs), the Index trait (:54-104) and get_element (:153-155).
The test shapes follow the reference's own tests (src/index/tests.rs:41-132) and BASELINE.json config 1.
"""
import numpy as np
import pytest

import granne_b200
from helpers.data import build_fixture, index_from_lists, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


def open_product(index_bytes, kind, elements_bytes, emb_bytes=None):
    return granne_b200.Granne.from_bytes(index_bytes, kind, elements_bytes, emb_bytes, device=0)


def assert_parity(ref, got, what=""):
    rids, rd, rc, rs = ref
    gids, gd, gc, gs = got
    assert np.array_equal(rc, gc), what + " counts"
    bad = np.nonzero((rids != gids).any(axis=1))[0]
    assert bad.size == 0, "%s ids differ for queries %s: ref %s got %s" % (what, bad[:5], rids[bad[:1]], gids[bad[:1]])
    # bit-identical distances (f32 tolerance stated by north_star is 1e-5; the kernel is built to be exact)
    assert np.array_equal(rd.view(np.uint32), gd.view(np.uint32)), what + " dists"
    assert np.array_equal(rs[:, :3], gs[:, :3]), what + " n_dist/n_expand/n_neighbors counters"


def run_both(oracle_index, product, queries, ef, k, already_element=False):
    ref = oracle_index.search_batch(queries, ef, k, already_element=already_element, with_stats=True)
    got = product.search_batch(queries, ef, k, already_element=already_element, with_stats=True)
    return ref, got


# ---- BASELINE config 1: 10k x 32 angular f32, M=10, ef=50 (plumbing, exact parity) ---------------------------------
@pytest.fixture(scope="module")
def c1(oracle):
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 10_000, 32, seed=1234, num_neighbors=10, max_search=50)
    p = open_product(ib, "angular", eb)
    yield el, g, p
    p.close()


def test_c1_parity_raw_queries(c1):
    el, g, p = c1
    q = random_vectors(1000, 32, seed=4321)
    ref, got = run_both(g, p, q, 50, 10)
    assert_parity(ref, got, "C1")
    assert (got[3][:, 3] == 0).all()  # nobody needed more than the fast pass


@pytest.mark.parametrize("ef,k", [(1, 1), (1, 5), (2, 2), (10, 10), (50, 1), (50, 50), (50, 80), (200, 10), (333, 100)])
def test_c1_parity_over_max_search_and_k(c1, ef, k):
    # num_neighbors > max_search yields max_search results (src/index/mod.rs:974-977)
    el, g, p = c1
    q = random_vectors(200, 32, seed=ef * 1000 + k)
    ref, got = run_both(g, p, q, ef, k)
    assert_parity(ref, got, "ef=%d k=%d" % (ef, k))
    assert (got[2] == min(ef, k)).all()


@pytest.mark.parametrize("ef", [600, 976, 977, 1500])
def test_large_max_search_uses_wider_lists(c1, ef):
    # 32*R list capacities up to R=31 (max_search <= 976), beyond that the generic 64-bit list is the fast pass
    el, g, p = c1
    q = random_vectors(24, 32, seed=ef)
    assert_parity(*run_both(g, p, q, ef, 20), what="ef=%d" % ef)


def test_rows_wider_than_a_warp(oracle):
    # num_neighbors > 32: adjacency rows span two 32-id chunks (the speculative single-register row is bypassed)
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 2500, 24, seed=8, num_neighbors=45, max_search=60)
    assert max(len(g.get_neighbors(i)) for i in range(0, 2500, 7)) > 32
    p = open_product(ib, "angular", eb)
    assert_parity(*run_both(g, p, random_vectors(200, 24, seed=9), 60, 10), what="M=45")
    p.close()


def test_c1_index_trait_and_get_element(c1, oracle):
    el, g, p = c1
    assert len(p) == len(g) == 10_000
    assert p.num_layers() == g.num_layers()
    assert [p.layer_len(l) for l in range(p.num_layers())] == [3, 45, 667, 10_000]  # SURVEY §8 / index/mod.rs:634-643
    rng = np.random.default_rng(0)
    for l in range(p.num_layers()):
        for i in rng.integers(0, p.layer_len(l), size=20):
            assert p.get_neighbors(int(i), l) == g.get_neighbors(int(i), l)
    assert p.get_neighbors(5) == g.get_neighbors(5)  # default layer = last (py/src/lib.rs:268-276)
    rows = el.rows()
    for i in [0, 1, 9_999, 1234]:
        assert np.array_equal(p.get_element(i), rows[i])
    assert p.dim == 32 and p.num_elements() == 10_000


def test_c1_self_recall_like_the_reference_tests(c1):
    # verify_search (src/index/tests.rs:50-62): searching an indexed element finds itself first
    el, g, p = c1
    rows = el.rows()[:3000]
    ids, dists, counts = p.search_batch(rows, 50, 1, already_element=True)
    assert (ids[:, 0] == np.arange(3000)).mean() > 0.95
    # single-query API == batch of one (py/src/lib.rs:227-233)
    one = p.search(random_vectors(1, 32, seed=99)[0], 50, 10)
    ref = g.search(random_vectors(1, 32, seed=99)[0], 50, 10)
    assert one == ref


# ---- every f32 dimension class: tail-only, V=1/2/4 layouts, generic, with/without tail -----------------------------
@pytest.mark.parametrize("dim", [3, 25, 28, 32, 50, 64, 96, 100, 128, 160, 192, 200, 256, 300])
def test_f32_dims(oracle, dim):
    n = 1500 if dim <= 128 else 800
    el, g, ib, eb, _ = build_fixture(oracle, "angular", n, dim, seed=dim, num_neighbors=20, max_search=20)
    p = open_product(ib, "angular", eb)
    q = random_vectors(150, dim, seed=dim + 7)
    assert_parity(*run_both(g, p, q, 40, 10), what="dim=%d raw" % dim)
    # pre-built elements (Rust callers pass &Element): normalised rows used as queries
    assert_parity(*run_both(g, p, el.rows()[:100], 10, 5, already_element=True), what="dim=%d element" % dim)
    for i in [0, n - 1]:
        assert np.array_equal(p.get_element(i), el.rows()[i])
    p.close()


def test_default_parameters_m30_ef200(oracle):
    # BuildConfig defaults (src/index/mod.rs:220-231): M=30, ef=200; search defaults 200 / 10 (py/src/lib.rs:14-15)
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 6000, 128, seed=5, num_neighbors=30, max_search=200, threads=8)
    p = open_product(ib, "angular", eb)
    q = random_vectors(256, 128, seed=6)
    ref, got = run_both(g, p, q, 200, 10)
    assert_parity(ref, got, "M30 ef200")
    p.close()


# ---- angular_int (i8, dp4a path) --------------------------------------------------------------------------------
@pytest.mark.parametrize("n,dim", [(500, 32), (2000, 100), (1000, 96), (600, 130), (700, 7)])
def test_i8(oracle, n, dim):
    el, g, ib, eb, _ = build_fixture(oracle, "angular_int", n, dim, seed=n + dim, num_neighbors=20, max_search=20)
    p = open_product(ib, "angular_int", eb)
    q = random_vectors(200, dim, seed=dim * 3)
    assert_parity(*run_both(g, p, q, 50, 10), what="i8 raw dim=%d" % dim)  # quantised on device (angular_int.rs:28-45)
    qi8 = el.rows()[:150]
    assert_parity(*run_both(g, p, qi8, 30, 5), what="i8 element dim=%d" % dim)
    assert np.array_equal(p.get_element(3), el.rows()[3])
    # a zero query: r/ (sqrt(dx)*0) = NaN -> r = 0 -> every distance is 1 (angular_int.rs:55)
    z = np.zeros((2, dim), dtype=np.float32)
    assert_parity(*run_both(g, p, z, 10, 5), what="i8 zero query")
    p.close()


# ---- SumEmbeddings ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,n_emb,n", [(20, 100, 600), (50, 200, 1000), (64, 150, 500)])
def test_sum_embeddings(oracle, dim, n_emb, n):
    el, g, ib, eb, mb = build_fixture(oracle, "embeddings", n, dim, seed=dim, num_neighbors=16, max_search=30,
                                      num_embeddings=n_emb)
    p = open_product(ib, "embeddings", eb, mb)
    q = random_vectors(120, dim, seed=dim + 1)
    assert_parity(*run_both(g, p, q, 40, 10), what="sum dim=%d" % dim)
    for i in [0, 1, n - 1]:
        assert np.array_equal(p.get_element(i), el.get(i))  # normalised ordered sum (embeddings/mod.rs:164-166)
    p.close()


# ---- distance ties / duplicates: exactness under equal distances, slow path --------------------------------------
def test_duplicates_and_ties(oracle):
    raw = random_vectors(3000, 16, seed=77)
    raw[100:140] = raw[50]
    raw[500:510] = raw[499]
    el = oracle.Elements.angular(raw)
    g0 = oracle.GranneBuilder(el, num_neighbors=12, max_search=40).build()
    ib, eb = g0.to_bytes(), el.to_bytes()
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", eb)
    q = random_vectors(300, 16, seed=78)
    q[:50] = raw[50:100] + 1e-3 * random_vectors(50, 16, seed=79)
    for ef in [1, 10, 30, 64]:
        assert_parity(*run_both(g, p, q, ef, ef), what="ties ef=%d" % ef)
    p.close()


def test_all_identical_vectors_take_the_exact_slow_path(oracle):
    # every distance is equal and every node has ~30 neighbours (disjoint fan-outs): while res is not yet full the reference pushes every
    # neighbour (src/index/mod.rs:1029), so the frontier holds a plateau of equal distances far wider than the fast
    # path's bounded list.  The kernel must detect that it cannot drop entries exactly and hand the query to the slow
    # path, which stays bit-exact.
    n, dim = 400, 8
    raw = np.tile(random_vectors(1, dim, seed=5), (n, 1))
    el = oracle.Elements.angular(raw)
    nb = [sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]  # disjoint fan-outs
    ib = index_from_lists(oracle, [nb])  # written in granne's format through the oracle's list encoder
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", el.to_bytes())
    q = random_vectors(8, dim, seed=6)
    ref, got = run_both(g, p, q, 20, 10)
    assert_parity(ref, got, "plateau")
    assert (got[3][:, 3] == 2).all()    # flagged twice (fast pass, retry pass): served by the slow pass
    assert (ref[3][:, 1] > 20).all()           # equal-distance frontier entries are expanded beyond max_search
    # the same index with a roomy max_search stays on the fast path
    ref, got = run_both(g, p, q, 300, 10)
    assert_parity(ref, got, "plateau ef=300")
    p.close()


# ---- edge cases ----------------------------------------------------------------------------------------------------
def test_empty_index_and_single_element(oracle):
    el = oracle.Elements.angular(random_vectors(5, 8, seed=1))
    ib = index_from_lists(oracle, [])  # no layers -> search returns Vec::new() (src/index/mod.rs:978-980)
    p = open_product(ib, "angular", el.to_bytes())
    ids, dists, counts = p.search_batch(random_vectors(3, 8, seed=2), 10, 4)
    assert (counts == 0).all() and (ids == 0xFFFFFFFF).all() and np.isinf(dists).all()
    assert len(p) == 0 and p.num_layers() == 0
    p.close()
    el1, g1, ib1, eb1, _ = build_fixture(oracle, "angular", 1, 8, seed=3, num_neighbors=5, max_search=5)
    p = open_product(ib1, "angular", eb1)
    assert_parity(*run_both(g1, p, random_vectors(4, 8, seed=4), 10, 3), what="single element")
    p.close()


def test_index_over_a_prefix_of_the_elements(oracle):
    # build_partial: the index may cover fewer elements than the container holds (src/index/mod.rs:74-83,374-402)
    raw = random_vectors(900, 16, seed=8)
    el = oracle.Elements.angular(raw)
    g0 = oracle.GranneBuilder(el, num_neighbors=10, max_search=30, expected_num_elements=900).build(num_elements=500)
    ib = g0.to_bytes()
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", el.to_bytes())
    assert len(p) == 500 and p.num_elements() == 900
    assert_parity(*run_both(g, p, random_vectors(100, 16, seed=9), 30, 10), what="prefix index")
    p.close()


def test_errors_are_statuses(c1):
    el, g, p = c1
    q = random_vectors(4, 32, seed=1)
    with pytest.raises(granne_b200.GranneError) as ei:
        p.search_batch(q, 0, 10)  # max_search == 0 panics in the reference (src/index/mod.rs:1019)
    assert ei.value.code == -1
    with pytest.raises(ValueError):
        p.search_batch(random_vectors(4, 31, seed=1), 10, 10)
    bad = q.copy()
    bad[2, 5] = np.nan  # NaN distance panics in the reference (angular.rs:70)
    with pytest.raises(granne_b200.GranneError) as ei:
        p.search_batch(bad, 10, 10)
    assert ei.value.code == -6
    # the handle stays usable
    assert_parity(*run_both(g, p, q, 10, 10), what="after errors")
    with pytest.raises(granne_b200.GranneError) as ei:
        p.get_neighbors(10_000, 3)
    assert ei.value.code == -8
    # nq == 0 is fine
    ids, dists, counts = p.search_batch(np.zeros((0, 32), dtype=np.float32), 10, 10)
    assert ids.shape == (0, 10)


def test_open_from_files_like_the_python_binding(oracle, tmp_path):
    # Granne(index_path, element_type, elements_path) (py/src/lib.rs:175-211)
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 800, 24, seed=21, num_neighbors=12, max_search=30)
    (tmp_path / "index.granne").write_bytes(ib)
    (tmp_path / "elements.bin").write_bytes(eb)
    p = granne_b200.Granne(str(tmp_path / "index.granne"), "angular", str(tmp_path / "elements.bin"))
    assert_parity(*run_both(g, p, random_vectors(64, 24, seed=22), 30, 10), what="from files")
    p.close()
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.Granne(str(tmp_path / "missing"), "angular", str(tmp_path / "elements.bin"))
    assert ei.value.code == -3


def test_device_pointer_api_matches_host_api(c1):
    import torch

    el, g, p = c1
    q = random_vectors(512, 32, seed=31)
    ref = p.search_batch(q, 50, 10)
    tq = torch.from_numpy(q).cuda()
    ids, dists, counts = p.search_batch_device(tq, 50, 10)
    torch.cuda.synchronize()
    p.stream_status()
    assert np.array_equal(ids.cpu().numpy().view(np.uint32), ref[0])
    assert np.array_equal(dists.cpu().numpy(), ref[1])
    assert np.array_equal(counts.cpu().numpy().view(np.uint32), ref[2])


def test_concurrent_host_threads(c1):
    # Granne::search takes &self and is Sync; several host threads may search one handle at once
    import threading

    el, g, p = c1
    qs = [random_vectors(200, 32, seed=100 + t) for t in range(4)]
    refs = [g.search_batch(q, 50, 10) for q in qs]
    outs = [None] * 4

    def work(t):
        for _ in range(3):
            outs[t] = p.search_batch(qs[t], 50, 10)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    for t in range(4):
        assert np.array_equal(outs[t][0], refs[t][0]) and np.array_equal(outs[t][1], refs[t][1])


def test_merge_topk_matches_a_cpu_merge(oracle):
    # range-partitioned mode (SURVEY §8e mode 2): per-shard top-k merged by (distance, global id)
    import torch

    shards = []
    for s in range(3):
        el, g, ib, eb, _ = build_fixture(oracle, "angular", 700 + 50 * s, 16, seed=40 + s, num_neighbors=10,
                                         max_search=30)
        shards.append((el, g, open_product(ib, "angular", eb)))
    q = random_vectors(100, 16, seed=50)
    k = 10
    base = [0, 700, 700 + 750]
    part_ids, part_d = [], []
    for el, g, p in shards:
        ids, d, c = p.search_batch(q, 30, k)
        part_ids.append(ids)
        part_d.append(d)
    pi = torch.from_numpy(np.stack(part_ids).view(np.int32)).cuda()
    pd = torch.from_numpy(np.stack(part_d)).cuda()
    out_ids, out_d = granne_b200.merge_topk_device(0, pi, pd, base)
    torch.cuda.synchronize()
    # CPU merge over the ORACLE's per-shard results
    for qi in range(q.shape[0]):
        cand = []
        for s, (el, g, p) in enumerate(shards):
            ids, d, c = g.search_batch(q[qi:qi + 1], 30, k)
            cand += [(float(d[0, j]), base[s] + int(ids[0, j])) for j in range(int(c[0]))]
        cand.sort()
        exp = cand[:k]
        assert out_ids[qi].cpu().tolist() == [e[1] for e in exp]
        assert np.array_equal(out_d[qi].cpu().numpy(), np.array([e[0] for e in exp], dtype=np.float32))
    for _, _, p in shards:
        p.close()


def test_multi_gpu_modes_under_torchrun():
    """Replicated / range-partitioned parity over NCCL (tests/multi_gpu_check.py) when the box has >= 2 GPUs."""
    import os
    import subprocess
    import sys

    import torch

    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(n, 8)),
           "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(root, "tests", "multi_gpu_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "multi-gpu check ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
