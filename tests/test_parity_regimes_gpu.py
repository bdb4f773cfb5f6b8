"""Search parity in the regimes the kernel really runs in (GPU).  search_kernel is persistent: every one-warp CTA takes
queries from a work counter until the batch is done, so at bench sizes one warp answers many queries in a row and the
speculative adjacency slots, visited buckets and per-query status carry over from one query (and one pass of the
fast / retry / slow ladder) to the next.  These tests compare such batches with the oracle query by query: same ids,
bit-identical distances, same counts and n_dist / n_expand / n_neighbors counters."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers.data import build_fixture, index_from_lists, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)
from test_parity_gpu import assert_parity, open_product

pytestmark = pytest.mark.gpu

MAX_CTAS_PER_SM = 32  # the most resident CTAs an H100 SM holds: the fast pass's grid never exceeds this x SMs


def queries_for_four_per_warp():
    import torch

    return 4 * MAX_CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count


def run_both(g, p, q, ef, k, already_element=False):
    ref = g.search_batch(q, ef, k, already_element=already_element, threads=8, with_stats=True)
    got = p.search_batch(q, ef, k, already_element=already_element, with_stats=True)
    return ref, got


# ---- many queries per warp, one engine each ------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim", [
    ("angular", 24),       # DistF32<0>
    ("angular", 32),       # DistF32<1>
    ("angular", 128),      # DistF32<4>
    ("angular", 160),      # DistF32Generic, staged
    ("angular_int", 100),  # DistI8
    ("embeddings", 50),    # DistSum
])
def test_many_queries_per_warp(oracle, kind, dim):
    nq = queries_for_four_per_warp()
    el, g, ib, eb, mb = build_fixture(oracle, kind, 2000, dim, seed=dim, num_neighbors=16, max_search=40, threads=8)
    p = open_product(ib, kind, eb, mb)
    q = random_vectors(nq, dim, seed=dim + 1)
    ref, got = run_both(g, p, q, 40, 10)
    assert_parity(ref, got, "%s dim=%d nq=%d" % (kind, dim, nq))
    p.close()


_ONE_CTA_PER_SM = r"""
import sys
sys.path[:0] = [%(root)r, %(tests)r]
import granne_b200, torch
from oracle import granne_oracle as go
from helpers.data import build_fixture, random_vectors
from test_parity_gpu import assert_parity
granne_b200.load_library()
sms = torch.cuda.get_device_properties(0).multi_processor_count
nq = 30 * sms
for kind, dim in [("angular", 24), ("angular", 100), ("angular_int", 100), ("embeddings", 50)]:
    el, g, ib, eb, mb = build_fixture(go, kind, 2000, dim, seed=dim, num_neighbors=16, max_search=40, threads=8)
    p = granne_b200.Granne.from_bytes(ib, kind, eb, mb, device=0)
    q = random_vectors(nq, dim, seed=dim + 2)
    ref = g.search_batch(q, 40, 10, threads=8, with_stats=True)
    got = p.search_batch(q, 40, 10, with_stats=True)
    assert_parity(ref, got, "%%s dim=%%d, one CTA per SM" %% (kind, dim))
    p.close()
print("one CTA per SM ok: %%d queries per warp" %% (nq // sms))
"""


def test_thirty_queries_per_warp_in_a_process_of_its_own():
    # GRANNE_B200_MAX_CTAS_PER_SM is read once per process: with 1 CTA per SM every warp answers ~30 queries
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _ONE_CTA_PER_SM % {"root": root, "tests": os.path.join(root, "tests")}
    env = dict(os.environ, GRANNE_B200_MAX_CTAS_PER_SM="1")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0 and "one CTA per SM ok: 30 queries per warp" in out.stdout, \
        out.stdout[-2000:] + out.stderr[-2000:]


# ---- mixed pass ladder in one launch -------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim,n,ef", [("angular", 24, 20_000, 40), ("angular", 48, 10_000, 20),
                                           ("embeddings", 48, 10_000, 40)])
def test_mixed_pass_ladder_in_one_launch(oracle, kind, dim, n, ef):
    # Uniform data (src/test_helper.rs:3-6) on a fresh handle: the visited tables start at their base size, so at
    # these max_search values a part of every batch overflows the fast pass (flag 1 or 2) and the warp that found out
    # moves straight on to its next query, while the rest is answered by the fast pass (flag 0).
    if kind == "angular":
        el = oracle.Elements.angular(random_vectors(n, dim, seed=41))
    else:
        rng = np.random.default_rng(3)
        terms = [rng.integers(0, 2000, size=int(rng.integers(1, 6))).tolist() for _ in range(n)]
        el = oracle.Elements.sum_embeddings(random_vectors(2000, dim, seed=5), terms)
    ib = oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8).to_bytes()
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, kind, el.to_bytes(0), el.to_bytes(1) if kind == "embeddings" else None)
    q = random_vectors(queries_for_four_per_warp(), dim, seed=42)
    ref, got = run_both(g, p, q, ef, 10)
    flags = got[3][:, 3]
    assert (flags == 0).any() and (flags >= 1).any(), "batch not mixed: %s" % np.bincount(flags.astype(np.int64))
    assert_parity(ref, got, "%s dim=%d ef=%d mixed ladder" % (kind, dim, ef))
    p.close()


def test_slow_pass_serves_many_queries_per_cta(oracle):
    # the all-identical plateau of test_parity_gpu: every query is handed to the slow pass (a few CTAs), so each of its
    # warps answers dozens of queries one after another
    n, dim = 400, 8
    raw = np.tile(random_vectors(1, dim, seed=5), (n, 1))
    el = oracle.Elements.angular(raw)
    nb = [sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]
    ib = index_from_lists(oracle, [nb])
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", el.to_bytes())
    ref, got = run_both(g, p, random_vectors(256, dim, seed=6), 20, 10)
    assert (got[3][:, 3] == 2).all()
    assert_parity(ref, got, "plateau, 256 queries")
    p.close()


# ---- one handle, changing calls -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shared(oracle):
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 5000, 32, seed=61, num_neighbors=16, max_search=40, threads=8)
    p = open_product(ib, "angular", eb)
    yield el, g, p
    p.close()


def test_one_handle_changing_launch_plans(shared):
    # workspaces, visited tables and output buffers are reused across calls whose plans differ
    el, g, p = shared
    rows = el.rows()
    for i, (nq, ef, k) in enumerate([(20_000, 50, 10), (7, 333, 100), (3000, 1, 1), (5000, 976, 64), (100, 1500, 20),
                                     (20_000, 50, 10)]):
        q = random_vectors(nq, 32, seed=70 + i)
        assert_parity(*run_both(g, p, q, ef, k), what="raw nq=%d ef=%d k=%d" % (nq, ef, k))
        e = rows[np.random.default_rng(i).integers(0, len(rows), size=min(nq, 2000))]
        assert_parity(*run_both(g, p, e, ef, k, already_element=True), what="element nq=%d ef=%d" % (e.shape[0], ef))


def _device_search(p, q, ef, k, already_element=False, stream=None):
    import torch

    tq = torch.from_numpy(q).cuda()
    stats = torch.empty((q.shape[0], 4), dtype=torch.int64, device="cuda")
    ids, d, c = p.search_batch_device(tq, ef, k, already_element=already_element, stats=stats,
                                      stream=None if stream is None else stream.cuda_stream)
    return ids, d, c, stats


def _host(dev):
    ids, d, c, s = (t.cpu().numpy() for t in dev)
    return ids.view(np.uint32), d, c.view(np.uint32), s.view(np.uint64)


def test_one_handle_host_and_device_calls_alternate(shared):
    import torch

    el, g, p = shared
    rows = el.rows()
    for i, (ef, k) in enumerate([(50, 10), (200, 30), (8, 8), (600, 5)]):
        q = random_vectors(3000 + 500 * i, 32, seed=80 + i)
        e = rows[(np.arange(1500) * (i + 7)) % len(rows)]
        assert_parity(*run_both(g, p, q, ef, k), what="host raw ef=%d" % ef)
        got = _host(_device_search(p, q, ef, k))
        torch.cuda.synchronize()
        assert_parity(g.search_batch(q, ef, k, threads=8, with_stats=True), got, "device raw ef=%d" % ef)
        got = _host(_device_search(p, e, ef, k, already_element=True))
        assert_parity(g.search_batch(e, ef, k, already_element=True, threads=8, with_stats=True), got,
                      "device element ef=%d" % ef)
        assert_parity(*run_both(g, p, e, ef, k, already_element=True), what="host element ef=%d" % ef)
    p.stream_status()


def test_one_handle_four_streams_at_once(shared):
    import torch

    el, g, p = shared
    plans = [(4000, 40, 10), (3000, 300, 20), (5000, 10, 5), (2000, 990, 50)]
    qs = [random_vectors(nq, 32, seed=90 + s) for s, (nq, _, _) in enumerate(plans)]
    streams = [torch.cuda.Stream() for _ in plans]
    outs = []
    for s, (q, (nq, ef, k)) in enumerate(zip(qs, plans)):
        with torch.cuda.stream(streams[s]):
            outs.append(_device_search(p, q, ef, k, stream=streams[s]))
    torch.cuda.synchronize()
    for s, (q, (nq, ef, k)) in enumerate(zip(qs, plans)):
        assert_parity(g.search_batch(q, ef, k, threads=8, with_stats=True), _host(outs[s]), "stream %d" % s)
    p.stream_status()
    for st in streams:
        p.release_stream(st)
