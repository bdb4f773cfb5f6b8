"""GPU tests of the multi-device C ABI (granne_b200_multi_*): several GPUs of one process behind one handle, no torch
and no NCCL in the path (what a Rust / C++ host of `Granne::from_bytes`, src/index/mod.rs:108-113, would bind).

Replicated mode must be bit-identical to the oracle's search of the whole batch; range-partitioned mode must equal the
oracle's per-shard searches merged by (distance, global id) — the tuple order of into_sorted_vec
(src/index/mod.rs:1036).  On a one-GPU box the device list names cuda:0 twice (two replicas / two shards on the same
device exercise exactly the same host logic); with more GPUs visible every device is used.
"""
import numpy as np
import pytest

import granne_b200
from granne_b200.distributed import merge_topk_host
from helpers.data import build_fixture, random_vectors

pytestmark = pytest.mark.gpu
INVALID = -1  # GRANNE_B200_ERR_INVALID_ARGUMENT


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


def _devices(minimum):
    import torch

    n = torch.cuda.device_count()
    devs = list(range(n))
    while len(devs) < minimum:
        devs.append(devs[len(devs) % n])
    return devs


@pytest.mark.parametrize("kind,dim", [("angular", 32), ("angular_int", 40)])
def test_replicated_multi_handle_equals_the_oracle(oracle, kind, dim):
    el, g, ib, eb, _ = build_fixture(oracle, kind, 6000, dim, seed=7, num_neighbors=12, max_search=50)
    devs = _devices(2)
    m = granne_b200.MultiGranne.replicated(ib, kind, eb, devs)
    assert len(m) == 6000 and m.num_parts() == len(devs)
    for nq in (1, 3, 1001):  # fewer queries than devices, uneven slices
        q = random_vectors(nq, dim, seed=100 + nq)
        ids, d, c = m.search_batch(q, 50, 10)
        rids, rd, rc = g.search_batch(q, 50, 10)
        want = np.where(rids == 0xFFFFFFFF, np.uint64(0xFFFFFFFFFFFFFFFF), rids.astype(np.uint64))
        assert np.array_equal(ids, want) and np.array_equal(d.view(np.uint32), rd.view(np.uint32))
        assert np.array_equal(c, rc)
    m.close()


def test_partitioned_multi_handle_equals_merged_oracle_shards(oracle):
    sizes = [2500, 3100, 1800]
    shards, refs = [], []
    for s, n in enumerate(sizes):
        el, g, ib, eb, _ = build_fixture(oracle, "angular", n, 32, seed=40 + s, num_neighbors=10, max_search=50)
        shards.append((ib, eb))
        refs.append(g)
    devs = _devices(2)  # three shards over the visible devices (round robin)
    m = granne_b200.MultiGranne.partitioned(shards, "angular", devs)
    bases = [0, sizes[0], sizes[0] + sizes[1]]
    assert [m.shard_base(s) for s in range(3)] == bases and len(m) == sum(sizes) and m.num_parts() == 3
    q = random_vectors(700, 32, seed=9)
    ids, d, c = m.search_batch(q, 50, 10)
    parts = [r.search_batch(q, 50, 10) for r in refs]
    ei, ed = merge_topk_host(np.stack([p[0] for p in parts]), np.stack([p[1] for p in parts]), bases, 10)
    assert np.array_equal(ids.view(np.int64), ei) and np.array_equal(d.view(np.uint32), ed.view(np.uint32))
    assert (c == 10).all()
    m.close()


def test_multi_open_reports_errors_as_status(oracle):
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 500, 16, seed=3, num_neighbors=8, max_search=20)
    with pytest.raises(granne_b200.GranneError):
        granne_b200.MultiGranne.replicated(ib, "angular", eb, [999])           # no such device
    with pytest.raises(granne_b200.GranneError):
        granne_b200.MultiGranne.partitioned([(ib, eb), (ib[:100], eb)], "angular", [0])  # a garbled shard
    m = granne_b200.MultiGranne.replicated(ib, "angular", eb, [0])
    with pytest.raises(granne_b200.GranneError):
        m.search_batch(random_vectors(4, 16, seed=1), 0, 5)                    # max_search == 0 panics in the reference
    m.close()


def test_multi_calls_report_the_single_device_rules(oracle):
    """Each multi call checks the rules of its single-device call before any part runs: on a one-device replicated
    handle, the same bad arguments give the single-device call's status and message, nq == 0 included."""
    from granne_b200 import api

    el, g, ib, eb, _ = build_fixture(oracle, "angular", 500, 16, seed=3, num_neighbors=8, max_search=20)
    L = granne_b200.load_library()
    s = granne_b200.Granne.from_bytes(ib, "angular", eb)
    m = granne_b200.MultiGranne.replicated(ib, "angular", eb, [0])
    q = random_vectors(2, 16, seed=1)
    ids32, ids64, dists = np.zeros(4000, np.uint32), np.zeros(4000, np.uint64), np.zeros(4000, np.float32)
    offsets, words = np.array([0, 2, 3], np.uint64), np.ones((1, 16), np.uint32)
    cand32, cand64 = np.array([0, 1, 2], np.uint32), np.array([0, 1, 2], np.uint64)

    def run(call, multi, nq=2, fmt=api.QUERY_RAW_F32, ef=20, k=5, queries=True, out=True, offs=True, cand=True,
            filters=True, nf=1):
        h = m._h if multi else s._h
        pq = api._ptr(q) if queries else None
        pi = api._ptr(ids64 if multi else ids32) if out else None
        pd = api._ptr(dists)
        stats = () if multi else (None,)
        if call == "search":
            fn = L.granne_b200_multi_search_batch if multi else L.granne_b200_search_batch
            rc = fn(h, pq, nq, fmt, ef, k, pi, pd, None, *stats)
        elif call == "exact":
            fn = L.granne_b200_multi_exact_search_batch if multi else L.granne_b200_exact_search_batch
            rc = fn(h, pq, nq, fmt, k, pi, pd, None)
        elif call == "within":
            fn = L.granne_b200_multi_exact_search_within_batch if multi else L.granne_b200_exact_search_within_batch
            rc = fn(h, pq, nq, fmt, api._ptr(offsets) if offs else None,
                    api._ptr(cand64 if multi else cand32) if cand else None, k, pi, pd, None)
        elif call == "filtered":
            fn = L.granne_b200_multi_search_filtered_batch if multi else L.granne_b200_search_filtered_batch
            rc = fn(h, pq, nq, fmt, ef, k, api._ptr(words) if filters else None, nf, 16, None, pi, pd, None, *stats)
        else:
            fn = L.granne_b200_multi_search_rerank_batch if multi else L.granne_b200_search_rerank_batch
            rc = fn(h, pq, nq, fmt, ef, 10, k, pi, pd, None, *stats)
        return rc, L.granne_b200_last_error().decode()

    shared = [dict(fmt=7), dict(nq=0, fmt=7), dict(nq=0xFFFFFFF1, queries=False), dict(queries=False), dict(out=False)]
    max_search = [dict(ef=0), dict(nq=0, ef=0), dict(ef=0, fmt=7)]
    exact_k = [dict(k=1025), dict(nq=0, k=1025)]
    cases = {
        "search": shared + max_search,
        "exact": shared + exact_k,
        "within": shared + exact_k + [dict(offs=False), dict(offs=False, cand=False), dict(cand=False)],
        "filtered": shared + max_search + exact_k + [dict(filters=False), dict(nf=0), dict(ef=0, k=1025)],
        # no re-rank container is attached: the rule reads the handle, the multi call reads its first part's
        "rerank": shared + max_search + [dict(), dict(fmt=api.QUERY_ELEMENT)],
    }
    for call, args in cases.items():
        for a in args:
            want = run(call, False, **a)
            assert want[0] == INVALID, (call, a, want)
            assert run(call, True, **a) == want, (call, a)
    m.close()
    s.close()
