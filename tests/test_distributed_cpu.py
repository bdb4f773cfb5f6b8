"""Host-side logic of the N > 1 path on CPU: world_size-2 gloo process groups (SURVEY.md §8e).

The per-rank local search is injected (the CPU oracle stands in for the GPU kernel, which needs a device); what is
under test is the sharding, the collectives and the merge: a replicated, query-sharded search must return exactly the
single-process result, and a range-partitioned search must equal the oracle's per-shard searches merged by
(distance, global id)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from granne_b200.distributed import PartitionedGranne, ReplicatedGranne, merge_topk_host, shard_bounds
from helpers.data import random_vectors
from helpers.topk_tiles import make_tiles, reference_merge, tie_bases


def test_shard_bounds_cover_everything():
    for n in [0, 1, 7, 8, 1024, 1025]:
        for world in [1, 2, 3, 8]:
            spans = [shard_bounds(n, world, r) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [e - b for b, e in spans]
            assert max(sizes) - min(sizes) <= 1


def test_merge_topk_host_orders_by_distance_then_global_id():
    ids = np.array([[[0, 2, 0xFFFFFFFF]], [[1, 0xFFFFFFFF, 0xFFFFFFFF]]], dtype=np.uint32)
    d = np.array([[[0.5, 0.7, np.inf]], [[0.5, np.inf, np.inf]]], dtype=np.float32)
    gi, gd = merge_topk_host(ids, d, [10, 0], 3)
    assert gi.tolist() == [[1, 10, 12]]  # equal distances: the smaller global id first (tuple order)
    assert gd.tolist() == [[0.5, 0.5, np.float32(0.7)]]


@pytest.mark.parametrize("P,k,nq", [(1, 200, 3), (2, 1, 129), (3, 10, 5000), (3, 33, 128), (64, 10, 127), (64, 200, 1)])
def test_merge_topk_host_on_tied_short_tiles(P, k, nq):
    # the numpy merge against the plain sort the GPU merge is held to (tests/test_merge_topk_gpu.py)
    ids, d = make_tiles(P, nq, k, seed=P * 1000 + k + nq)
    base = tie_bases(P)
    want_ids, want_d = reference_merge(ids, d, base, k)
    gi, gd = merge_topk_host(ids, d, base, k)
    assert np.array_equal(gi.view(np.uint64), want_ids)
    assert np.array_equal(gd.view(np.uint32), want_d.view(np.uint32))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, mode, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import granne_oracle as go

        q = random_vectors(37, 16, seed=5)  # deliberately not divisible by the world size
        if mode == "replicated":
            el = go.Elements.angular(random_vectors(1500, 16, seed=1))
            g = go.GranneBuilder(el, num_neighbors=12, max_search=30).build()

            def local(queries, ef, k):
                ids, d, c = g.search_batch(queries.numpy(), ef, k)
                return torch.from_numpy(ids.view(np.int32)), torch.from_numpy(d)

            r = ReplicatedGranne(local_search=local)
            ids, d = r.search_batch(torch.from_numpy(q), 30, 10)
            ref_ids, ref_d, _ = g.search_batch(q, 30, 10)
            ok = np.array_equal(ids.numpy().view(np.uint32), ref_ids) and np.array_equal(d.numpy(), ref_d)
        else:
            sizes = [700, 900]
            base = [0, 700]
            shards = []
            for s in range(world):
                el = go.Elements.angular(random_vectors(sizes[s], 16, seed=10 + s))
                shards.append(go.GranneBuilder(el, num_neighbors=12, max_search=30).build())
            mine = shards[rank]

            def local(queries, ef, k):
                ids, d, c = mine.search_batch(queries.numpy(), ef, k)
                return torch.from_numpy(ids.view(np.int32)), torch.from_numpy(d)

            p = PartitionedGranne(shard_base=base[rank], local_search=local, host_merge=True)
            gi, gd = p.search_batch(torch.from_numpy(q), 30, 10)
            parts = [s.search_batch(q, 30, 10) for s in shards]
            ei, ed = merge_topk_host(np.stack([x[0] for x in parts]), np.stack([x[1] for x in parts]), base, 10)
            ok = np.array_equal(gi.numpy(), ei) and np.array_equal(gd.numpy(), ed) and p.bases == base
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["replicated", "partitioned"])
def test_world_size_2_gloo(mode, oracle):
    world = 2
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, mode, ret)) for r in range(world)]
    [p.start() for p in procs]
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert dict(ret) == {0: True, 1: True}
