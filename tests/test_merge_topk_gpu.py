"""The range-partitioned merge on one GPU: merge_topk_kernel (granne_b200_merge_topk_device) and the C ABI's host merge
(granne_b200_multi_search_batch, partitioned) against the plain statement of the merge: the first k of
sorted((distance, shard base + local id)).

Synthetic tiles put equal distances (0.0 and -0.0 among them) in every part, short parts anywhere in the part list,
up to the 64-part limit, and global ids above 2**32 from bases that are not ascending.  Three shards that are copies
of one index tie on every result, so there the global id alone orders them."""
import numpy as np
import pytest

import granne_b200
from helpers.data import build_fixture, random_vectors
from helpers.fixtures import library  # noqa: F401  (autouse)
from helpers.topk_tiles import PAD_GID, make_tiles, reference_merge, tie_bases
from test_multi_capi_gpu import _devices
from test_parity_gpu import open_product

pytestmark = pytest.mark.gpu


def device_tiles(ids, dists):
    import torch

    return torch.from_numpy(ids.view(np.int32)).cuda(), torch.from_numpy(dists).cuda()


def assert_merged(got_ids, got_d, want_ids, want_d, what):
    gi = got_ids.cpu().numpy().view(np.uint64)
    gd = got_d.cpu().numpy().view(np.uint32)
    bad = np.nonzero((gi != want_ids).any(axis=1) | (gd != want_d.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, "%s: queries %s differ, first: got %s / %s, want %s / %s" % (
        what, bad[:5], gi[bad[0]], got_d.cpu().numpy()[bad[0]], want_ids[bad[0]], want_d[bad[0]])


# ---- synthetic tiles: ties everywhere, short parts, 64 parts ------------------------------------------------------
@pytest.mark.parametrize("P,k,nq", [
    (1, 10, 129), (1, 200, 1),
    (2, 1, 5000), (2, 33, 128),
    (3, 10, 5000), (3, 200, 127), (3, 33, 129),
    (64, 1, 128), (64, 10, 129), (64, 33, 127), (64, 200, 1),
])
def test_merge_of_tied_short_tiles(P, k, nq):
    import torch

    ids, d = make_tiles(P, nq, k, seed=P * 1000 + k + nq)
    base = tie_bases(P)
    want_ids, want_d = reference_merge(ids, d, base, k)
    pi, pd = device_tiles(ids, d)
    out_ids, out_d = granne_b200.merge_topk_device(0, pi, pd, base)
    torch.cuda.synchronize()
    assert_merged(out_ids, out_d, want_ids, want_d, "P=%d k=%d nq=%d" % (P, k, nq))


def test_merge_on_a_stream_of_its_own_into_given_buffers():
    import torch

    P, nq, k = 5, 300, 17
    ids, d = make_tiles(P, nq, k, seed=5)
    base = tie_bases(P)
    want_ids, want_d = reference_merge(ids, d, base, k)
    pi, pd = device_tiles(ids, d)
    out_ids = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    out_d = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = granne_b200.merge_topk_device(0, pi, pd, base, out_ids=out_ids, out_dists=out_d, stream=stream.cuda_stream)
    assert got[0] is out_ids and got[1] is out_d
    stream.synchronize()
    assert_merged(out_ids, out_d, want_ids, want_d, "own stream")


def test_more_than_64_parts_is_an_error():
    ids, d = make_tiles(65, 2, 3, seed=65)
    pi, pd = device_tiles(ids, d)
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.merge_topk_device(0, pi, pd, tie_bases(65))
    assert ei.value.code == -1


# ---- real shards that tie on every result ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def copies(oracle):
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 2000, 32, seed=21, num_neighbors=12, max_search=40)
    q = random_vectors(300, 32, seed=22)
    k, n, S = 10, 2000, 3
    rids, rd, rc = g.search_batch(q, 40, k)
    want_ids = np.full((q.shape[0], k), PAD_GID, dtype=np.uint64)
    want_d = np.full((q.shape[0], k), np.inf, dtype=np.float32)
    for qi in range(q.shape[0]):
        cand = sorted((float(rd[qi, j]), s * n + int(rids[qi, j]), rd[qi, j]) for s in range(S) for j in range(rc[qi]))
        want_ids[qi, :min(k, len(cand))] = [c[1] for c in cand[:k]]
        want_d[qi, :min(k, len(cand))] = [c[2] for c in cand[:k]]
    return ib, eb, q, k, [s * n for s in range(S)], want_ids, want_d


def test_device_merge_of_identical_shards(copies):
    import torch

    ib, eb, q, k, base, want_ids, want_d = copies
    p = open_product(ib, "angular", eb)
    ids, d, _ = p.search_batch(q, 40, k)
    pi, pd = device_tiles(np.stack([ids] * 3), np.stack([d] * 3))
    out_ids, out_d = granne_b200.merge_topk_device(0, pi, pd, base)
    torch.cuda.synchronize()
    assert_merged(out_ids, out_d, want_ids, want_d, "three identical shards, device merge")
    p.close()


def test_multi_handle_merge_of_identical_shards(copies):
    ib, eb, q, k, base, want_ids, want_d = copies
    m = granne_b200.MultiGranne.partitioned([(ib, eb)] * 3, "angular", _devices(2))
    assert [m.shard_base(s) for s in range(3)] == base
    ids, d, c = m.search_batch(q, 40, k)
    assert np.array_equal(ids, want_ids) and np.array_equal(d.view(np.uint32), want_d.view(np.uint32))
    assert np.array_equal(c, (want_ids != PAD_GID).sum(axis=1))
    m.close()


# ---- the Python wrapper checks what the library cannot -----------------------------------------------------------
def test_merge_wrapper_rejects_bad_tensors():
    import torch

    P, nq, k = 3, 4, 5
    ids = torch.zeros((P, nq, k), dtype=torch.int32, device="cuda")
    d = torch.zeros((P, nq, k), dtype=torch.float32, device="cuda")
    base = [0, 10, 20]
    out_ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_d = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    bad = {
        "ids int64": dict(part_ids=ids.long()),
        "dists float64": dict(part_dists=d.double()),
        "ids 2-D": dict(part_ids=ids[0]),
        "dists 2-D": dict(part_dists=d[0]),
        "dists shape": dict(part_dists=d[:, :, :4].contiguous()),
        "ids strided": dict(part_ids=ids.transpose(1, 2).contiguous().transpose(1, 2)),
        "dists strided": dict(part_dists=d.transpose(0, 1).contiguous().transpose(0, 1)),
        "ids on the host": dict(part_ids=ids.cpu()),
        "dists on the host": dict(part_dists=d.cpu()),
        "other device": dict(device=1),
        "short base": dict(part_base=base[:2]),
        "long base": dict(part_base=base + [30]),
        "out_ids dtype": dict(out_ids=out_ids.int()),
        "out_ids shape": dict(out_ids=out_ids[:3]),
        "out_dists shape": dict(out_dists=out_d[:, :4]),
        "out_dists on the host": dict(out_dists=out_d.cpu()),
        "only out_ids": dict(out_dists=None),
    }
    for what, change in bad.items():
        args = dict(device=0, part_ids=ids, part_dists=d, part_base=base, out_ids=out_ids, out_dists=out_d)
        args.update(change)
        with pytest.raises(ValueError):
            granne_b200.merge_topk_device(**args)
            pytest.fail(what)
    got = granne_b200.merge_topk_device(0, ids, d, base, out_ids=out_ids, out_dists=out_d)
    torch.cuda.synchronize()
    assert got[0] is out_ids
