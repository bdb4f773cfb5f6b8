"""Full-size checks at BASELINE.json's bench configuration (1M x 128 angular f32, M=30, max_search=200, k=10):
size-independent properties of the search results on thousands of queries, plus bit parity with the oracle on a
sample of queries searched on the very same 1M index file (written by the GPU builder, loaded by the oracle)."""
import numpy as np
import pytest

import granne_b200
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

N, DIM, EF, K = 1_000_000, 128, 200, 10


@pytest.fixture(scope="module")
def big():
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import clustered

    nc = 4096
    eb = granne_b200.elements_from_raw("angular", clustered(N, DIM, 1234, nc))
    b = granne_b200.GranneBuilder("angular", eb, num_neighbors=30, max_search=200)
    b.build()
    index = b.get_index()
    image = b.index_bytes()
    b.close()
    q = clustered(4096, DIM, 4321, nc)
    yield index, eb, image, q
    index.close()


def test_result_properties_at_full_size(big):
    import torch

    index, eb, image, q = big
    ids, d, c, st = index.search_batch(q, EF, K, with_stats=True)
    assert (c == K).all() and (st[:, 3] == 0).all()
    # ascending by (distance, id): the order of into_sorted_vec (src/index/mod.rs:1036); ids are distinct and in range
    assert (np.diff(d, axis=1) >= 0).all()
    ties = np.diff(d, axis=1) == 0
    assert (np.diff(ids.astype(np.int64), axis=1)[ties] > 0).all()
    assert all(len(set(r.tolist())) == K for r in ids[:512]) and int(ids.max()) < N
    # every reported distance is the angular distance of that element: max(0, 1 - <x, q/|q|>) within float tolerance
    rows = torch.from_numpy(np.frombuffer(eb, dtype=np.float32, offset=8).reshape(N, DIM))
    qn = torch.nn.functional.normalize(torch.from_numpy(q[:512]), dim=1)
    got = torch.from_numpy(ids[:512].astype(np.int64))
    recomputed = 1.0 - (rows[got] * qn[:, None, :]).sum(dim=2)
    assert np.allclose(np.maximum(recomputed.numpy(), 0.0), d[:512], atol=1e-5)
    # results do not depend on how queries are batched, and a repeated call is identical
    a1 = index.search_batch(q[:1000], EF, K)
    a2 = index.search_batch(q[:1000], EF, K)
    h1 = index.search_batch(q[:300], EF, K)
    h2 = index.search_batch(q[300:1000], EF, K)
    assert np.array_equal(a1[0], a2[0]) and np.array_equal(a1[1], a2[1])
    assert np.array_equal(a1[0], np.concatenate([h1[0], h2[0]])) and np.array_equal(a1[1], np.concatenate([h1[1], h2[1]]))
    assert np.array_equal(a1[0], ids[:1000])
    # searching for an indexed element finds it first (verify_search, src/index/tests.rs:50-62)
    sample = np.arange(0, N, N // 2000)[:2000]
    self_ids, _, _ = index.search_batch(rows[sample].numpy(), EF, 1, already_element=True)
    assert (self_ids[:, 0] == sample).mean() > 0.95
    # recall@10 against the exact top-10 (the metric's condition)
    dev = torch.device("cuda")
    best = None
    qd = qn[:256].to(dev)
    for s0 in range(0, N, 1 << 18):
        sc = qd @ rows[s0:s0 + (1 << 18)].to(dev).T
        v, i = torch.topk(sc, K, dim=1)
        i = i + s0
        best = (v, i) if best is None else tuple(
            torch.gather(t, 1, torch.topk(torch.cat([best[0], v], 1), K, dim=1).indices)
            for t in (torch.cat([best[0], v], 1), torch.cat([best[1], i], 1)))
    gt = best[1].cpu().numpy()
    recall = np.mean([len(set(gt[i].tolist()) & set(ids[i].tolist())) / K for i in range(256)])
    assert recall >= 0.95, recall


def test_sampled_parity_with_the_oracle_at_full_size(big, oracle):
    index, eb, image, q = big
    el = oracle.Elements.from_bytes("angular", eb.tobytes())
    g = oracle.Granne.from_bytes(image.tobytes(), el)
    assert len(g) == N and [g.layer_len(l) for l in range(g.num_layers())] == \
        [index.layer_len(l) for l in range(index.num_layers())]
    sample = q[:96]
    ref = g.search_batch(sample, EF, K, with_stats=True, threads=8)
    got = index.search_batch(sample, EF, K, with_stats=True)
    assert np.array_equal(ref[0], got[0])
    assert np.array_equal(ref[1].view(np.uint32), got[1].view(np.uint32))
    assert np.array_equal(ref[2], got[2]) and np.array_equal(ref[3][:, :3], got[3][:, :3])
