"""The fused peer gather on one GPU (granne_b200_search_batch_device_gather): the kernels store every result row into
up to 8 peer buffers at `row_offset + query` and, once the last pass is through, release flags[p][my_rank] = seq.

The kernels take plain device pointers and do not care whether a pointer is peer-mapped, so local buffers stand in for
the peers.  Every buffer and flag starts as a sentinel; after a call each peer must hold the oracle's ids and distance
bits in its own rows, padding after them, the sentinel everywhere else, and `seq` in exactly one flag entry.  What
this cannot show — the peer mapping, visibility over NVLink and the system-scope ordering of the release — is checked
with two or more GPUs by tests/multi_gpu_check.py."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from helpers.data import build_fixture, index_from_lists, random_vectors
from test_parity_gpu import assert_parity, open_product
from test_parity_regimes_gpu import queries_for_four_per_warp

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5A5A5A5
PAD_ID = 0xFFFFFFFF
INF_BITS = 0x7F800000
SPARE_FLAGS = 2  # flag entries past n_peers, which must stay untouched too
INVALID_ARGUMENT = -1


@pytest.fixture(scope="module", autouse=True)
def _lib():
    from granne_b200 import build

    build.build()
    granne_b200.load_library()


class Peers:
    """n_peers stand-in peer buffers on cuda:0: ids and distance bits [total_rows, width], flags [n_peers + 2]."""

    def __init__(self, n_peers, total_rows, width):
        import torch

        def make(*shape):
            return torch.empty(shape, dtype=torch.int32, device="cuda")

        self.n_peers = n_peers
        self.ids = [make(total_rows, width) for _ in range(n_peers)]
        self.dists = [make(total_rows, width) for _ in range(n_peers)]
        self.flags = [make(n_peers + SPARE_FLAGS) for _ in range(n_peers)]
        self.fill()

    def fill(self):
        sentinel = int(np.uint32(SENTINEL).view(np.int32))
        for t in self.ids + self.dists + self.flags:
            t.fill_(sentinel)

    def spec(self, my_rank, row_offset, seq):
        g = granne_b200.PeerGather()
        g.n_peers, g.my_rank, g.row_offset, g.seq = self.n_peers, my_rank, row_offset, seq
        for p in range(self.n_peers):
            g.ids[p], g.dists[p], g.flags[p] = (self.ids[p].data_ptr(), self.dists[p].data_ptr(),
                                                self.flags[p].data_ptr())
        return g

    def host(self):
        def u32(t):
            return t.cpu().numpy().view(np.uint32)

        return [(u32(self.ids[p]), u32(self.dists[p]), u32(self.flags[p])) for p in range(self.n_peers)]

    def untouched(self):
        return all((a == SENTINEL).all() for peer in self.host() for a in peer)


def gather(p, peers, q, ef, k, my_rank, row_offset, seq, stream=None):
    """One gather call; returns (queries, counts, stats) device tensors — keep them until the stream is synchronised."""
    import torch

    tq = torch.from_numpy(q).cuda()
    counts = torch.empty((q.shape[0],), dtype=torch.int32, device="cuda")
    stats = torch.empty((q.shape[0], 4), dtype=torch.int64, device="cuda")
    p.search_batch_device_gather(tq, peers.spec(my_rank, row_offset, seq), ef, k, counts=counts, stats=stats,
                                 stream=None if stream is None else stream.cuda_stream)
    return tq, counts, stats


def check_peers(peers, ref, counts, stats, my_rank, row_offset, seq, what, rows=None):
    """Every peer holds `ref` (the oracle's (ids, dists, counts, stats)) in rows [row_offset, row_offset + nq) and the
    sentinel elsewhere; flags[p][my_rank] == seq and no other entry moved.  `rows` limits the parity check to some
    queries (the others are checked by the caller)."""
    nq = ref[0].shape[0]
    got_counts = counts.cpu().numpy().view(np.uint32)
    got_stats = stats.cpu().numpy().view(np.uint64)
    keep = np.arange(nq) if rows is None else rows
    want_flags = np.full(peers.n_peers + SPARE_FLAGS, SENTINEL, dtype=np.uint32)
    want_flags[my_rank] = seq
    for p, (ids, dists, flags) in enumerate(peers.host()):
        mine = ids[row_offset:row_offset + nq], dists[row_offset:row_offset + nq]
        assert_parity(tuple(x[keep] for x in ref),
                      (mine[0][keep], mine[1][keep].view(np.float32), got_counts[keep], got_stats[keep]),
                      "%s, peer %d" % (what, p))
        others = np.ones(ids.shape[0], dtype=bool)
        others[row_offset:row_offset + nq] = False
        assert (ids[others] == SENTINEL).all() and (dists[others] == SENTINEL).all(), "%s: peer %d rows outside " \
            "[%d, %d) were written" % (what, p, row_offset, row_offset + nq)
        assert np.array_equal(flags, want_flags), "%s: peer %d flags %s" % (what, p, flags)
    # the oracle pads after the count; so every peer did
    k = ref[0].shape[1]
    pad = np.arange(k)[None, :] >= ref[2][:, None].astype(np.int64)
    assert (ref[0][pad] == PAD_ID).all() and (ref[1][pad].view(np.uint32) == INF_BITS).all()


def search_and_check(g, p, q, ef, k, n_peers, my_rank, row_offset, seq=1, what=""):
    import torch

    nq = q.shape[0]
    peers = Peers(n_peers, row_offset + nq + 3, k)
    keep = gather(p, peers, q, ef, k, my_rank, row_offset, seq)
    torch.cuda.synchronize()
    p.stream_status()
    ref = g.search_batch(q, ef, k, threads=8, with_stats=True)
    check_peers(peers, ref, keep[1], keep[2], my_rank, row_offset, seq, what)
    return keep[2].cpu().numpy()[:, 3]


@pytest.fixture(scope="module")
def c1(oracle):
    # BASELINE config 1 reduced (as in test_parity_gpu): random queries are all answered by the fast pass
    el, g, ib, eb, _ = build_fixture(oracle, "angular", 10_000, 32, seed=1234, num_neighbors=10, max_search=50)
    p = open_product(ib, "angular", eb)
    yield el, g, p
    p.close()


# ---- where the rows go ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_peers,my_rank,offset_rows,offset_extra", [(1, 0, 0, 0), (3, 2, 1, 0), (8, 5, 7, 13)])
def test_rows_land_at_the_offset_of_every_peer(c1, n_peers, my_rank, offset_rows, offset_extra):
    el, g, p = c1
    nq = 300
    q = random_vectors(nq, 32, seed=10 + n_peers)
    search_and_check(g, p, q, 50, 10, n_peers, my_rank, offset_rows * nq + offset_extra,
                     what="n_peers=%d rank=%d" % (n_peers, my_rank))


# ---- every engine family, several queries per warp ---------------------------------------------------------------
@pytest.mark.parametrize("kind,dim", [
    ("angular", 24),       # DistF32<0>
    ("angular", 128),      # DistF32<4>
    ("angular", 160),      # DistF32Generic
    ("angular_int", 100),  # DistI8
    ("embeddings", 50),    # DistSum
])
def test_every_engine_family(oracle, kind, dim):
    nq = queries_for_four_per_warp()
    el, g, ib, eb, mb = build_fixture(oracle, kind, 2000, dim, seed=dim, num_neighbors=16, max_search=40, threads=8)
    p = open_product(ib, kind, eb, mb)
    search_and_check(g, p, random_vectors(nq, dim, seed=dim + 3), 40, 10, 3, 1, nq + 5,
                     what="%s dim=%d" % (kind, dim))
    p.close()


# ---- every list size ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ef,k", [(40, 10), (40, 64), (40, 100), (200, 10), (200, 64), (400, 10), (400, 64),
                                  (976, 10), (976, 64), (1500, 10), (1500, 64)])
def test_every_list_size(c1, ef, k):
    # max_search 40 / 200 / 400 / 976 reach the fast lists R = 3 / 7 / 15 / 31, 1500 the generic list (R = 0);
    # k = 100 at max_search 40 pads 60 columns, over several 32-lane rounds
    el, g, p = c1
    q = random_vectors(200, 32, seed=ef + k)
    search_and_check(g, p, q, ef, k, 2, 1, 150, what="ef=%d k=%d" % (ef, k))


# ---- each pass ladder: the flag is published by whichever pass is last ------------------------------------------
def test_fast_pass_only_flag_comes_from_the_slow_kernels_early_exit(c1):
    el, g, p = c1
    passes = search_and_check(g, p, random_vectors(1000, 32, seed=4321), 50, 10, 3, 1, 1000, what="fast only")
    assert (passes == 0).all()


def test_mixed_pass_ladder(oracle):
    # the uniform-data recipe of test_parity_regimes_gpu.test_mixed_pass_ladder_in_one_launch, on a fresh handle
    el = oracle.Elements.angular(random_vectors(20_000, 24, seed=41))
    ib = oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8).to_bytes()
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", el.to_bytes())
    nq = queries_for_four_per_warp()
    passes = search_and_check(g, p, random_vectors(nq, 24, seed=42), 40, 10, 2, 0, 7, what="mixed ladder")
    assert (passes == 0).any() and (passes >= 1).any(), np.bincount(passes.astype(np.int64))
    p.close()


def test_slow_pass_serves_every_query(oracle):
    # the all-identical plateau of test_parity_regimes_gpu.test_slow_pass_serves_many_queries_per_cta
    n, dim = 400, 8
    el = oracle.Elements.angular(np.tile(random_vectors(1, dim, seed=5), (n, 1)))
    ib = index_from_lists(oracle, [[sorted({(i * 30 + j) % n for j in range(1, 31)} - {i}) for i in range(n)]])
    g = oracle.Granne.from_bytes(ib, el)
    p = open_product(ib, "angular", el.to_bytes())
    passes = search_and_check(g, p, random_vectors(256, dim, seed=6), 20, 10, 3, 2, 256, what="plateau")
    assert (passes == 2).all()
    p.close()


# ---- steps in flight, as in bench.py's step loop -----------------------------------------------------------------
def test_steps_in_flight_on_four_streams(c1):
    import torch

    el, g, p = c1
    nq, k, n_slots, n_steps = 400, 10, 4, 12
    streams = [torch.cuda.Stream() for _ in range(n_slots)]
    slots = [Peers(2, 2 * nq + 3, k) for _ in range(n_slots)]
    torch.cuda.synchronize()
    qs = [random_vectors(nq, 32, seed=500 + step) for step in range(n_steps)]
    keep = []
    for step in range(n_steps):
        slot = step % n_slots
        with torch.cuda.stream(streams[slot]):
            keep.append(gather(p, slots[slot], qs[step], 50, k, 1, nq, step + 1, stream=streams[slot]))
    torch.cuda.synchronize()
    p.stream_status()
    for slot in range(n_slots):
        step = slot + 2 * n_slots  # the last step that used this slot
        ref = g.search_batch(qs[step], 50, k, threads=8, with_stats=True)
        check_peers(slots[slot], ref, keep[step][1], keep[step][2], 1, nq, step + 1, "slot %d" % slot)
    for st in streams:
        p.release_stream(st)


# ---- error and empty rows ----------------------------------------------------------------------------------------
def test_nan_query_leaves_a_padded_row_and_the_flag_published(c1):
    import torch

    el, g, p = c1
    nq, bad = 300, 17
    q = random_vectors(nq, 32, seed=77)
    q[bad, 3] = np.nan
    peers = Peers(3, 2 * nq + 3, 10)
    stream = torch.cuda.Stream()
    keep = gather(p, peers, q, 50, 10, 2, nq, 41, stream=stream)
    torch.cuda.synchronize()
    with pytest.raises(granne_b200.GranneError) as ei:
        p.stream_status()
    assert ei.value.code == -6
    clean = q.copy()
    clean[bad] = 0.25  # the oracle rejects a NaN query; its row is replaced and left out of the parity check
    ref = g.search_batch(clean, 50, 10, threads=8, with_stats=True)
    others = np.delete(np.arange(nq), bad)
    check_peers(peers, ref, keep[1], keep[2], 2, nq, 41, "NaN batch", rows=others)
    assert keep[1].cpu().numpy()[bad] == 0
    for ids, dists, _ in peers.host():
        assert (ids[nq + bad] == PAD_ID).all() and (dists[nq + bad] == INF_BITS).all()
    # the next call on that stream is clean
    peers.fill()
    q2 = random_vectors(nq, 32, seed=78)
    keep = gather(p, peers, q2, 50, 10, 2, nq, 42, stream=stream)
    torch.cuda.synchronize()
    p.stream_status()
    check_peers(peers, g.search_batch(q2, 50, 10, threads=8, with_stats=True), keep[1], keep[2], 2, nq, 42,
                "after the NaN batch")
    p.release_stream(stream)


def test_index_without_layers_pads_every_row(oracle):
    import torch

    el = oracle.Elements.angular(random_vectors(5, 8, seed=1))
    p = open_product(index_from_lists(oracle, []), "angular", el.to_bytes())
    peers = Peers(2, 10, 4)
    keep = gather(p, peers, random_vectors(3, 8, seed=2), 10, 4, 1, 5, 9)
    torch.cuda.synchronize()
    p.stream_status()
    assert (keep[1].cpu().numpy() == 0).all()
    for ids, dists, flags in peers.host():
        assert (ids[5:8] == PAD_ID).all() and (dists[5:8] == INF_BITS).all()
        assert (ids[:5] == SENTINEL).all() and (ids[8:] == SENTINEL).all()
        assert (dists[:5] == SENTINEL).all() and (dists[8:] == SENTINEL).all()
        assert flags.tolist() == [SENTINEL, 9, SENTINEL, SENTINEL]
    p.close()


def test_zero_neighbors_touches_no_row_and_publishes(c1):
    import torch

    el, g, p = c1
    peers = Peers(2, 100, 1)  # one spare column: the call stores none of it
    keep = gather(p, peers, random_vectors(50, 32, seed=3), 50, 0, 0, 20, 5)
    torch.cuda.synchronize()
    p.stream_status()
    assert (keep[1].cpu().numpy() == 0).all()
    for ids, dists, flags in peers.host():
        assert (ids == SENTINEL).all() and (dists == SENTINEL).all()
        assert flags.tolist() == [5, SENTINEL, SENTINEL, SENTINEL]


def test_empty_slice_publishes_the_flag_on_the_callers_stream(c1):
    # a rank whose slice of an uneven batch is empty must still tell its peers that it is done
    import torch

    el, g, p = c1
    peers = Peers(3, 20, 10)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    p.search_batch_device_gather(torch.empty((0, 32), dtype=torch.float32, device="cuda"), peers.spec(1, 20, 7), 50,
                                 10, stream=stream.cuda_stream)
    stream.synchronize()
    p.stream_status()
    for ids, dists, flags in peers.host():
        assert (ids == SENTINEL).all() and (dists == SENTINEL).all()
        assert flags.tolist() == [SENTINEL, 7, SENTINEL, SENTINEL, SENTINEL]
    p.release_stream(stream)


# ---- validation ----------------------------------------------------------------------------------------------------
def _null(field, p):
    def edit(g):
        getattr(g, field)[p] = None

    return edit


@pytest.mark.parametrize("edit", [
    lambda g: setattr(g, "n_peers", 0),
    lambda g: setattr(g, "n_peers", 9),
    lambda g: setattr(g, "my_rank", 3),
    _null("ids", 2), _null("dists", 1), _null("flags", 0),
], ids=["no_peers", "nine_peers", "rank_out_of_range", "null_ids", "null_dists", "null_flags"])
def test_bad_descriptors_are_rejected_before_anything_runs(c1, edit):
    import torch

    el, g, p = c1
    peers = Peers(3, 40, 10)
    torch.cuda.synchronize()
    spec = peers.spec(1, 10, 3)
    edit(spec)
    q = torch.from_numpy(random_vectors(20, 32, seed=4)).cuda()
    before = p.launch_count()
    with pytest.raises(granne_b200.GranneError) as ei:
        p.search_batch_device_gather(q, spec, 50, 10)
    assert ei.value.code == INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert p.launch_count() == before and peers.untouched()


def test_null_descriptor_is_rejected(c1):
    import torch

    el, g, p = c1
    q = torch.from_numpy(random_vectors(20, 32, seed=4)).cuda()
    before = p.launch_count()
    rc = granne_b200.load_library().granne_b200_search_batch_device_gather(
        p._h, C.c_void_p(q.data_ptr()), 20, granne_b200.QUERY_RAW_F32, 50, 10, None, None, None, None)
    assert rc == INVALID_ARGUMENT and p.launch_count() == before


def test_stats_argument_is_checked(c1):
    import torch

    el, g, p = c1
    peers = Peers(1, 20, 10)
    q = torch.from_numpy(random_vectors(20, 32, seed=4)).cuda()
    for bad in (torch.empty((20, 4), dtype=torch.int32, device="cuda"),
                torch.empty((19, 4), dtype=torch.int64, device="cuda"),
                torch.empty((4, 20), dtype=torch.int64, device="cuda").t(),
                torch.empty((20, 4), dtype=torch.int64)):
        with pytest.raises(ValueError):
            p.search_batch_device_gather(q, peers.spec(0, 0, 1), 50, 10, stats=bad)
    torch.cuda.synchronize()
    assert peers.untouched()
