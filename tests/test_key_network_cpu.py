"""The bitonic network the exact family sorts and merges make_key keys with (granne_b200/csrc/keys.cuh), modelled index
for index on the CPU (tests/helpers/key_network.py) and compared with sorted(): the sort of every power-of-two length
the kernels use, the merge of within_kernel's segment keys with a running list, and range_finish_kernel's tiles plus
global stages.  The GPU tests check the kernels' outputs against the oracle; these check the network itself, at every
size, with ~0 padding and with the duplicate keys the filter-id sort meets."""
import os
import random

import pytest

from helpers.key_network import PAD, key_merge, key_sort, next_pow2, range_finish, sort_steps

KEYS_CUH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "granne_b200", "csrc", "keys.cuh")

K_EXACT_MAX_K = 1024   # kExactMaxK: the largest k of the within path
K_SEL_SLOTS = 4096     # kExactSelSlots: exact_select_kernel's flush


def random_keys(rng, n, dup):
    """n keys below ~0; with dup, drawn from few values so that most keys repeat."""
    hi = max(2, n // 8) if dup else 1 << 63
    return [rng.randrange(hi) for _ in range(n)]


def test_model_uses_the_device_comparators():
    src = open(KEYS_CUH).read()
    for expr in ("j == k2 / 2 ? k2 - 1 : j", "2 * t - (t & (j - 1)), l = i ^ m", "t < p / 2", "k2 <= p", "x > y",
                 "key_steps(g, keys, p, k2, k2 / 2)", "key_steps(g, keys, p, p, p / 2)",
                 "key_steps(g, keys, p, 4 * j, j)"):
        assert expr in src, expr


@pytest.mark.parametrize("p", [1 << e for e in range(13)])
def test_steps_are_disjoint_and_in_range(p):
    for pairs in sort_steps(p):
        seen = [i for pair in pairs for i in pair]
        assert len(seen) == len(set(seen)) == p
        assert all(0 <= i < j < p for i, j in pairs)


@pytest.mark.parametrize("p", [1 << e for e in range(13)])
def test_sort_equals_sorted(p):
    rng = random.Random(p)
    for n in sorted({0, 1, p // 2 + 1, p - 1, p, rng.randint(0, p), rng.randint(0, p)}):
        if n > p:
            continue
        for dup in (False, True):
            keys = random_keys(rng, n, dup)
            s = keys + [PAD] * (p - n)
            key_sort(s, p)
            assert s == sorted(keys) + [PAD] * (p - n), (p, n, dup)


def test_sort_filter_ids():
    # exact_chunk_filters_kernel: u32 filter ids of up to 1024 queries, ~0u past the chunk or for an invalid entry
    rng = random.Random(7)
    for qc in (1, 5, 512, 1000, 1024):
        ids = [rng.randrange(4) if rng.random() < 0.9 else 0xFFFFFFFF for _ in range(qc)]
        s = ids + [0xFFFFFFFF] * (1024 - qc)
        key_sort(s, 1024)
        assert s == sorted(s)
        assert s == sorted(ids) + [0xFFFFFFFF] * (1024 - qc)


def test_select_flush():
    # exact_flush: the running list (k keys, then ~0 to kExactMaxK), the candidates, ~0 to kExactSelSlots
    for k, cand in ((1, 0), (10, 2048), (1024, 3072), (100, 1)):
        keys = random.Random(k).sample(range(1 << 40), k + cand)
        running = sorted(keys[:k])
        s = running + [PAD] * (K_EXACT_MAX_K - k) + keys[k:] + [PAD] * (K_SEL_SLOTS - K_EXACT_MAX_K - cand)
        key_sort(s, K_SEL_SLOTS)
        assert s[:k] == sorted(keys)[:k]


@pytest.mark.parametrize("k", sorted({k for k in range(1, K_EXACT_MAX_K + 1) if k & (k - 1) == 0} | {3, 10, 100, 1000}))
def test_merge_equals_sorted(k):
    # within_kernel: keys[0, P) the segment's mp keys below the running k-th key, ascending, then ~0; keys[P, 2P) the
    # running list (k entries, some still ~0), ascending, then ~0 to P
    P = next_pow2(k)
    rng = random.Random(k)
    for _ in range(4):
        listed = rng.randint(0, k)
        mp = rng.randint(1, P)
        pool = rng.sample(range(1 << 40), listed + mp)
        run = sorted(pool[:listed]) + [PAD] * (P - listed)
        seg = sorted(pool[listed:]) + [PAD] * (P - mp)
        s = seg + run
        key_merge(s, 2 * P)
        assert s == sorted(pool) + [PAD] * (2 * P - listed - mp), (k, listed, mp)


@pytest.mark.parametrize("tile", [4, 16, 64])
def test_range_finish_equals_sorted(tile):
    rng = random.Random(tile)
    lengths = {0, 1, 2, tile - 1, tile, tile + 1, 2 * tile, 2 * tile + 1, 4 * tile - 1, 8 * tile + 3, 16 * tile}
    lengths |= {rng.randint(tile + 1, 16 * tile) for _ in range(6)}
    for n in sorted(lengths):
        for dup in (False, True):
            keys = random_keys(rng, n, dup)
            assert range_finish(keys, tile) == sorted(keys), (tile, n, dup)
