"""Synthetic per-shard result tiles for the range-partitioned k-way merge, and the merge stated as a plain sort.

Distances come from a five-value set that holds both zeros, so equal distances meet inside a part and across parts and
the global id has to decide.  Every part's row has a random length from 0 to k and is padded after it, so short shards
sit anywhere in the part list."""
import numpy as np

PAD_ID = 0xFFFFFFFF
PAD_GID = 0xFFFFFFFFFFFFFFFF
INF_BITS = 0x7F800000
TIE_DISTANCES = np.array([0.0, -0.0, 0.25, 0.5, 1.0], dtype=np.float32)


def tie_bases(P):
    """One global id offset per part: not ascending, all above 2**32, and far enough apart that global ids stay
    unique."""
    return [(2 ** 32 + 5) + (((P - 1 - p) * 37) % P) * 2 ** 33 for p in range(P)]


def make_tiles(P, nq, k, seed):
    """(ids uint32 [P, nq, k], dists float32 [P, nq, k]): each row sorted by (distance, local id) with unique local ids,
    then 0xFFFFFFFF / +inf."""
    rng = np.random.default_rng(seed)
    ids = np.full((P, nq, k), PAD_ID, dtype=np.uint32)
    dists = np.full((P, nq, k), np.inf, dtype=np.float32)
    lengths = rng.integers(0, k + 1, size=(P, nq))
    for p in range(P):
        for q in range(nq):
            n = int(lengths[p, q])
            lid = np.unique(rng.integers(0, PAD_ID, size=n, dtype=np.uint64))  # may drop a repeat: still 0..k
            d = TIE_DISTANCES[rng.integers(0, TIE_DISTANCES.size, size=lid.size)]
            row = sorted(zip(d.tolist(), lid.tolist()))
            ids[p, q, :len(row)] = [i for _, i in row]
            dists[p, q, :len(row)] = [x for x, _ in row]
    return ids, dists


def reference_merge(ids, dists, bases, k):
    """The first k of sorted((distance, base[p] + local id)) over every part: (uint64 ids padded with UINT64_MAX,
    float32 dists padded with +inf).  The distance kept is the chosen entry's own, so -0.0 stays -0.0."""
    P, nq, kk = ids.shape
    out_ids = np.full((nq, k), PAD_GID, dtype=np.uint64)
    out_d = np.full((nq, k), np.inf, dtype=np.float32)
    for q in range(nq):
        cand = [(float(dists[p, q, j]), int(bases[p]) + int(ids[p, q, j]), dists[p, q, j])
                for p in range(P) for j in range(kk) if ids[p, q, j] != PAD_ID]
        best = sorted(cand, key=lambda t: (t[0], t[1]))[:k]
        out_ids[q, :len(best)] = [g for _, g, _ in best]
        out_d[q, :len(best)] = [d for _, _, d in best]
    return out_ids, out_d
