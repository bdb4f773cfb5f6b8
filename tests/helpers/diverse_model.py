"""A lane-level CPU model of diverse_kernel's selection by elimination (granne_b200/csrc/diverse_kernels.cuh), for
checking the scheme against the reference's sequential select_neighbors (src/index/mod.rs:849-883) without a GPU.

The model keeps the kernel's state as the kernel does: the alive (id, distance) pairs compacted at the front of one
list, a round that keeps the first alive candidate and judges the later ones in batches of 32 lanes, a ballot of the
survivors and their in-place compaction by prefix count."""


def select_by_elimination(ids, dists, k, pair_dist):
    """(kept ids, kept dists, pair distances computed) of select_neighbors(list, k) for one list ascending by distance.
    pair_dist(s, c) is the distance of candidate c to the kept element s (dist_to_element(c, get(s)))."""
    n = len(ids)
    if n <= k:
        return list(ids), list(dists), 0
    if k == 0:
        return [], [], 0
    alive_id, alive_d = list(ids), list(dists)
    m, out_i, out_d, pairs = n, [], [], 0
    while True:
        s = alive_id[0]
        out_i.append(s)
        out_d.append(alive_d[0])
        if len(out_i) == k or m == 1:
            break
        kept = 0
        for b in range(1, m, 32):
            nb = min(32, m - b)
            lanes = [(alive_id[b + t], alive_d[b + t]) for t in range(nb)]
            ds = [pair_dist(s, c) for c, _ in lanes]
            pairs += nb
            keep = [d <= dsc for (_, d), dsc in zip(lanes, ds)]
            ballot = sum(1 << t for t in range(nb) if keep[t])
            for t in range(nb):
                if keep[t]:
                    p = kept + bin(ballot & ((1 << t) - 1)).count("1")
                    alive_id[p], alive_d[p] = lanes[t]
            kept += bin(ballot).count("1")
        if kept == 0:
            break
        m = kept
    return out_i, out_d, pairs


def select_sequential(ids, dists, k, pair_dist):
    """The reference's loop, stated directly: keep candidate j if d(q, j) <= d(s, j) for every s kept so far."""
    if len(ids) <= k:
        return list(ids), list(dists)
    out_i, out_d = [], []
    for j, d in zip(ids, dists):
        if len(out_i) >= k:
            break
        if all(d <= pair_dist(s, j) for s in out_i):
            out_i.append(j)
            out_d.append(d)
    return out_i, out_d
