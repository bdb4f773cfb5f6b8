"""Index-for-index model of the bitonic network in granne_b200/csrc/keys.cuh (key_sort, key_merge, key_clean) and of
range_finish_kernel's use of it for segments longer than a shared-memory tile (granne_b200/csrc/range_kernels.cuh).

The loop bounds and comparator pairs are the device code's (key_steps): stage k2 is the steps j = k2 / 2 .. 1, and
comparator t of step j joins i = 2t - (t & (j - 1)) with its mirror i ^ (k2 - 1) (the flip step, j = k2 / 2) or with
i + j (a half-cleaner).  Each comparator puts the smaller key first.  The comparators of one step touch disjoint
positions (sort_steps lets a test check that), so running them one after the other gives what the threads of a group
give between two barriers, whichever thread takes which comparator (a block's threads take comparators, a warp's lanes
the lower ends of the pairs)."""

PAD = (1 << 64) - 1  # ~0: the key that pads a list to a power of two


def next_pow2(n):
    """rerank_key_slots (rerank_kernels.cuh): the next power of two, at least 1."""
    p = 1
    while p < n:
        p <<= 1
    return p


def step_pairs(p, k2, j):
    """The comparators of step j of stage k2 over p keys: the flip step (partner i ^ (k2 - 1)) when j = k2 / 2, else
    the half-cleaner j (partner i + j, which is i ^ j: bit j of i is clear)."""
    m = k2 - 1 if j == k2 // 2 else j
    for t in range(p // 2):
        i = 2 * t - (t & (j - 1))
        yield i, i ^ m


def sort_steps(p):
    """Every step of key_sort over p keys, in order, as its list of comparator pairs."""
    k2 = 2
    while k2 <= p:
        j = k2 // 2
        while j > 0:
            yield list(step_pairs(p, k2, j))
            j >>= 1
        k2 <<= 1


def _run(keys, pairs):
    for i, j in pairs:
        if keys[i] > keys[j]:
            keys[i], keys[j] = keys[j], keys[i]


def key_steps(keys, p, k2, j):
    while j > 0:
        _run(keys, step_pairs(p, k2, j))
        j >>= 1


def key_sort(keys, p):
    k2 = 2
    while k2 <= p:
        key_steps(keys, p, k2, k2 // 2)
        k2 <<= 1


def key_merge(keys, p):
    key_steps(keys, p, p, p // 2)


def key_clean(keys, p, j):
    key_steps(keys, p, 4 * j, j)


def range_finish(keys, tile):
    """The segment's keys as range_finish_kernel leaves them, with `tile` keys per shared-memory tile (kRangeTile):
    one tile sort when the padded length fits a tile; else every tile sorted, then per wider stage k2 its flip step and
    its half-cleaners down to `tile` in global memory, and the half-cleaners below `tile` tile by tile."""
    seg = list(keys)
    n = len(seg)
    if n < 2:
        return seg
    p = 2
    while p < n:
        p <<= 1
    if p <= tile:
        s = seg + [PAD] * (p - n)
        key_sort(s, p)
        return s[:n]

    def per_tile(op):
        for t0 in range(0, n, tile):
            s = [seg[t0 + i] if t0 + i < n else PAD for i in range(tile)]
            op(s)
            for i in range(min(tile, n - t0)):
                seg[t0 + i] = s[i]

    def global_run(pairs):  # range_global_cmpswap: a partner at or past n is a ~0 key
        _run(seg, ((i, j) for i, j in pairs if j < n))

    per_tile(lambda s: key_sort(s, tile))
    k2 = 2 * tile
    while k2 <= p:
        j = k2 // 2
        while j >= tile:
            global_run(step_pairs(p, k2, j))
            j >>= 1
        per_tile(lambda s: key_clean(s, tile, tile // 2))
        k2 <<= 1
    return seg
