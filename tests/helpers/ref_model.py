"""A third statement of the reference's arithmetic and search loop, in NumPy, for checking the CPU oracle
(oracle/granne_oracle.cpp) and the CUDA kernels against something neither of them was written from.

It imports numpy and the standard library only, and shares no code with the oracle, the kernels or the other test
helpers: a misreading of the reference made in both of those would otherwise pass every parity test.  Each function
cites the reference code (src/...) whose semantics it restates.

Every f32 operation is the correctly rounded IEEE one: NumPy's float32 add, subtract, multiply, divide and sqrt are,
and the fused multiply-add, which NumPy lacks, is built exactly below from float64 (fma_f32).
"""
import heapq

import numpy as np

F32, F64 = np.float32, np.float64
_TWO_128 = 2.0 ** 128  # where float32 rounding of a finite value stops being finite


# ---- arithmetic ------------------------------------------------------------------------------------------------------
def fma_f32(a, b, c):
    """f32::mul_add (math.rs:23,38): a*b + c rounded once to float32, element-wise.

    The float64 product of two float32 values is exact (24 + 24 bits).  The float64 sum s = p + c is not, but TwoSum
    gives its error e exactly (p + c == s + e).  Rounding s to float32 is then the single rounding of p + c except when
    s lands exactly on a float32 rounding midpoint while e != 0: the true sum lies on e's side of that midpoint, so the
    neighbour on e's side is the answer.  Float32 midpoints, subnormal ones included, are float64 values, so no other
    case can round differently."""
    a64, b64, c64 = (np.asarray(v, dtype=F32).astype(F64) for v in (a, b, c))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a64 * b64
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(F32)
        r64 = r.astype(F64)
        # a finite sum that rounded up to infinity was rounded to 2^128, the next float32 "value" past FLT_MAX
        r64 = np.where(np.isinf(r) & np.isfinite(s), np.copysign(_TWO_128, s), r64)
        toward = np.where(s > r64, F32(np.inf), F32(-np.inf))
        other = np.nextafter(r, toward)  # the float32 neighbour of r on s's side
        mid = (r64 + other.astype(F64)) * 0.5 == s
        fix = mid & (e != 0) & np.isfinite(e) & ((e > 0) == (other.astype(F64) > r64))
    return np.where(fix, other, r).astype(F32)


def dot_f32(x, y):
    """dot_product_f32 (math.rs:16-42) of every row pair, broadcast over the leading axes of x and y (last axis: the
    vector): 32 chunk lanes accumulated with FMA over the full 32-wide chunks, the 32 partials summed in lane order,
    then one FMA per remainder component, in order."""
    x, y = np.asarray(x, dtype=F32), np.asarray(y, dtype=F32)
    dim = x.shape[-1]
    full = dim // 32
    shape = np.broadcast_shapes(x.shape[:-1], y.shape[:-1])
    lanes = np.zeros(shape + (32,), dtype=F32)
    for ch in range(full):
        lanes = fma_f32(x[..., ch * 32:(ch + 1) * 32], y[..., ch * 32:(ch + 1) * 32], lanes)
    r = np.zeros(shape, dtype=F32)
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(32):
            r = (r + lanes[..., i]).astype(F32)
    for t in range(full * 32, dim):
        r = fma_f32(x[..., t], y[..., t], r)
    return r


def normalize_f32(rows):
    """normalize_f32 (math.rs:124-150) of each row: divide by sqrt(dot(x, x)) when that norm is > 0.  A row whose
    norm underflows to 0 stays as it is; one whose squared norm overflows is divided by +inf (finite parts -> +-0)."""
    x = np.array(rows, dtype=F32, ndmin=2)
    norm = np.sqrt(dot_f32(x, x)).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where((norm > 0)[:, None], (x / norm[:, None]).astype(F32), x)
    return out.astype(F32)


def quantize(rows):
    """angular_int::Vector::quantize (angular_int.rs:28-45) of each row: x * 127 / max|x| in f32, then `as i8`, which
    truncates toward zero, saturates at -128 and 127, and maps NaN to 0.  An empty row's max is 127."""
    x = np.array(rows, dtype=F32, ndmin=2)
    mx = np.abs(x).max(axis=1) if x.shape[1] else np.full(x.shape[0], 127, dtype=F32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        v = ((x * F32(127.0)).astype(F32) / mx[:, None]).astype(F32)
        q = np.trunc(np.nan_to_num(v, nan=0.0, posinf=127.0, neginf=-128.0))
    return np.clip(q, -128, 127).astype(np.int8)


def r_dx_dy_i8(x, y):
    """dot_product_and_squared_norms_i8 (math.rs:59-89) as exact integers: (x.y, x.x, y.y), broadcast like dot_f32."""
    x = np.asarray(x).astype(np.int64)
    y = np.asarray(y).astype(np.int64)
    return (x * y).sum(-1), (x * x).sum(-1), (y * y).sum(-1)


def dist_i8(x, y):
    """angular_int Vector::dist (angular_int.rs:47-59): the exact i32 sums each rounded once to f32, then
    1 - r / (sqrt(dx) * sqrt(dy)) in f32 with a NaN quotient (0 / 0) taken as r = 0, clamped at 0."""
    return _dist_from_sums(*r_dx_dy_i8(x, y))


def _dist_from_sums(r, dx, dy):
    r, dx, dy = r.astype(F32), dx.astype(F32), dy.astype(F32)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = (r / (np.sqrt(dx).astype(F32) * np.sqrt(dy).astype(F32)).astype(F32)).astype(F32)
    q = np.where(np.isnan(q), F32(0.0), q)
    return np.maximum(F32(0.0), (F32(1.0) - q).astype(F32)).astype(F32)


def dist_f32(x, y):
    """angular Vector::dist (angular.rs:63-74): 1 - dot_product_f32(x, y) in f32, clamped at 0."""
    return np.maximum(F32(0.0), (F32(1.0) - dot_f32(x, y)).astype(F32)).astype(F32)


def sum_embedding(table, terms):
    """SumEmbeddings::get_embedding_internal (embeddings/mod.rs:124-143): a copy of the first term's row, then each
    further term's row added in order (sum_into_f32, math.rs:92-116); no terms: a row of zeros."""
    table = np.asarray(table, dtype=F32)
    if len(terms) == 0:
        return np.zeros(table.shape[1], dtype=F32)
    x = table[terms[0]].copy()
    for t in terms[1:]:
        x = (x + table[t]).astype(F32)
    return x


def element_rows(kind, raw):
    """Vector::from for raw f32 rows (angular.rs:55-61, angular_int.rs:19-23): what an index stores and what a raw
    query becomes.  "embeddings" elements and queries are angular vectors (embeddings/mod.rs:164-174)."""
    return quantize(raw) if kind == "angular_int" else normalize_f32(raw)


def sum_elements(table, term_lists):
    """The rows of a SumEmbeddings container as ElementContainer::get makes them (embeddings/mod.rs:164-170)."""
    return normalize_f32(np.stack([sum_embedding(table, t) for t in term_lists]))


def distances(kind, rows, queries):
    """[q, i] = dist(element i, query q) for element rows (normalised f32 or i8) and query elements of that kind."""
    rows, queries = np.asarray(rows), np.asarray(queries)
    if kind != "angular_int":
        step = max(1, (1 << 22) // max(1, 32 * rows.shape[0]))  # queries per block: bounded temporaries
        return np.concatenate([dist_f32(rows[None, :, :], queries[q:q + step, None, :])
                               for q in range(0, queries.shape[0], step)] or [np.zeros((0, rows.shape[0]), F32)])
    x, y = rows.astype(np.int64), queries.astype(np.int64)  # integer matmul: exact
    r = y @ x.T
    return _dist_from_sums(r, (x * x).sum(1)[None, :] + 0 * r, (y * y).sum(1)[:, None] + 0 * r)


# ---- ranking ---------------------------------------------------------------------------------------------------------
def rank(d, ids, k):
    """The first min(k, |set(ids)|) of the distinct ids by (d[id], id): the order of into_sorted_vec over
    (NotNan<f32>, usize) tuples (src/index/mod.rs:1036).  Returns [(id, dist)]."""
    u = np.unique(np.asarray(ids, dtype=np.int64))
    order = np.lexsort((u, np.asarray(d, dtype=F32)[u]))[:k]
    return [(int(u[o]), F32(d[u[o]])) for o in order]


def rank_prefix(d, n, k):
    """Exact k-NN over the container prefix [0, n)."""
    return rank(d, np.arange(n), k)


# ---- search ----------------------------------------------------------------------------------------------------------
class _Count:
    def __init__(self):
        self.n_dist = self.n_expand = self.n_nbr = 0


def _search_layer(adj, entry, d, max_search, cnt, scored=None):
    """search_for_neighbors (src/index/mod.rs:999-1037) with its max_size_heap.rs result heap.  d[i] is the query's
    distance to element i, looked up (and counted) where the reference calls dist_to_element; adj[i] is element i's
    neighbour list in this layer.  Every order in the loop is total on (dist, id), so the result is unique."""
    cnt.n_dist += 1
    visited = {entry}
    if scored is not None:
        scored.add(entry)
    pq = [(float(d[entry]), entry)]
    res = []  # max-heap of (dist, id) kept as (-dist, -id)
    while pq:
        dd, idx = heapq.heappop(pq)
        if len(res) >= max_search and dd > -res[0][0]:  # compares the distance only
            break
        if len(res) < max_search:  # MaxSizeHeap::push (max_size_heap.rs:18-33)
            heapq.heappush(res, (-dd, -idx))
        elif (dd, idx) < (-res[0][0], -res[0][1]):
            heapq.heapreplace(res, (-dd, -idx))
        nbrs = adj[idx]
        cnt.n_expand += 1
        cnt.n_nbr += len(nbrs)
        for j in nbrs:
            j = int(j)
            if j in visited:
                continue
            visited.add(j)
            cnt.n_dist += 1
            if scored is not None:
                scored.add(j)
            dj = float(d[j])
            if len(res) < max_search or dj < -res[0][0]:
                heapq.heappush(pq, (dj, j))
    return sorted((-a, -b) for a, b in res)


def search(layers, d, max_search, k):
    """Granne::search (src/index/mod.rs:140-150, 962-997): find_entrypoint through the top layers with max_search 1
    from element 0, then search_for_neighbors in the bottom layer, first k results.  layers: neighbour lists, top layer
    first.  Returns (results [(id, dist)], stats (n_dist, n_expand, n_nbr) over all layers — columns 0..2 of
    include/granne_b200.h:77-82 —, S(q): the bottom-layer elements whose distance was computed)."""
    cnt, scored = _Count(), set()
    if not layers:
        return [], (0, 0, 0), scored
    entry = 0
    for adj in layers[:-1]:
        entry = _search_layer(adj, entry, d, 1, cnt)[0][1]
    res = _search_layer(layers[-1], entry, d, max_search, cnt, scored)
    return [(i, F32(x)) for x, i in res[:k]], (cnt.n_dist, cnt.n_expand, cnt.n_nbr), scored


# ---- the calls of include/granne_b200.h that are not reference functions ------------------------------------------------
def within(d, ids, k):
    """granne_b200_exact_search_within_batch: the list's distinct ids ranked by (distance, id)."""
    return rank(d, ids, k)


def filtered(layers, d, max_search, k, admitted):
    """granne_b200_search_filtered_batch (granne_b200.h:254-266): S(q) ∩ A ranked by (distance, id); stats are the
    unfiltered search's."""
    _, stats, scored = search(layers, d, max_search, 0)
    return rank(d, [i for i in scored if admitted[i]], k), stats


def rerank(layers, d_stage1, d_stage2, max_search, num_candidates, k):
    """granne_b200_search_rerank_batch: the ids of search(max_search, num_candidates) over the stage-1 distances,
    ranked by their stage-2 distances."""
    res, stats, _ = search(layers, d_stage1, max_search, num_candidates)
    return rank(d_stage2, [i for i, _ in res], k), stats


def excluding_self(results, self_id, k):
    """QUERY_ID_EXCLUDING (granne_b200.h:72-75): a call's k + 1 results without the entry of id self_id, cut to k."""
    return [(i, x) for i, x in results if i != self_id][:k]


def merge(parts, bases, k):
    """The multi-handle merge: per-part results [(local id, dist)] with global id = base + local id, the first k by
    (dist, global id)."""
    allr = [(F32(x), b + i) for res, b in zip(parts, bases) for i, x in res]
    return [(i, x) for x, i in sorted(allr, key=lambda t: (float(t[0]), t[1]))[:k]]


def knn_graph(layers, dmat, max_search, k, exact=False):
    """Granne.knn_graph: for every element i of the index, the by-id search (exact: exact k-NN) of i without i."""
    n = len(layers[-1]) if layers else 0
    out = []
    for i in range(n):
        res = rank_prefix(dmat[i], n, k + 1) if exact else search(layers, dmat[i], max_search, k + 1)[0]
        out.append(excluding_self(res, i, k))
    return out


def as_arrays(results, k, id_dtype=np.uint32):
    """[[(id, dist)]] -> (ids padded with all-ones, dists padded with +inf, counts), the calls' output layout."""
    nq = len(results)
    ids = np.full((nq, k), np.iinfo(id_dtype).max, dtype=id_dtype)
    dists = np.full((nq, k), np.inf, dtype=F32)
    counts = np.zeros(nq, dtype=np.uint32)
    for q, res in enumerate(results):
        counts[q] = len(res)
        for j, (i, x) in enumerate(res):
            ids[q, j] = i
            dists[q, j] = x
    return ids, dists, counts
