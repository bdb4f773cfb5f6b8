"""Containers past the 32-bit row offsets whose exact answers the NumPy model (ref_model.py) computes from a few
thousand distinct rows, for tests/test_wide_offsets_*.py.

Row i of a container of n rows is palette[h(i)], h(i) = ((i * 2654435761) mod 2^32) mod P, except at the planted ids,
which hold rows of their own: each is one query's element plus a little noise, nearer to that query than every
palette row.  The planted ids are the ids on each side of every byte boundary 2^k the container crosses, both ends of
the id range and random ids past 2^22.  One planted id past the last boundary holds an exact copy of id 1's row, so a
tie crosses the boundary, and palette row `twin` has the same distance to query 0 as palette row 0 (it differs only
where query 0 is zero).  The palette holds the edge rows of edge_raw_f32 (and, for i8 containers, edge_i8_rows).

The model keeps the P + |S| distinct element rows and each query's distance to them; a query's distance to every
element is then one gather (`Wide.dvec`).  `rank` ranks a distance vector like M.rank without sorting all of it, and
`sparse_index` writes the image of a graph whose rows are nearly all empty without a Python list per row."""
import json

import numpy as np

from helpers import ref_model as M
from helpers.data import edge_i8_rows, edge_raw_f32, random_vectors

F32 = np.float32
HASH_MUL = 2654435761
PALETTE = 4093          # a prime: h spreads the ids of each palette row over the whole range
NUM_QUERIES = 16
NUM_RANDOM_PLANTED = 48
RANDOM_PLANTED_FROM = 1 << 22
PLANTED_NOISE = {"angular": 1e-3, "angular_int": 3e-2}   # i8: large enough to survive quantisation
NEAR_NOISE = 0.3        # palette row q: query q's element plus this much noise, the nearest palette row of query q


def row_bytes(kind, dim, f32_floats=4, i8_bytes=32):
    """Bytes per staged row (DESIGN §3): f32 rows padded to a multiple of f32_floats floats, i8 rows to a multiple of
    i8_bytes bytes."""
    if kind == "angular_int":
        return -(-dim // i8_bytes) * i8_bytes
    return -(-dim // f32_floats) * f32_floats * 4


def first_id_at(boundary, stride):
    """The first id whose row starts at or past byte `boundary`."""
    return -(-boundary // stride)


def boundary_ids(boundaries, stride):
    """b - 1, b and b + 1 for the first id b at or past each byte boundary."""
    return sorted({first_id_at(x, stride) + o for x in boundaries for o in (-1, 0, 1)})


def hash_label(ids, p=PALETTE):
    """h(i) for an int64 array (numpy or torch) of ids."""
    return ((ids * HASH_MUL) & 0xFFFFFFFF) % p


def rank(d, k, ids=None):
    """M.rank(d, ids, k) (ids None: every id of d, M.rank_prefix) without sorting all of d: the k smallest by
    argpartition, widened to every id whose distance equals the k-th (ties and +-0 compare equal, as in M.rank's float
    order), then lexsorted by (distance, id)."""
    d = np.asarray(d, dtype=F32)
    if ids is not None:
        ids = np.unique(np.asarray(ids, dtype=np.int64))
    vals = d if ids is None else d[ids]
    if k <= 0 or vals.size == 0:
        return []
    keep = np.arange(vals.size)
    if k < vals.size:
        kth = vals[np.argpartition(vals, k - 1)[k - 1]]
        keep = np.flatnonzero(vals <= kth)
    sel, vals = (keep if ids is None else ids[keep]), vals[keep]
    order = np.lexsort((sel, vals))[:k]
    return [(int(sel[o]), F32(vals[o])) for o in order]


class Bits:
    """admitted[i] of one packed filter (uint32 words, id i is bit i % 32 of word i // 32)."""

    def __init__(self, words):
        self.words = words

    def __getitem__(self, i):
        return bool((int(self.words[i >> 5]) >> (i & 31)) & 1)


def words_of(ids, n):
    """The packed filter (uint32 [ceil(n / 32)]) that admits exactly `ids`."""
    ids = np.asarray(ids, dtype=np.int64)
    w = np.zeros((n + 31) // 32, dtype=np.uint32)
    np.bitwise_or.at(w, ids >> 5, (np.uint32(1) << (ids & 31).astype(np.uint32)))
    return w


class Wide:
    """The model of one container: kind, dim, n, the planted ids and the element rows each id holds."""

    def __init__(self, kind, dim, n, boundaries, seed, i8_edges=True, stride=None, random_from=RANDOM_PLANTED_FROM):
        """boundaries: the byte offsets 2^k whose neighbouring ids are planted, for rows of `stride` bytes (default:
        this container's own rows; a re-rank case plants the boundaries of its attached rows).  The random planted
        ids are drawn from [random_from, n)."""
        self.kind, self.dim, self.n = kind, dim, n
        self.stride = stride or row_bytes(kind, dim)
        self.boundaries = list(boundaries)
        rng = np.random.default_rng(seed)
        nq = NUM_QUERIES
        raw_q = random_vectors(nq, dim, seed)
        raw_q[0, dim // 2:] = 0.0                  # query 0 is zero on its upper half (the twin rows)
        self.raw_queries = raw_q

        def noisy(base, scale):
            x = base.astype(np.float64)
            e = rng.standard_normal(x.shape) * (scale * np.linalg.norm(x, axis=-1, keepdims=True) / np.sqrt(dim))
            return (x + e).astype(F32)

        # palette: near rows of each query, the twin of palette row 0, edge rows, random rows
        pal = random_vectors(PALETTE, dim, seed + 1)
        pal[:nq] = noisy(raw_q, NEAR_NOISE)
        self.twin = nq
        pal[nq] = pal[0]
        pal[nq, dim // 2:] *= F32(-1)
        pal[nq + 1:nq + 13] = edge_raw_f32(12, dim, seed + 2)
        self.i8_edge_slots = (nq + 13, nq + 21) if (kind == "angular_int" and i8_edges) else None

        # planted ids: around every boundary, both ends, random ids past 2^22
        fixed = boundary_ids(self.boundaries, self.stride) + [0, 1, n - 2, n - 1]
        assert max(fixed) < n and min(fixed) >= 0
        extra = random_from + rng.choice(n - random_from, size=NUM_RANDOM_PLANTED, replace=False)
        self.planted = np.unique(np.concatenate([np.asarray(fixed, dtype=np.int64), extra]))
        self.boundary = np.asarray(boundary_ids(self.boundaries, self.stride), dtype=np.int64)
        s = self.planted.size
        self.planted_query = np.arange(s) % nq
        self.planted_label = PALETTE + np.arange(s)
        # the last planted id at or past the last boundary copies id 1's row exactly
        self.copy_id = int(first_id_at(self.boundaries[-1], self.stride) + 1)
        ci, oi = np.searchsorted(self.planted, [self.copy_id, 1])
        self.planted_query[ci] = self.planted_query[oi]
        self.planted_label[ci] = self.planted_label[oi]
        planted_raw = noisy(raw_q[self.planted_query], PLANTED_NOISE[kind])
        self.raw_distinct = np.concatenate([pal, planted_raw])
        self.distinct = self.elements(kind)
        self.queries = M.element_rows(kind, raw_q)
        self.D = M.distances(kind, self.distinct, self.queries)        # [q, distinct row]
        self.check_premises(self.D)

    def elements(self, kind):
        """The distinct element rows of `kind` (the re-rank attaches the angular rows of an angular_int container)."""
        el = M.element_rows(kind, self.raw_distinct)
        if kind == "angular_int" and self.i8_edge_slots:
            a, b = self.i8_edge_slots
            el[a:b] = edge_i8_rows(b - a, self.dim, 3)   # zero, +-127 and -128 rows
        return el

    def check_premises(self, D):
        """Each query's planted rows are nearer to it than every palette row, every other query's planted rows are
        not, and the twin ties with palette row 0 for query 0."""
        for q in range(D.shape[0]):
            mine = self.planted_label[self.planted_query == q]
            others = self.planted_label[self.planted_query != q]
            assert D[q, mine].max() < D[q, :PALETTE].min(), q
            assert D[q, mine].max() < D[q, others].min(), q
        assert D[0, self.twin] == D[0, 0]
        assert np.argmin(D[0, :PALETTE]) in (0, self.twin)

    def labels(self, ids):
        """The distinct row each id holds."""
        ids = np.asarray(ids, dtype=np.int64)
        lab = hash_label(ids)
        pos = np.clip(np.searchsorted(self.planted, ids), 0, self.planted.size - 1)
        hit = self.planted[pos] == ids
        return np.where(hit, self.planted_label[pos], lab)

    def all_labels(self):
        lab = hash_label(np.arange(self.n, dtype=np.int64)).astype(np.int32)
        lab[self.planted] = self.planted_label
        return lab

    def rows(self, ids, kind=None):
        return (self.distinct if kind is None else self.elements(kind))[self.labels(ids)]

    def __getitem__(self, ids):   # element rows by id (assert_within_f64_bound)
        return self.rows(ids)

    def device_rows(self, torch, device, kind=None):
        """The container on the device: palette rows gathered by h in int64, then the planted rows."""
        el = self.distinct if kind is None else self.elements(kind)
        pal = torch.from_numpy(np.ascontiguousarray(el[:PALETTE])).to(device)
        i = torch.arange(self.n, dtype=torch.int64, device=device)
        rows = pal[hash_label(i)]
        del i
        rows[torch.from_numpy(self.planted).to(device)] = torch.from_numpy(el[self.planted_label]).to(device)
        return rows


# ---- the index: a sparse graph and its image ----------------------------------------------------------------------------
class SparseAdj:
    """A layer's neighbour lists where only some nodes have any."""

    def __init__(self, n, lists):
        self.n, self.lists = n, lists

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return self.lists.get(int(i), ())


def sparse_graph(n, members, seed, degree=10, top=64):
    """Layers [top, bottom]: the top layer is [0, top), each node linked to 4 random others and its successor; in the
    bottom layer only C = [0, top) + members has neighbours, each node of C `degree` random members of C and its
    successor in a cycle of C, so all of C is reachable from node 0."""
    rng = np.random.default_rng(seed)
    c = np.unique(np.concatenate([np.arange(top), np.asarray(members, dtype=np.int64)]))
    top_lists = {i: sorted((set(rng.integers(0, top, size=4).tolist()) | {(i + 1) % top}) - {i}) for i in range(top)}
    bottom = {}
    for j, i in enumerate(c.tolist()):
        nb = set(c[rng.integers(0, c.size, size=degree)].tolist()) | {int(c[(j + 1) % c.size])}
        bottom[i] = sorted(nb - {i})
    return [SparseAdj(top, top_lists), SparseAdj(n, bottom)]


def sparse_index(oracle, layers):
    """index_from_lists(oracle, [[adj[i] for i in range(len(adj))] for adj in layers]) for SparseAdj layers, byte for
    byte, without a list per row: an empty list is set_encode([]) (one zero byte), and the chunk table (per 60 rows a
    u64 initial offset and 60 u16 deltas, 0xFFFF past the last offset) is written with array arithmetic."""
    empty = oracle.set_encode([])
    assert empty == b"\x00", empty
    blobs = []
    for adj in layers:
        n = len(adj)
        enc = {i: oracle.set_encode(sorted(l)) for i, l in adj.lists.items()}
        lens = np.ones(n, dtype=np.int64)
        if enc:
            keys = np.fromiter(enc.keys(), dtype=np.int64, count=len(enc))
            lens[keys] = [len(enc[int(i)]) for i in keys]
        offsets = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=offsets[1:])
        nchunks = 1 + n // 60
        padded = np.full(nchunks * 60, -1, dtype=np.int64)
        padded[:n + 1] = offsets
        table = padded.reshape(nchunks, 60)
        prev = np.concatenate([table[:, :1], table[:, :-1]], axis=1)
        deltas = np.where(table >= 0, table - prev, 0xFFFF)
        assert (deltas <= 0xFFFF).all()
        chunks = np.empty(nchunks, dtype=[("initial", "<u8"), ("deltas", "<u2", (60,))])
        chunks["initial"] = table[:, 0]
        chunks["deltas"] = deltas
        data = np.zeros(int(offsets[-1]), dtype=np.uint8)
        for i, e in enc.items():
            data[offsets[i]:offsets[i] + len(e)] = np.frombuffer(e, dtype=np.uint8)
        chunk_bytes = chunks.tobytes()
        blobs.append(len(chunk_bytes).to_bytes(8, "little") + chunk_bytes + data.tobytes())
    meta = "granne" + json.dumps({"compressed": True, "granne_version": "0.5.2",
                                  "layer_counts": [len(l) for l in layers], "layer_sizes": [len(b) for b in blobs],
                                  "num_elements": len(layers[-1]) if layers else 0, "num_layers": len(layers),
                                  "num_neighbors": len(layers[-1][0]) if layers else 0, "version": 2},
                                 separators=(",", ":"))
    return meta.encode().ljust(1024, b" ") + b"".join(blobs)
