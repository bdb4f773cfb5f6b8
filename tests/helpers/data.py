"""Seeded synthetic data in the reference's own test distribution (src/test_helper.rs:3-46) + fixture builders.

Everything here drives the ORACLE (test infrastructure) to produce granne-format files that the product then loads.
"""
import numpy as np


def random_vectors(n, dim, seed):
    """test_helper::random_vectors: each component U(0,1) - 0.5 (src/test_helper.rs:3-18)."""
    rng = np.random.default_rng(seed)
    return (rng.random((n, dim), dtype=np.float32) - np.float32(0.5)).astype(np.float32)


def random_sum_embeddings(go, dim, num_embeddings, num_elements, seed):
    """test_helper::random_sum_embeddings (src/test_helper.rs:29-46): element i = ids i..i+len, len = 2 + i % 8."""
    emb = random_vectors(num_embeddings, dim, seed)
    elements = [[j % num_embeddings for j in range(i, i + 2 + i % 8)] for i in range(num_elements)]
    return go.Elements.sum_embeddings(emb, elements)


def varied_sum_embeddings(go, dim, num_embeddings, num_elements, seed, special=((7, 0), (13, 1), (19, 33), (24, 70))):
    """Sum-of-embeddings elements whose term lists are drawn at random with repetition (a term can occur more than
    once), 2 to 9 terms each, except that element i has exactly m terms when (i % 25, m) is in `special`: by default
    elements without terms (zero vectors), of one term, and of more than 32 and 64 terms (more than one and two warp
    widths of term ids)."""
    rng = np.random.default_rng(seed)
    emb = random_vectors(num_embeddings, dim, seed)
    lengths = dict(special)
    lists = [rng.integers(0, num_embeddings, size=lengths.get(i % 25, int(rng.integers(2, 10)))).tolist()
             for i in range(num_elements)]
    return go.Elements.sum_embeddings(emb, lists)


def clustered_vectors(n, dim, seed, n_centers=None, sub_dim=16, spread=0.3):
    """Measurement distribution (SURVEY.md §8d): Gaussian mixture on a random low-dimensional subspace."""
    rng = np.random.default_rng(seed)
    n_centers = n_centers or max(8, int(4096 * (n / 1e6) ** 0.5))
    basis = rng.standard_normal((sub_dim, dim)).astype(np.float32)
    centers = rng.standard_normal((n_centers, sub_dim)).astype(np.float32)
    which = rng.integers(0, n_centers, size=n)
    pts = centers[which] + spread * rng.standard_normal((n, sub_dim)).astype(np.float32)
    return (pts @ basis).astype(np.float32)


def build_fixture(go, kind, n, dim, seed, num_neighbors, max_search, threads=1, **kw):
    """Returns (elements, oracle Granne, index_bytes, elements_bytes, embeddings_bytes|None)."""
    if kind == "angular":
        el = go.Elements.angular(random_vectors(n, dim, seed))
    elif kind == "angular_int":
        el = go.Elements.angular_int(random_vectors(n, dim, seed))
    elif kind == "embeddings":
        el = random_sum_embeddings(go, dim, kw.get("num_embeddings", 200), n, seed)
    else:
        raise ValueError(kind)
    g = go.GranneBuilder(el, num_neighbors=num_neighbors, max_search=max_search,
                         layer_multiplier=kw.get("layer_multiplier", 15.0),
                         reinsert_elements=kw.get("reinsert", True)).build(threads=threads)
    index_bytes = g.to_bytes()
    elements_bytes = el.to_bytes(0)
    emb_bytes = el.to_bytes(1) if kind == "embeddings" else None
    # search through the from_bytes path (compressed layers), like a user of the reference would
    g2 = go.Granne.from_bytes(index_bytes, el)
    return el, g2, index_bytes, elements_bytes, emb_bytes


def index_from_lists(oracle, layers):
    """Writes an index file from explicit adjacency lists (oracle writer, src/index/io.rs:11-70)."""
    import json

    blobs = []
    for lists in layers:
        enc = [oracle.set_encode(sorted(l)) for l in lists]
        offsets = [0]
        for e in enc:
            offsets.append(offsets[-1] + len(e))
        nchunks = 1 + len(lists) // 60
        chunks = bytearray()
        for c in range(nchunks):
            offs = offsets[c * 60:(c + 1) * 60]
            initial = offs[0] if offs else 0
            chunks += int(initial).to_bytes(8, "little")
            prev = initial
            for i in range(60):
                if i < len(offs):
                    chunks += int(offs[i] - prev).to_bytes(2, "little")
                    prev = offs[i]
                else:
                    chunks += b"\xff\xff"
        blobs.append(len(chunks).to_bytes(8, "little") + bytes(chunks) + b"".join(enc))
    meta = "granne" + json.dumps({"compressed": True, "granne_version": "0.5.2",
                                  "layer_counts": [len(l) for l in layers], "layer_sizes": [len(b) for b in blobs],
                                  "num_elements": len(layers[-1]) if layers else 0, "num_layers": len(layers),
                                  "num_neighbors": len(layers[-1][0]) if layers else 0, "version": 2},
                                 separators=(",", ":"))
    return meta.encode().ljust(1024, b" ") + b"".join(blobs)


def edge_raw_f32(n, dim, seed):
    """Raw f32 rows (n >= 12) at the edges of the reference's arithmetic, the rest random: an all-zero row, duplicates,
    -0.0 and subnormal components, rows whose squared norm underflows to 0 (normalize_f32 leaves them as they are) or
    overflows to +inf (they normalise to +-0), rows of subnormals only, and a row of equal components."""
    x = random_vectors(n, dim, seed)
    rng = np.random.default_rng(seed + 1)
    x[0] = 0.0
    x[2] = x[1]
    x[3] = -0.0
    x[3, ::3] = x[1, ::3]
    x[4, rng.random(dim) < 0.3] = np.float32(-0.0)
    sub = rng.random(dim) < 0.3
    x[4, sub] = np.float32(1e-40) * np.where(rng.random(int(sub.sum())) < 0.5, -1, 1).astype(np.float32)
    x[5] = np.float32(1e-25) * np.sign(x[5])             # squares are below the smallest subnormal: norm 0
    x[6] = np.float32(1e20) * np.sign(x[6])              # squares overflow: norm +inf
    x[7] = np.float32(3e-39) * np.sign(x[7])             # subnormal components
    x[8] = np.float32(0.25)
    x[9] = x[0]
    x[10, : dim // 2] = np.float32(1e-38)
    x[11] = np.float32(1.7e19) * np.sign(x[11])           # the squared norm just overflows for dim > 1
    return x


def edge_i8_rows(n, dim, seed):
    """int8 element rows (n >= 8): random quantised rows plus saturated rows of +-127 and of -128 (which quantize never
    makes, but an elements image may hold), whose r, dx and dy pass 2^24 once dim > 1040, and all-zero rows."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-127, 128, size=(n, dim)).astype(np.int8)
    x[0] = 0
    x[1] = 127
    x[2] = np.where(rng.random(dim) < 0.5, 127, -127)
    x[3] = -128
    x[4] = np.where(rng.random(dim) < 0.5, -128, 127)
    x[5] = x[2]
    x[6] = -x[2]
    x[7] = 0
    return x
