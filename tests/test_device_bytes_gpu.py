"""granne_b200_device_bytes, exactly, from shapes: a handle counts its layer rows, its element container and an attached
re-rank container, every allocation at least 16 bytes.  A handle opened from an index image (or over device-resident
rows) stores each layer at the image's row width; a handle from GranneBuilder.get_index stores it at the builder's
stride (num_neighbors rounded up to 8) and shares it with the builder, so a snapshot keeps its count while the builder
grows."""
import glob
import os

import numpy as np
import pytest

import granne_b200
from granne_b200 import words
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))
M = 12  # the builders' num_neighbors: stride 16, wider than the rows the builder keeps


def _alloc(nbytes):
    return max(nbytes, 16)


def _dense_bytes(kind, n, dim):
    """Staged dense rows: f32 rows padded to 4 floats, i8 rows to 32 bytes."""
    return _alloc(n * ((dim + 3) & ~3) * 4) if kind == "angular" else _alloc(n * ((dim + 31) & ~31))


def _sum_bytes(table_rows, dim, terms):
    """A staged SumEmbeddings container: the table (rows padded to 4 floats), n + 1 u64 offsets, the u32 term ids."""
    return (_alloc(table_rows * ((dim + 3) & ~3) * 4) + _alloc((len(terms) + 1) * 8) +
            _alloc(sum(len(t) for t in terms) * 4))


def _dense_shape(image, esz):
    dim = int(np.frombuffer(bytes(image[:8]), "<u8")[0])
    return (len(image) - 8) // (dim * esz), dim


def _container_bytes(kind, eb, mb):
    if kind == "embeddings":
        rows, dim = _dense_shape(mb, 4)
        return _sum_bytes(rows, dim, words.read_sum_terms(bytes(eb)))
    return _dense_bytes(kind, *_dense_shape(eb, 4 if kind == "angular" else 1))


def _image_layers_bytes(ib):
    return sum(_alloc(n * width * 4) for n, _, width in granne_b200.inspect_index(ib))


def _builder_layers_bytes(g):
    stride = (M + 7) & ~7
    return sum(_alloc(g.layer_len(l) * stride * 4) for l in range(g.num_layers()))


def _golden(path):
    z = np.load(path)
    mb = z["embeddings"].tobytes() if z["embeddings"].size else None
    return str(z["kind"]), z["index"].tobytes(), z["elements"].tobytes(), mb


def _data(kind, n, dim, seed):
    """n random elements: raw f32 rows, or for "embeddings" term lists over a 100-row table; and the table's image."""
    rng = np.random.default_rng(seed)
    if kind == "embeddings":
        table = rng.standard_normal((100, dim)).astype(np.float32)
        terms = [[int(t) for t in rng.integers(0, 100, i % 7)] for i in range(n)]
        return terms, np.uint64(dim).tobytes() + table.tobytes()
    return rng.standard_normal((n, dim)).astype(np.float32), None


def _elements_image(kind, data):
    if kind == "embeddings":
        return bytes(words.write_sum_terms(data))
    return granne_b200.elements_from_raw(kind, data).tobytes()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_opened_handles(path):
    kind, ib, eb, mb = _golden(path)
    want = _image_layers_bytes(ib) + _container_bytes(kind, eb, mb)
    g = granne_b200.Granne.from_bytes(ib, kind, eb, mb)
    assert g.device_bytes() == want
    g.close()
    if kind == "embeddings":
        return
    import torch

    n, dim = _dense_shape(eb, 4 if kind == "angular" else 1)
    rows = torch.from_numpy(np.frombuffer(eb[8:], np.float32 if kind == "angular" else np.int8).reshape(n, dim).copy())
    g = granne_b200.Granne.from_device_elements(ib, kind, rows.cuda(0))
    assert g.device_bytes() == want
    g.close()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_resumed_builder(path, tmp_path):
    kind, ib, eb, mb = _golden(path)
    files = {}
    for name, data in (("index", ib), ("elements", eb), ("embeddings", mb)):
        if data is not None:
            files[name] = str(tmp_path / name)
            with open(files[name], "wb") as f:
                f.write(data)
    b = granne_b200.GranneBuilder.from_files(kind, files["elements"], index_path=files["index"],
                                             embeddings_path=files.get("embeddings"), num_neighbors=M, max_search=40)
    g = b.get_index()
    assert [g.layer_len(l) for l in range(g.num_layers())] == [n for n, _, _ in granne_b200.inspect_index(ib)]
    assert g.device_bytes() == _container_bytes(kind, eb, mb) + _builder_layers_bytes(g)
    g.close()
    b.close()


@pytest.mark.parametrize("kind,dim", [("angular", 32), ("angular_int", 100), ("embeddings", 20)])
def test_builder_snapshots(kind, dim):
    n0, add = 700, 300
    data, mb = _data(kind, n0 + add, dim, dim)

    def container(n):
        return _sum_bytes(100, dim, data[:n]) if kind == "embeddings" else _dense_bytes(kind, n, dim)

    b = granne_b200.GranneBuilder(kind, _elements_image(kind, data[:n0]), mb, num_neighbors=M, max_search=40)
    b.build()
    before = b.get_index()
    want_before = container(n0) + _builder_layers_bytes(before)
    assert before.device_bytes() == want_before

    for e in data[n0:]:
        b.append(e)
    b.build()
    after = b.get_index()
    assert len(after) == n0 + add
    assert after.device_bytes() == container(n0 + add) + _builder_layers_bytes(after)
    assert after.device_bytes() > want_before
    # the snapshot taken first still holds the container and layers it was given
    assert len(before) == n0
    assert before.device_bytes() == want_before
    for h in (before, after, b):
        h.close()


def test_rerank_on_builder_snapshot():
    n, dim = 600, 48
    raw, _ = _data("angular_int", n, dim, 7)
    b = granne_b200.GranneBuilder("angular_int", _elements_image("angular_int", raw), num_neighbors=M, max_search=40)
    b.build()
    g = b.get_index()
    before = g.device_bytes()
    assert before == _dense_bytes("angular_int", n, dim) + _builder_layers_bytes(g)

    # an attach rejected by its checks stages nothing
    with pytest.raises(granne_b200.GranneError):
        g.set_rerank_elements(granne_b200.elements_from_raw("angular", raw[:, :32]).tobytes())
    assert g.device_bytes() == before

    g.set_rerank_elements(granne_b200.elements_from_raw("angular", raw).tobytes())
    assert g.device_bytes() == before + _dense_bytes("angular", n, dim)
    # a second attach fails and changes nothing
    with pytest.raises(granne_b200.GranneError):
        g.set_rerank_elements(granne_b200.elements_from_raw("angular", raw).tobytes())
    assert g.device_bytes() == before + _dense_bytes("angular", n, dim)
    g.close()
    b.close()
