"""compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152) on the GPU
(granne_b200_compute_embeddings / _device): images byte-identical to the oracle's restatement for both output kinds, at
every width class, term count, table size and row value that matters; and the materialised angular rows searched and
built over exactly like the SumEmbeddings container they come from."""
import os
import subprocess

import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co
from helpers.data import random_vectors
from helpers.fixtures import assert_same, compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_FINITE = -6
WINDOW_BYTES = 64 << 20  # kEmbWindowBytes in granne_b200.cu: raw f32 rows per window


def _rows(kind, image, n=None):
    dim = int(np.frombuffer(image[:8], dtype=np.uint64)[0])
    dt = np.float32 if kind == "angular" else np.int8
    a = np.frombuffer(np.asarray(image)[8:].tobytes(), dtype=dt)
    return a.reshape(-1 if dim else (n or 0), dim)


def _check(kind, ei, ti, stream=False):
    """GPU image == oracle image, and the device variant's rows == the image's rows."""
    import torch

    want = co.compute_embeddings(kind, ei, ti, threads=8)
    got = granne_b200.compute_embeddings(kind, ei, ti)
    assert got.size == want.size and np.array_equal(got, want), kind
    s = torch.cuda.Stream() if stream else None  # a non-default stream
    prev = torch.cuda.current_device()
    dev = granne_b200.compute_embeddings_device(kind, ei, ti, stream=s.cuda_stream if s is not None else None)
    assert torch.cuda.current_device() == prev
    n = int(np.frombuffer(ei[:8], dtype=np.uint64)[0])
    assert tuple(dev.shape) == _rows(kind, want, n).shape
    assert np.array_equal(dev.cpu().numpy().view(np.uint8), _rows(kind, want, n).view(np.uint8))
    return want


def _random_case(dim, counts, num_rows, seed):
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((num_rows, dim)) * 2).astype(np.float32)
    elements = []
    for i, c in enumerate(counts):
        ids = rng.integers(0, num_rows, c)
        if c > 3:
            ids[c // 2] = ids[0]  # repeated ids
        elements.append([int(t) for t in ids])
    return table, elements


@pytest.mark.parametrize("dim", [1, 31, 32, 33, 100, 128, 300, 1000, 4096])
def test_images_equal_the_oracle(dim):
    counts = [0, 1, 2, 9, 32, 33, 300] * 4
    table, elements = _random_case(dim, counts, 500, seed=dim)
    ei, ti = co.elements_image(elements), co.table_image(table)
    for kind in ("angular_int", "angular"):
        _check(kind, ei, ti, stream=dim % 2 == 1)


def test_golden_embeddings_fixture():
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    for kind in ("angular_int", "angular"):
        img = _check(kind, z["elements"].tobytes(), z["embeddings"].tobytes(), stream=True)
        assert _rows(kind, img).shape == (600, 20)


def test_the_largest_term_id():
    rows = 1 << 24
    table = np.arange(rows, dtype=np.float32).reshape(rows, 1) - np.float32(rows / 2)
    elements = [[0xFFFFFF], [0xFFFFFF, 0, 5], [], [1 << 23, 0xFFFFFF]]
    ei, ti = co.elements_image(elements), co.table_image(table)
    for kind in ("angular_int", "angular"):
        _check(kind, ei, ti)


def test_row_values():
    tiny = np.float32(1e-40)
    table = np.array([[-0.0, -0.0, -0.0], [1.5, -2.0, 3.0], [-1.5, 2.0, -3.0], [tiny, -tiny, 2 * tiny],
                      [3e38, -3e38, 1.0], [1e-39, 0.0, -1e-39]], dtype=np.float32)
    # -0.0, cancelling (x + -x), subnormal sums, a finite row whose squared norm overflows (normalises to +-0)
    finite = [[0], [1, 2], [2, 1, 1], [3], [3, 3, 5], [5, 5], [], [0, 0], [1], [4]]
    ei, ti = co.elements_image(finite), co.table_image(table)
    for kind in ("angular_int", "angular"):
        _check(kind, ei, ti)
    ang = _rows("angular", granne_b200.compute_embeddings("angular", ei, ti))
    assert np.signbit(ang[0]).all()  # a single -0.0 row stays -0.0
    overflow = co.elements_image([[1], [4, 4], [4, 4, 4, 1]])  # +-inf sums: 3e38 + 3e38
    _check("angular_int", overflow, ti)
    for fn in (granne_b200.compute_embeddings, granne_b200.compute_embeddings_device):
        with pytest.raises(granne_b200.GranneError) as e:
            fn("angular", overflow, ti)
        assert e.value.code == NOT_FINITE


def test_nan_rows():
    table = np.array([[1.0, 2.0], [np.nan, 0.0], [0.5, 0.5]], dtype=np.float32)
    ti = co.table_image(table)
    unused = co.elements_image([[0, 2], [2]])
    for kind in ("angular_int", "angular"):
        _check(kind, unused, ti)
        for fn in (granne_b200.compute_embeddings, granne_b200.compute_embeddings_device):
            with pytest.raises(granne_b200.GranneError) as e:
                fn(kind, co.elements_image([[0], [0, 1], [2]]), ti)
            assert e.value.code == NOT_FINITE
        with pytest.raises(co.NotFinite):
            co.compute_embeddings(kind, co.elements_image([[0], [0, 1], [2]]), ti)


def test_sizes():
    ti = co.table_image(random_vectors(10, 7, seed=1))
    for kind in ("angular_int", "angular"):
        assert _check(kind, co.elements_image([]), ti).tobytes() == bytes(8)
        # a table without rows (width 1: the loader rejects a width wider than the payload)
        assert _check(kind, co.elements_image([[], [], []]), np.uint64(1).tobytes()).tobytes() == bytes(8)
    # more than two windows and a remainder: 64 MB of raw rows per window is 4096 rows of width 4096
    dim = 4096
    window = WINDOW_BYTES // (4 * dim)
    n = 2 * window + 17
    table, _ = _random_case(dim, [], 64, seed=5)
    rng = np.random.default_rng(6)
    elements = [[int(t) for t in rng.integers(0, 64, 1 + i % 3)] for i in range(n)]
    ei, ti = co.elements_image(elements), co.table_image(table)
    for kind in ("angular_int", "angular"):
        img = _check(kind, ei, ti, stream=True)
        assert img.size == 8 + n * dim * (4 if kind == "angular" else 1)


def test_save_to_disk(tmp_path):
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    (tmp_path / "elements").write_bytes(z["elements"].tobytes())
    (tmp_path / "embeddings").write_bytes(z["embeddings"].tobytes())
    for kind in ("angular_int", "angular"):
        out = tmp_path / ("out_" + kind)
        granne_b200.compute_embeddings_and_save_to_disk(str(tmp_path / "elements"), str(tmp_path / "embeddings"),
                                                        str(out), False, element_type=kind)
        want = co.compute_embeddings(kind, z["elements"].tobytes(), z["embeddings"].tobytes())
        assert out.read_bytes() == want.tobytes()


def test_search_over_materialised_rows_equals_sum_embeddings():
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    index, el, emb = z["index"].tobytes(), z["elements"].tobytes(), z["embeddings"].tobytes()
    rows = granne_b200.compute_embeddings_device("angular", el, emb)
    summed = granne_b200.Granne.from_bytes(index, "embeddings", el, emb)
    dense = granne_b200.Granne.from_device_elements(index, "angular", rows)
    raw_q = np.concatenate([z["queries"], random_vectors(200, 20, seed=3)])
    elem_q = rows[::7].cpu().numpy()
    for ms in (10, 200, 1000):
        assert_same(summed.search_batch(raw_q, ms, 10, with_stats=True),
                    dense.search_batch(raw_q, ms, 10, with_stats=True), "raw queries, max_search %d" % ms, stats=True)
        assert_same(summed.search_batch(elem_q, ms, 10, already_element=True, with_stats=True),
                    dense.search_batch(elem_q, ms, 10, already_element=True, with_stats=True),
                    "element queries, max_search %d" % ms, stats=True)
    for i in (0, 17, 599):
        assert np.array_equal(summed.get_element(i).view(np.uint32), dense.get_element(i).view(np.uint32))


def test_build_over_materialised_rows_equals_sum_embeddings(monkeypatch):
    monkeypatch.setenv("GRANNE_B200_BUILD_MAX_BATCH", "1")  # every insertion sees all earlier links
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    el, emb = z["elements"].tobytes(), z["embeddings"].tobytes()
    rows = granne_b200.compute_embeddings_device("angular", el, emb)
    a = granne_b200.GranneBuilder("embeddings", el, emb, num_neighbors=16, max_search=50)
    b = granne_b200.GranneBuilder.from_device_elements("angular", rows, num_neighbors=16, max_search=50)
    a.build()
    b.build()
    assert bytes(a.index_bytes()) == bytes(b.index_bytes())


def test_index_over_angular_int_rows_matches_the_oracle(oracle):
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    img = granne_b200.compute_embeddings("angular_int", z["elements"].tobytes(), z["embeddings"].tobytes()).tobytes()
    el = oracle.Elements.from_bytes("angular_int", img)
    g = oracle.GranneBuilder(el, num_neighbors=16, max_search=50).build()
    index = g.to_bytes()
    ref = oracle.Granne.from_bytes(index, el)
    gpu = granne_b200.Granne.from_bytes(index, "angular_int", img)
    q = random_vectors(300, 20, seed=9)
    assert_same(ref.search_batch(q, 50, 10, with_stats=True), gpu.search_batch(q, 50, 10, with_stats=True), "angular_int",
                stats=True)


def test_cxx_client(tmp_path):
    exe = compile_cxx_client("cxx_embeddings_client.cpp", tmp_path)
    z = np.load(os.path.join(ROOT, "tests", "golden", "embeddings_600x20_m16.npz"))
    (tmp_path / "elements").write_bytes(z["elements"].tobytes())
    (tmp_path / "embeddings").write_bytes(z["embeddings"].tobytes())
    r = subprocess.run([exe, "gpu", str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "gpu ok" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    for kind in ("angular", "angular_int"):
        want = co.compute_embeddings(kind, z["elements"].tobytes(), z["embeddings"].tobytes())
        assert (tmp_path / kind).read_bytes() == want.tobytes()
