"""GPU tests of the device-resident element containers (granne_b200_elements_from_raw_device,
granne_b200_builder_new_device_elements, granne_b200_open_device_elements) and of the pass ladder (fast pass -> retry
pass -> slow pass) behind Granne::search.

The reference borrows its element container from the caller (`Vectors::from_slice`, src/elements/dense_vector.rs:66-72;
`Granne::from_bytes(index, &elements)`, src/index/mod.rs:108-113); here the container may already live in HBM.  Bar:
the device path must be indistinguishable from the file-image path, and both bit-identical to the oracle.
"""
import numpy as np
import pytest

import granne_b200
from helpers.data import random_vectors
from helpers.fixtures import assert_same
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind,n,dim", [("angular", 6000, 64), ("angular_int", 4000, 100), ("angular", 3000, 28)])
def test_device_resident_elements_equal_the_file_image_path(oracle, kind, n, dim):
    import torch

    raw = random_vectors(n, dim, seed=31)
    image = granne_b200.elements_from_raw(kind, raw)                     # host path: elements file image
    dev_rows = granne_b200.elements_from_raw_device(kind, torch.from_numpy(raw).cuda())
    dt = np.int8 if kind == "angular_int" else np.float32
    host_rows = np.frombuffer(image, dtype=dt, offset=8).reshape(n, dim)
    assert np.array_equal(dev_rows.cpu().numpy().view(np.uint8), host_rows.view(np.uint8))  # Vector::from, bit for bit

    b = granne_b200.GranneBuilder.from_device_elements(kind, dev_rows, num_neighbors=20, max_search=50)
    b.build()
    index_bytes = b.index_bytes()
    built = b.get_index()
    from_dev = granne_b200.Granne.from_device_elements(index_bytes, kind, dev_rows)
    from_img = granne_b200.Granne.from_bytes(index_bytes, kind, image)
    assert len(from_dev) == len(from_img) == n and from_dev.dim == dim
    q = random_vectors(400, dim, seed=32)
    got_dev = from_dev.search_batch(q, 50, 10, with_stats=True)
    got_img = from_img.search_batch(q, 50, 10, with_stats=True)
    got_built = built.search_batch(q, 50, 10, with_stats=True)
    assert_same(got_dev, got_img, "device vs image", stats=True)
    assert_same(got_dev, got_built, "device vs builder snapshot", stats=True)
    # and against the oracle on the very same files
    g = oracle.Granne.from_bytes(index_bytes, oracle.Elements.from_bytes(kind, image))
    ref = g.search_batch(q, 50, 10, with_stats=True)
    assert_same(ref, got_dev, "oracle vs device", stats=True)
    assert np.array_equal(from_dev.get_element(17), from_img.get_element(17))
    for h in (from_dev, from_img, built):
        h.close()
    b.close()


def test_device_rows_are_validated():
    import torch

    raw = torch.zeros((8, 32), dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError):
        granne_b200.elements_from_raw_device("angular", raw.double())
    with pytest.raises(ValueError):
        granne_b200.elements_from_raw_device("angular", raw.t())
    el = granne_b200.elements_from_raw_device("angular", raw + 1.0)
    with pytest.raises(ValueError):
        granne_b200.GranneBuilder.from_device_elements("angular_int", el)  # float rows for an i8 container
    # a host pointer is not device memory: status code, no crash
    import ctypes as C

    L = granne_b200.load_library()
    host = np.zeros((8, 32), dtype=np.float32)
    h = C.c_void_p()
    cfg = granne_b200.BuildConfig()
    L.granne_b200_build_config_default(C.byref(cfg))
    rc = L.granne_b200_builder_new_device_elements(C.byref(cfg), 0, host.ctypes.data_as(C.c_void_p), 8, 32, 0,
                                                   C.byref(h))
    assert rc != 0 and b"device memory" in L.granne_b200_last_error()


def test_search_batch_device_validates_its_tensors(oracle):
    """ADVICE r1: a wrong dtype / width / device / layout must be an error, not an out-of-bounds read."""
    import torch

    raw = random_vectors(2000, 32, seed=5)
    image = granne_b200.elements_from_raw("angular", raw)
    b = granne_b200.GranneBuilder("angular", image, num_neighbors=10, max_search=30)
    b.build()
    idx = b.get_index()
    q = torch.from_numpy(random_vectors(64, 32, seed=6)).cuda()
    ids, d, c = idx.search_batch_device(q, 30, 5)
    ids2, d2, c2 = idx.search_batch_device(q.t().contiguous().t(), 30, 5)   # strided view: made contiguous, same result
    torch.cuda.synchronize()
    assert torch.equal(ids, ids2) and torch.equal(d, d2)
    for bad in (q.double(), q[:, :16], q.cpu(), q.reshape(-1)):
        with pytest.raises(ValueError):
            idx.search_batch_device(bad, 30, 5)
    with pytest.raises(ValueError):
        idx.search_batch_device(q, 30, 5, out=(ids.long(), d, c))
    # a retired stream hands its workspace back; the handle keeps working on other streams
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ids3, d3, _ = idx.search_batch_device(q, 30, 5, stream=side.cuda_stream)
    idx.release_stream(side)
    assert torch.equal(ids, ids3) and torch.equal(d, d3)
    idx.release_stream(side)          # releasing twice is harmless
    idx.stream_status()
    idx.close()
    b.close()


def test_retry_pass_serves_heavy_queries_exactly(oracle):
    """Uniform random vectors (the reference's own test distribution, src/test_helper.rs:3-6) have little
    neighbourhood overlap: a search visits almost max_search x degree nodes and overflows the fast pass's visited
    table.  Those queries are answered by the retry pass (stat 3 == 1) — bit-identical to the oracle — and after a few
    thousand queries the handle has grown its tables so that the fast pass serves (nearly) all of them."""
    raw = random_vectors(20_000, 48, seed=41)
    el = oracle.Elements.angular(raw)
    g = oracle.GranneBuilder(el, num_neighbors=30, max_search=60).build(threads=8)
    ib, eb = g.to_bytes(), el.to_bytes()
    ref_index = oracle.Granne.from_bytes(ib, el)
    p = granne_b200.Granne.from_bytes(ib, "angular", eb)
    q = random_vectors(3000, 48, seed=42)
    ref = ref_index.search_batch(q, 60, 10, with_stats=True)
    got = p.search_batch(q, 60, 10, with_stats=True)
    assert_same(ref, got, "first batch", stats=True)
    first = int((got[3][:, 3] != 0).sum())
    for _ in range(4):  # the scale adapts between calls (the counter is read back without synchronising)
        got = p.search_batch(q, 60, 10, with_stats=True)
        assert_same(ref, got, "later batch", stats=True)
    later = int((got[3][:, 3] != 0).sum())
    assert (got[3][:, 3] <= 1).all(), "nobody should need the 4-CTA slow pass here"
    if first > 30:
        assert later * 4 < first, "visited tables did not adapt: %d -> %d retried queries" % (first, later)
    p.close()
