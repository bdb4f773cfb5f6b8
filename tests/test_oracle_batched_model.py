"""The oracle's model of the GPU builder's batch schedule (GranneBuilder.build_batched), which
test_builder_batched_gpu.py compares the GPU build with.  With batches of one it must be the reference's sequential
build; its image must not depend on how many threads run the searches of a batch; and larger batches must really
change the graph."""
import pytest

from helpers.data import random_sum_embeddings, random_vectors

CFG = dict(num_neighbors=20, max_search=40)


def _elements(oracle, kind, n, seed):
    if kind == "embeddings":
        return random_sum_embeddings(oracle, 24, 200, n, seed)
    raw = random_vectors(n, 24, seed)
    return oracle.Elements.angular(raw) if kind == "angular" else oracle.Elements.angular_int(raw)


@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_batches_of_one_are_the_sequential_build(oracle, kind):
    el = _elements(oracle, kind, 2000, seed=1)
    seq = oracle.GranneBuilder(el, **CFG).build(threads=1)
    rb = oracle.GranneBuilder(el, **CFG)
    one = rb.build_batched(1, threads=4)
    assert seq.num_layers() > 2
    assert one.to_bytes() == seq.to_bytes()
    ctr = rb.counters()
    assert ctr["max_batch"] == 1 and ctr["batches"] > 2000 and ctr["connect_overflow"] > 0, ctr


def test_batches_of_one_are_the_sequential_incremental_build(oracle):
    n0, n = 1500, 2000
    raw = random_vectors(n, 24, seed=8)
    cfg = dict(CFG, expected_num_elements=n0)
    seq_el, one_el = oracle.Elements.angular(raw[:n0]), oracle.Elements.angular(raw[:n0])
    seq, one = oracle.GranneBuilder(seq_el, **cfg), oracle.GranneBuilder(one_el, **cfg)
    for step in (1, 40, 700, n0):
        assert one.build_partial(step, threads=4, max_batch=1).to_bytes() == seq.build_partial(step).to_bytes()
    seq_el.push(raw[n0:])
    one_el.push(raw[n0:])
    assert one.build_partial(n, threads=4, max_batch=1).to_bytes() == seq.build_partial(n).to_bytes()


@pytest.mark.parametrize("kind", ["angular", "angular_int", "embeddings"])
def test_model_does_not_depend_on_threads_and_batches_are_real(oracle, kind):
    el = _elements(oracle, kind, 3000, seed=2)
    images = []
    for threads in (1, 3, 8):
        rb = oracle.GranneBuilder(el, **CFG)
        images.append(rb.build_batched(64, threads=threads).to_bytes())
        assert rb.counters()["max_batch"] == 64
    assert images[0] == images[1] == images[2]
    assert images[0] != oracle.GranneBuilder(el, **CFG).build(threads=1).to_bytes()
