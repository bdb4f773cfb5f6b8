"""What test_wide_offsets_gpu rests on, without a GPU:

- each of its cases crosses the byte boundaries it names, with row strides read from the sources (stage_dense pads f32
  rows to a multiple of 4 floats and i8 rows to a multiple of 32 bytes), and names every power-of-two boundary from
  2^31 up that its rows cross, so shrinking n or a width fails here;
- each case reaches the engine and layout it names (the engine choice of test_builder_engines_cpu, read from
  DistDispatch and DistI8::load_query), and the i8 cases reach both DistI8 layouts;
- the sparse index writer is byte-identical to index_from_lists, the fast ranking equals the model's, and the
  fixture's premises hold on a scaled-down container."""
import os
import re

import numpy as np
import pytest

from helpers import ref_model as M
from helpers.data import index_from_lists
from helpers.wide_fixture import (PALETTE, SparseAdj, Wide, boundary_ids, first_id_at, rank, row_bytes, sparse_graph,
                                  sparse_index)
from test_builder_engines_cpu import engine_choice
from test_wide_offsets_gpu import CASES, N, RERANK

CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "granne_b200", "csrc",
                  "granne_b200.cu")


def _strides():
    """(f32 floats, i8 bytes) that stage_dense rounds a row up to."""
    with open(CU) as f:
        text = f.read()
    block = text[text.index("int stage_dense("):]
    block = block[:block.index("\n}")]
    i8 = re.findall(r"d\.row_stride = \(dim \+ (\d+)u\) & ~(\d+)u;\s*// rows start on 32-byte", block)
    f32 = re.findall(r"d\.row_stride = \(dim \+ (\d+)u\) & ~(\d+)u;\n", block)
    assert len(i8) == 1 and len(f32) == 1, (i8, f32)
    for add, mask in i8 + f32:
        assert add == mask, (add, mask)
    return int(f32[0][0]) + 1, int(i8[0][0]) + 1


def _stride(kind, dim):
    f32_floats, i8_bytes = _strides()
    return row_bytes(kind, dim, f32_floats, i8_bytes)


def _all_cases():
    return [(kind, dim, engine, b) for kind, dim, engine, b in CASES + RERANK]


# ---- the cases ---------------------------------------------------------------------------------------------------------
def test_each_case_crosses_the_boundaries_it_names():
    for kind, dim, _, boundaries in _all_cases():
        stride = _stride(kind, dim)
        assert stride == row_bytes(kind, dim), (kind, dim)   # the fixture plants ids by the same stride
        # every power of two from 2^31 that a row of the container starts at or past, and no other
        crossed = [1 << e for e in range(31, 64) if first_id_at(1 << e, stride) + 1 < N]
        assert list(boundaries) == crossed, (kind, dim, stride)
        assert max(boundary_ids(boundaries, stride)) < N
    f32 = {(k, d): b for k, d, _, b in _all_cases() if k == "angular"}
    # the f32 rows reach 2^32 floats (the offset of a float index past uint32)
    assert all(max(b) >= 4 << 32 for b in f32.values())
    # the widest i8 rows reach 2^34 bytes (2^32 four-byte words); the 128-byte rows 2^32 bytes
    assert max(max(b) for k, d, _, b in CASES if k == "angular_int") >= 1 << 34
    assert all(max(b) >= 1 << 32 for k, d, _, b in _all_cases())


def test_each_case_reaches_the_engine_it_names():
    engine, _ = engine_choice()
    for kind, dim, named, _ in _all_cases():
        assert engine(kind, dim) == named, (kind, dim)
    # DistF32<4> reads lane-permuted rows in groups of 4 chunks: dim / 32 a multiple of 4
    assert all((dim // 32) % 4 == 0 for kind, dim, _, _ in _all_cases() if kind == "angular")
    layouts = {engine(kind, dim)[1] for kind, dim, _, _ in CASES if kind == "angular_int"}
    assert layouts == {"sub-warp groups", "one row at a time"}, layouts


# ---- the sparse index writer ---------------------------------------------------------------------------------------------
def _dense(layers):
    return [[list(adj[i]) for i in range(len(adj))] for adj in layers]


@pytest.mark.parametrize("n", [1, 59, 60, 61, 120, 149, 301])
def test_sparse_index_matches_index_from_lists(oracle, n):
    rng = np.random.default_rng(n)
    # a component spread over several 60-node chunks, every other row empty
    comp = np.unique(rng.integers(0, n, size=max(1, n // 4)))
    lists = {int(i): sorted(set(rng.choice(comp, size=min(5, comp.size)).tolist()) - {int(i)}) for i in comp}
    lists.setdefault(0, [])
    bottom = SparseAdj(n, lists)
    top_n = min(n, 7)
    top = SparseAdj(top_n, {i: sorted({(i + 1) % top_n} - {i}) for i in range(top_n)})
    for layers in ([bottom], [top, bottom], [SparseAdj(n, {})]):
        assert sparse_index(oracle, layers) == index_from_lists(oracle, _dense(layers))


def test_sparse_graph_image_matches_index_from_lists(oracle):
    n = 1000
    layers = sparse_graph(n, [3, 500, 998, 999, 120, 121], 5, top=16)
    assert sparse_index(oracle, layers) == index_from_lists(oracle, _dense(layers))
    # every node of C is reachable from node 0 in the bottom layer
    seen, todo = {0}, [0]
    while todo:
        for j in layers[1][todo.pop()]:
            if j not in seen:
                seen.add(j)
                todo.append(j)
    assert seen == set(layers[1].lists)


# ---- the fast ranking ---------------------------------------------------------------------------------------------------
def test_fast_ranking_matches_the_model():
    rng = np.random.default_rng(3)
    for trial in range(40):
        m = int(rng.integers(1, 300))
        d = rng.choice(np.array([0.0, -0.0, 0.25, 0.5, 0.5, 1.0, 1e-40, 2.0], dtype=np.float32), size=m)
        if trial % 2:
            d = np.where(rng.random(m) < 0.5, d, rng.random(m).astype(np.float32))
        d = d.astype(np.float32)
        for k in (1, 2, 3, 10, m - 1, m, m + 5):   # k past the number of distinct rows too
            if k < 1:
                continue
            ids = rng.integers(0, m, size=2 * k)    # with duplicates
            for got, want in ((rank(d, k), M.rank_prefix(d, m, k)), (rank(d, k, ids), M.rank(d, ids, k))):
                assert [i for i, _ in got] == [i for i, _ in want], (trial, k)
                assert np.array_equal(np.array([x for _, x in got], np.float32).view(np.uint32),
                                      np.array([x for _, x in want], np.float32).view(np.uint32)), (trial, k)


# ---- the fixture on a scaled-down container -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind,dim", [("angular", 128), ("angular_int", 513), ("angular_int", 100)])
def test_fixture_premises_on_a_small_container(oracle, kind, dim):
    import torch

    n = 6000
    stride = row_bytes(kind, dim)
    boundaries = [1 << e for e in range(12, 40) if first_id_at(1 << e, stride) + 1 < n]
    m = Wide(kind, dim, n, boundaries, seed=dim, random_from=1000)   # the constructor checks the model's premises
    assert len(boundaries) >= 3
    # the container's rows: the gather of the device recipe, the labels, and the distances by gather
    rows = m.device_rows(torch, torch.device("cpu")).numpy()
    assert rows.tobytes() == m.rows(np.arange(n)).tobytes()
    lab = m.all_labels()
    assert np.array_equal(lab, m.labels(np.arange(n)))
    assert lab.max() < PALETTE + m.planted.size and np.array_equal(lab[m.planted], m.planted_label)
    direct = M.distances(kind, rows, m.queries)
    assert np.array_equal(direct.view(np.uint32), m.D[:, lab].view(np.uint32))
    # the planted ids: each boundary's neighbours, both ends, a copy of id 1 past the last boundary
    assert set(boundary_ids(boundaries, stride)) | {0, 1, n - 2, n - 1} <= set(m.planted.tolist())
    assert m.copy_id >= first_id_at(boundaries[-1], stride) and rows[m.copy_id].tobytes() == rows[1].tobytes()
    for q in range(m.queries.shape[0]):
        res = M.rank_prefix(direct[q], n, 1024)
        mine = set(m.planted[m.planted_query == q].tolist())
        assert {i for i, _ in res[:len(mine)]} == mine, q        # the planted rows come first
        assert rank(direct[q], 1024) == res
    # query 0's nearest palette row and its twin tie, and both are held by many ids
    assert direct[0, lab == 0][0] == direct[0, lab == m.twin][0]
    # the graph: boundary ids and planted ids are in C
    layers = sparse_graph(n, m.planted, 1)
    assert set(m.planted.tolist()) <= set(layers[1].lists)
