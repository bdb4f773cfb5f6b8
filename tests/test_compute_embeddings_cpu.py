"""compute_embeddings_and_save_to_disk (src/elements/embeddings/parsing.rs:102-152) without a device: the oracle's
restatement against a hand-worked answer and a plain-numpy one, every host-side status of
granne_b200_compute_embeddings(_device), and the Python argument checks."""
import ctypes as C

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers import composed_oracle as co
from helpers.fixtures import library  # noqa: F401  (autouse)

OK, INVALID, FORMAT, NO_DEVICE = 0, -1, -2, -5


def test_oracle_known_answer():
    table = co.table_image([[1, 2, -3], [0.5, 0, 1]])
    el = co.elements_image([[0, 1], [], [1]])
    img = co.compute_embeddings("angular_int", el, table)
    # [1.5, 2, -2] * 127 / 2 -> 95.25, 127, -127;  [] -> zeros;  [0.5, 0, 1] * 127 / 1 -> 63.5, 0, 127
    want = np.uint64(3).tobytes() + np.array([95, 127, -127, 0, 0, 0, 63, 0, 127], dtype=np.int8).tobytes()
    assert img.tobytes() == want
    ang = np.frombuffer(co.compute_embeddings("angular", el, table)[8:].tobytes(), dtype=np.float32).reshape(3, 3)
    assert np.array_equal(ang[1], np.zeros(3, np.float32))


def _numpy_image(kind, table, elements, normalize):
    """The image restated with numpy: the first term's row copied, the others added in order in f32; quantise the raw
    sum (angular_int) or normalise it (angular, with the oracle's pinned normalize_f32)."""
    table = np.asarray(table, dtype=np.float32)
    width = table.shape[1] if len(table) else 0
    rows = []
    for terms in elements:
        if width == 0:
            continue
        x = table[terms[0]].copy() if terms else np.zeros(width, np.float32)
        for t in terms[1:]:
            x = (x + table[t]).astype(np.float32)
        if kind == "angular":
            assert np.isfinite(x).all()
            rows.append(normalize(x).astype(np.float32).tobytes())
        else:
            assert not np.isnan(x).any()
            mx = np.abs(x).max() if x.size else np.float32(127)
            with np.errstate(all="ignore"):
                v = x * np.float32(127) / mx
            q = np.where(np.isnan(v), 0, np.clip(np.trunc(np.nan_to_num(v, posinf=127, neginf=-128)), -128, 127))
            rows.append(q.astype(np.int8).tobytes())
    return np.uint64(width if elements else 0).tobytes() + b"".join(rows)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_numpy(oracle, seed):
    rng = np.random.default_rng(seed)
    dim = int(rng.choice([1, 3, 31, 32, 33, 70]))
    m = int(rng.integers(1, 40))
    table = (rng.standard_normal((m, dim)) * 4).astype(np.float32)
    table[0] = -0.0                                   # a -0.0 row: stays -0.0 as a single term
    if m > 2:
        table[2] = -table[1]                          # x and -x: a zero sum
    if m > 3:
        table[3] = np.float32(1e-39) * rng.integers(-3, 4, dim)  # subnormal rows
    n = int(rng.integers(0, 250))
    elements = []
    for i in range(n):
        c = int(rng.integers(0, 12)) if i % 7 else 0  # empty elements
        elements.append([int(t) for t in rng.integers(0, m, c)])
    if n > 3 and m > 3:
        elements[1], elements[2], elements[3] = [0], [1, 2], [3, 3]
    ti, ei = co.table_image(table), co.elements_image(elements)
    for kind in ("angular_int", "angular"):
        img = co.compute_embeddings(kind, ei, ti, threads=3)
        assert img.tobytes() == _numpy_image(kind, table, elements, oracle.normalize_f32), (kind, seed)
    if n > 3 and m > 3:
        row = np.frombuffer(co.compute_embeddings("angular", ei, ti)[8 + 4 * dim: 8 + 8 * dim].tobytes(), np.float32)
        assert np.array_equal(np.signbit(row), np.ones(dim, bool))  # -0.0 / 0 norm: the row is kept


def test_oracle_empty_cases():
    table = co.table_image(np.ones((4, 5), np.float32))
    assert co.compute_embeddings("angular_int", co.elements_image([]), table).tobytes() == bytes(8)
    empty_table = np.uint64(5).tobytes()  # width 5, no rows
    assert co.compute_embeddings("angular", co.elements_image([[], []]), empty_table).tobytes() == bytes(8)
    with pytest.raises(co.NotFinite):
        co.compute_embeddings("angular_int", co.elements_image([[0]]), co.table_image([[np.nan, 1.0]]))
    with pytest.raises(co.NotFinite):
        co.compute_embeddings("angular", co.elements_image([[0, 0]]), co.table_image([[3e38, 1.0]]))
    # +inf in an angular_int sum quantises like the reference: inf/inf and finite/inf give 0
    img = co.compute_embeddings("angular_int", co.elements_image([[0, 0]]), co.table_image([[3e38, 1.0]]))
    assert img.tobytes() == np.uint64(2).tobytes() + bytes(2)


# ---- the C ABI without a device -----------------------------------------------------------------------------------
def _call(lib, kind, el, emb, out=None, cap=0, use_len=True):
    need = C.c_size_t(12345)
    eb = np.frombuffer(el, dtype=np.uint8) if el is not None else None
    mb = np.frombuffer(emb, dtype=np.uint8) if emb is not None else None
    rc = lib.granne_b200_compute_embeddings(kind, api._ptr(eb) if eb is not None else None, 0 if eb is None else eb.size,
                                            api._ptr(mb) if mb is not None else None, 0 if mb is None else mb.size, 0,
                                            out, cap, C.byref(need) if use_len else None)
    return rc, need.value


def _call_device(lib, kind, el, emb, d_out=None):
    n, dim = C.c_uint64(7), C.c_uint32(7)
    eb, mb = np.frombuffer(el, dtype=np.uint8), np.frombuffer(emb, dtype=np.uint8)
    rc = lib.granne_b200_compute_embeddings_device(kind, api._ptr(eb), eb.size, api._ptr(mb), mb.size, 0, d_out,
                                                   C.byref(n), C.byref(dim), None)
    return rc, n.value, dim.value


TABLE = co.table_image(np.arange(12, dtype=np.float32).reshape(4, 3))
ELEMENTS = co.elements_image([[0, 1], [], [3, 3, 2]])


@pytest.mark.parametrize("cut", [0, 4, 7, 8, 12, 20, 23])
def test_truncated_images_are_format_errors(library, cut):
    assert _call(library, 1, ELEMENTS[:cut], TABLE)[0] == FORMAT
    assert _call_device(library, 0, ELEMENTS[:cut], TABLE)[0] == FORMAT
    if cut < len(TABLE) and (cut < 8 or (cut - 8) % 12):
        assert _call(library, 0, ELEMENTS, TABLE[:max(cut, 3)])[0] == FORMAT


def test_format_errors(library):
    width0 = np.uint64(0).tobytes() + bytes(12)
    assert _call(library, 1, ELEMENTS, width0)[0] == FORMAT
    assert _call(library, 1, co.elements_image([[0], [4]]), TABLE)[0] == FORMAT  # id 4 >= 4 rows
    assert _call(library, 0, co.elements_image([[0xFFFFFF]]), TABLE)[0] == FORMAT
    assert _call_device(library, 1, co.elements_image([[0xFFFFFF]]), TABLE)[0] == FORMAT
    assert _call(library, 1, co.elements_image([[0]]), np.uint64(1).tobytes())[0] == FORMAT  # a table without rows
    assert "missing embedding id" in library.granne_b200_last_error().decode()
    # the table loader's rule: a width wider than the payload is malformed, so only width 1 can have no rows
    assert _call(library, 1, co.elements_image([[]]), np.uint64(3).tobytes())[0] == FORMAT


def test_invalid_arguments(library):
    for kind in (2, -1, 3):
        assert _call(library, kind, ELEMENTS, TABLE)[0] == INVALID
        assert _call_device(library, kind, ELEMENTS, TABLE)[0] == INVALID
    assert _call(library, 1, None, TABLE)[0] == INVALID
    assert _call(library, 1, ELEMENTS, None)[0] == INVALID
    assert _call(library, 1, ELEMENTS, TABLE, use_len=False)[0] == INVALID
    eb, mb = np.frombuffer(ELEMENTS, np.uint8), np.frombuffer(TABLE, np.uint8)
    assert library.granne_b200_compute_embeddings_device(1, api._ptr(eb), eb.size, api._ptr(mb), mb.size, 0, None, None,
                                                         None, None) == INVALID
    wide = co.table_image(np.zeros((2, 4097), np.float32))
    assert _call(library, 1, co.elements_image([[1]]), wide)[0] == INVALID
    assert _call_device(library, 0, co.elements_image([[1]]), wide)[0] == INVALID
    buf = np.zeros(64, np.uint8)
    rc, need = _call(library, 1, ELEMENTS, TABLE, out=api._ptr(buf), cap=8 + 9 - 1)
    assert rc == INVALID and need == 8 + 9
    assert _call(library, 1, ELEMENTS, TABLE, out=api._ptr(buf), cap=0)[0] == INVALID


def test_size_queries_need_no_device(library):
    assert _call(library, 1, ELEMENTS, TABLE) == (OK, 8 + 3 * 3)
    assert _call(library, 0, ELEMENTS, TABLE) == (OK, 8 + 3 * 3 * 4)
    assert _call_device(library, 0, ELEMENTS, TABLE) == (OK, 3, 3)
    big = co.elements_image([[i % 4] for i in range(1000)])
    assert _call(library, 0, big, TABLE) == (OK, 8 + 1000 * 3 * 4)
    assert _call(library, 1, co.elements_image([]), TABLE) == (OK, 8)
    assert _call(library, 1, co.elements_image([[], []]), np.uint64(1).tobytes()) == (OK, 8)
    assert _call_device(library, 1, co.elements_image([[], []]), np.uint64(1).tobytes()) == (OK, 2, 0)


def test_valid_input_without_a_device(library):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    buf = np.zeros(64, np.uint8)
    assert _call(library, 1, ELEMENTS, TABLE, out=api._ptr(buf), cap=buf.size)[0] == NO_DEVICE
    assert _call(library, 0, co.elements_image([]), TABLE, out=api._ptr(buf), cap=buf.size)[0] == NO_DEVICE
    assert _call_device(library, 1, ELEMENTS, TABLE, d_out=api._ptr(buf))[0] == NO_DEVICE
    with pytest.raises(granne_b200.GranneError) as e:
        granne_b200.compute_embeddings("angular_int", ELEMENTS, TABLE)
    assert e.value.code == NO_DEVICE


def test_python_argument_checks(library, tmp_path):
    for bad in ("embeddings", "nope"):
        with pytest.raises(ValueError):
            granne_b200.compute_embeddings(bad, ELEMENTS, TABLE)
        with pytest.raises(ValueError):
            granne_b200.compute_embeddings_device(bad, ELEMENTS, TABLE)
    with pytest.raises(ValueError):
        granne_b200.compute_embeddings("angular_int", ELEMENTS, TABLE, out=np.zeros(8 + 9 - 1, np.uint8))
    with pytest.raises(ValueError):
        granne_b200.compute_embeddings("angular_int", ELEMENTS, TABLE, out=np.zeros(64, np.float32))
    ro = np.zeros(64, np.uint8)
    ro.flags.writeable = False
    with pytest.raises(ValueError):
        granne_b200.compute_embeddings("angular_int", ELEMENTS, TABLE, out=ro)
    with pytest.raises(granne_b200.GranneError) as e:
        granne_b200.compute_embeddings("angular", ELEMENTS[:9], TABLE)
    assert e.value.code == FORMAT
    (tmp_path / "el").write_bytes(co.elements_image([[9]]))
    (tmp_path / "emb").write_bytes(TABLE)
    with pytest.raises(granne_b200.GranneError) as e:
        granne_b200.compute_embeddings_and_save_to_disk(str(tmp_path / "el"), str(tmp_path / "emb"),
                                                        str(tmp_path / "out"), show_progress=False)
    assert e.value.code == FORMAT
    assert not (tmp_path / "out").exists()
