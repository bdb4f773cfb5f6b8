"""GranneBuilder::from_bytes (granne_b200_builder_from_index) without a GPU: the config and the index image are checked
on the host before any device call, so bad input gives a status, never a crash, and a valid image reaches the device
check (GRANNE_B200_ERR_NO_DEVICE: there is no CPU fallback).  GranneBuilder.from_files rejects incomplete arguments
before it calls the library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.data import build_fixture, index_from_lists
from helpers.fixtures import compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, INVALID, FORMAT, NO_DEVICE = 0, -1, -2, -5


@pytest.fixture(scope="module")
def fixture(library, oracle):
    el, g, index_bytes, elements_bytes, _ = build_fixture(oracle, "angular", 300, 8, seed=21, num_neighbors=10,
                                                          max_search=20)
    assert g.num_layers() >= 2
    return index_bytes, elements_bytes


def _no_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")


def from_index(lib, index_bytes, elements_bytes, kind=api.ANGULAR, **cfg):
    """Calls granne_b200_builder_from_index; returns (status, builder handle)."""
    c = api._build_config(cfg.get("num_neighbors", 30), cfg.get("max_search", 200), cfg.get("layer_multiplier", 15.0),
                          True, None)
    ib = np.frombuffer(index_bytes, dtype=np.uint8) if index_bytes else np.zeros(1, dtype=np.uint8)
    eb = np.frombuffer(elements_bytes, dtype=np.uint8)
    h = C.c_void_p()
    rc = lib.granne_b200_builder_from_index(C.byref(c), api._ptr(ib), len(index_bytes), kind, api._ptr(eb), eb.size,
                                            None, 0, 0, C.byref(h))
    return rc, h


def test_truncated_or_corrupted_images_are_format_errors(library, fixture):
    index_bytes, elements_bytes = fixture
    garbled = bytearray(index_bytes)
    garbled[1024 + 8:1024 + 40] = b"\xff" * 32  # the first layer's offset chunk
    for bad in [b"", b"granne", index_bytes[:1024], index_bytes[:-7], index_bytes[:len(index_bytes) // 2],
                b"grannf" + index_bytes[6:], b"granne{not json".ljust(1024, b" ") + index_bytes[1024:],
                bytes(garbled)]:
        rc, h = from_index(library, bad, elements_bytes)
        assert rc == FORMAT and not h.value, (bad[:16], len(bad), rc)
        assert library.granne_b200_last_error()


def test_too_many_layers_is_a_format_error(library, oracle, fixture):
    _, elements_bytes = fixture
    image = index_from_lists(oracle, [[[]]] * 25)  # 25 one-node layers; the builder holds at most 24
    assert len(api.inspect_index(image)) == 25
    rc, h = from_index(library, image, elements_bytes)
    assert rc == FORMAT and not h.value
    assert "layers" in library.granne_b200_last_error().decode()


@pytest.mark.parametrize("m", [0, 256])
def test_num_neighbors_outside_the_format_is_rejected(library, fixture, m):
    index_bytes, elements_bytes = fixture
    rc, h = from_index(library, index_bytes, elements_bytes, num_neighbors=m)
    assert rc == INVALID and not h.value
    assert "num_neighbors" in library.granne_b200_last_error().decode()


def test_null_arguments_are_rejected(library, fixture):
    index_bytes, elements_bytes = fixture
    c = api._build_config(30, 200, 15.0, True, None)
    h = C.c_void_p()
    assert library.granne_b200_builder_from_index(C.byref(c), None, 0, 0, None, 0, None, 0, 0, C.byref(h)) == INVALID
    ib = np.frombuffer(index_bytes, dtype=np.uint8)
    assert library.granne_b200_builder_from_index(None, api._ptr(ib), ib.size, 0, None, 0, None, 0, 0,
                                                  C.byref(h)) == INVALID
    assert library.granne_b200_builder_from_index_device_elements(C.byref(c), api._ptr(ib), ib.size, 0, None, 10, 8, 0,
                                                                  C.byref(h)) == INVALID
    assert not h.value


def test_a_valid_image_reaches_the_device_check(library, fixture):
    _no_gpu()
    index_bytes, elements_bytes = fixture
    rc, h = from_index(library, index_bytes, elements_bytes, num_neighbors=5)
    assert rc == NO_DEVICE and not h.value
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.GranneBuilder("angular", elements_bytes, index_bytes=index_bytes)
    assert ei.value.code == NO_DEVICE


def test_from_files_rejects_incomplete_arguments(tmp_path, fixture, monkeypatch):
    index_bytes, elements_bytes = fixture
    (tmp_path / "index").write_bytes(index_bytes)
    (tmp_path / "elements").write_bytes(elements_bytes)

    def no_library(*a, **k):
        raise AssertionError("the library was called")

    monkeypatch.setattr(api, "load_library", no_library)
    with pytest.raises(ValueError, match="elements_path"):
        granne_b200.GranneBuilder.from_files("angular", None, index_path=str(tmp_path / "index"))
    with pytest.raises(ValueError, match="embeddings_path"):
        granne_b200.GranneBuilder.from_files("embeddings", str(tmp_path / "elements"),
                                             index_path=str(tmp_path / "index"))
    with pytest.raises(ValueError, match="Invalid element type"):
        granne_b200.GranneBuilder.from_files("bogus", str(tmp_path / "elements"))


def test_from_files_reaches_the_library(library, tmp_path, fixture):
    _no_gpu()
    index_bytes, elements_bytes = fixture
    (tmp_path / "index").write_bytes(index_bytes)
    (tmp_path / "elements").write_bytes(elements_bytes)
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.GranneBuilder.from_files("angular", str(tmp_path / "elements"), index_path=str(tmp_path / "index"),
                                             num_neighbors=5)
    assert ei.value.code == NO_DEVICE
    (tmp_path / "short").write_bytes(index_bytes[:2000])
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.GranneBuilder.from_files("angular", str(tmp_path / "elements"), index_path=str(tmp_path / "short"))
    assert ei.value.code == FORMAT


def test_cxx_from_bytes_reports_statuses_without_a_device(library, tmp_path, fixture):
    _no_gpu()
    exe = compile_cxx_client("cxx_resume_client.cpp", tmp_path)
    index_bytes, elements_bytes = fixture
    (tmp_path / "index").write_bytes(index_bytes)
    (tmp_path / "elements").write_bytes(elements_bytes)
    r = subprocess.run([exe, "nodevice", str(tmp_path / "index"), str(tmp_path / "elements")], capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0 and "nodevice ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
