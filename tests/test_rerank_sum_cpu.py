"""Host-side checks of the SumEmbeddings re-rank container that need no device: the statuses of the attach calls
without a handle, the exported symbols, and their declarations in the Rust shim and the C++ header."""
import os
import re

import numpy as np
import pytest

import granne_b200
from granne_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1
NEW_SYMBOLS = ("granne_b200_set_rerank_embeddings", "granne_b200_multi_set_rerank_embeddings")


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def _images():
    from helpers import embeddings_oracle as eo

    table = np.ones((3, 4), np.float32)
    return (np.frombuffer(eo.elements_image([[0, 1], [2]]), np.uint8),
            np.frombuffer(eo.table_image(table), np.uint8))


def test_calls_without_a_handle_are_invalid(lib):
    el, emb = _images()
    assert lib.granne_b200_set_rerank_embeddings(None, api._ptr(el), el.size, api._ptr(emb), emb.size) == INVALID
    assert b"null" in lib.granne_b200_last_error()
    assert lib.granne_b200_set_rerank_embeddings(None, None, 0, None, 0) == INVALID
    assert b"null" in lib.granne_b200_last_error()
    import ctypes as C

    ptrs = (C.c_void_p * 1)(el.ctypes.data)
    lens = (C.c_size_t * 1)(el.size)
    assert lib.granne_b200_multi_set_rerank_embeddings(None, ptrs, lens, api._ptr(emb), emb.size) == INVALID
    assert b"null" in lib.granne_b200_last_error()
    assert lib.granne_b200_multi_set_rerank_embeddings(None, None, None, None, 0) == INVALID
    assert b"null" in lib.granne_b200_last_error()


def test_symbols_exported(lib):
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name


def test_rust_shim_and_cxx_header_declare_them():
    rust = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\bfn %s\(" % name, rust), name
        assert re.search(r"\bint %s\(" % name, header), name
    hpp = open(os.path.join(ROOT, "include", "granne_b200.hpp")).read()
    assert "granne_b200_set_rerank_embeddings(" in hpp
