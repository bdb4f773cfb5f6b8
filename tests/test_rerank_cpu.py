"""Host-side checks of the two-stage search calls that need no device: the candidate cap the header and the Python
binding share, and the statuses of calls without a handle."""
import os
import re

import numpy as np
import pytest

import granne_b200
from granne_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1


@pytest.fixture(scope="module")
def lib():
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def test_candidate_cap_matches_the_header():
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    m = re.search(r"#define GRANNE_B200_RERANK_MAX_CANDIDATES (\d+)", header)
    assert m and int(m.group(1)) == api.RERANK_MAX_CANDIDATES == api.EXACT_MAX_K


def test_calls_without_a_handle_are_invalid(lib):
    image = np.zeros(8 + 4 * 4, np.uint8)
    image[0] = 4
    assert lib.granne_b200_set_rerank_elements(None, api._ptr(image), image.size) == INVALID
    assert lib.granne_b200_set_rerank_elements_device(None, None, 0, 4) == INVALID
    q = np.zeros((1, 4), np.float32)
    ids = np.zeros(10, np.uint32)
    d = np.zeros(10, np.float32)
    assert lib.granne_b200_search_rerank_batch(None, api._ptr(q), 1, api.QUERY_RAW_F32, 200, 10, 10, api._ptr(ids),
                                               api._ptr(d), None, None) == INVALID
    assert lib.granne_b200_search_rerank_batch_device(None, None, 0, api.QUERY_RAW_F32, 200, 10, 10, None, None, None,
                                                      None, None) == INVALID
    assert lib.granne_b200_multi_set_rerank_elements(None, None, None) == INVALID
    assert lib.granne_b200_multi_search_rerank_batch(None, api._ptr(q), 1, api.QUERY_RAW_F32, 200, 10, 10,
                                                     None, None, None) == INVALID
    assert b"null" in lib.granne_b200_last_error()
