"""The reference's index tests written against include/granne_b200.hpp and run on the GPU (tests/helpers/
cxx_client.cpp: build_and_search_float / _int8, write_and_load, append_elements, reorder_index, compute_distance).
Named to run after the Python suites."""
import pytest

from helpers.fixtures import cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)

pytestmark = pytest.mark.gpu


def test_reference_style_cxx_tests_pass_on_the_gpu(tmp_path):
    r = cxx_client("cxx_client.cpp", ["gpu"], tmp_path, timeout=900)
    assert r.returncode == 0 and "gpu ok" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
