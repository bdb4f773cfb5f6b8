"""include/granne_b200.hpp (the C++ mirror of granne's Rust API) compiles warning-free, links against the C ABI
library and, without a GPU, fails loudly with GRANNE_B200_ERR_NO_DEVICE instead of falling back to the CPU."""
import subprocess

import pytest

from helpers.fixtures import compile_cxx_client
from helpers.fixtures import library  # noqa: F401  (autouse)


def test_cxx_header_compiles_and_has_no_cpu_fallback(tmp_path):
    import torch

    exe = compile_cxx_client("cxx_client.cpp", tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    r = subprocess.run([exe, "nodevice"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "nodevice ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
