"""What the test modules share: the built library, the C++ clients, dense element images, the exact calls' cases, a
SumEmbeddings case generator and the exact comparison of a query call's results.  A module imports the fixtures it uses
by name (`from helpers.fixtures import library`)."""
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

import granne_b200
from helpers import composed_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@pytest.fixture(scope="module", autouse=True)
def library():
    """The extension, built for sm_90a if it is out of date, and loaded: once per module that imports this."""
    from granne_b200 import build

    build.build()
    return granne_b200.load_library()


def compile_cxx_client(source, out_dir):
    """Compiles tests/helpers/<source> against include/ and the built library (the `library` fixture), warnings as
    errors; returns the executable's path.  Skips the test when there is no g++."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    libdir = os.path.dirname(granne_b200.library_path())
    exe = os.path.join(str(out_dir), os.path.splitext(source)[0])
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "helpers", source), "-o", exe,
                           "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    return exe


def cxx_client(source, args, tmp_path, timeout=120):
    """Compiles tests/helpers/<source> (compile_cxx_client) and runs it with `args`; returns the completed process
    with its stdout and stderr as text."""
    exe = compile_cxx_client(source, tmp_path)
    return subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=timeout)


def elements_image(rows):
    """The file image of dense element rows (f32 or i8): u64 width | rows."""
    rows = np.ascontiguousarray(rows)
    return np.uint64(rows.shape[1]).tobytes() + rows.tobytes()


def image_rows(image, dtype):
    """The rows of a dense elements file image."""
    dim = int(np.frombuffer(bytes(image[:8]), dtype=np.uint64)[0])
    return np.frombuffer(bytes(image[8:]), dtype=dtype).reshape(-1, dim)


def elements_from_raw(kind, raw):
    """The element rows elements_from_raw makes of raw vectors: normalised f32 ("angular") or quantised i8."""
    return image_rows(granne_b200.elements_from_raw(kind, raw), np.float32 if kind == "angular" else np.int8)


class ExactCase:
    """A GPU handle over single_layer_index(index_len) (exact calls read no neighbour list) and the oracle container
    over the same elements: dense `rows`, or the file `images` (elements, embeddings table) of a SumEmbeddings
    container.  index_len defaults to the container's length."""

    def __init__(self, go, kind, rows=None, index_len=None, images=None):
        self.go, self.kind = go, kind
        self.eb, self.mb = (elements_image(rows), None) if images is None else images
        self.o = co.Container(kind, self.eb, self.mb)
        self.n = len(self.o) if index_len is None else index_len
        self.index_bytes = co.single_layer_index(go, self.n)
        self.g = granne_b200.Granne.from_bytes(self.index_bytes, kind, self.eb, self.mb)

    @functools.cached_property
    def el(self):
        """The CPU oracle's Elements over the same images (for dist_to_element)."""
        return self.go.Elements.from_bytes(self.kind, self.eb, self.mb)


def sum_images(el):
    """The file images (elements, embeddings table) of an oracle SumEmbeddings container."""
    return el.to_bytes(0), el.to_bytes(1)


def sum_case(dim, n, seed, num_rows=300, repeat_terms=False):
    """File images (elements, embeddings table) of n SumEmbeddings elements of 0, 1, 2, 7, 33 and 40 terms in turn
    over a standard-normal table of num_rows rows; repeat_terms: an element of more than 3 terms repeats its first
    term third."""
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((num_rows, dim))).astype(np.float32)
    counts = [0, 1, 2, 7, 33, 40]
    elements = []
    for i in range(n):
        ids = rng.integers(0, num_rows, counts[i % len(counts)])
        if repeat_terms and ids.size > 3:
            ids[2] = ids[0]
        elements.append([int(t) for t in ids])
    return co.elements_image(elements), co.table_image(table)


def _bits(a):
    a = np.asarray(a)
    return a.view("u%d" % a.itemsize)


def assert_same(got, want, what="", stats=False):
    """A query call's (ids, dists, counts[, stats]) equal `want` exactly: counts, ids (naming the first queries whose
    ids differ), distance bits and, with `stats`, stats[:, :3] (not compared when either side has None: a call without
    stats).  Ids and counts of 4 bytes are compared as uint32 bits, so int32 device tensors match uint32 arrays."""
    gi, gd, gc = (_bits(x) for x in got[:3])
    wi, wd, wc = (_bits(x) for x in want[:3])
    assert np.array_equal(gc, wc), what + " counts"
    bad = np.nonzero((gi != wi).any(axis=1))[0] if gi.shape == wi.shape else np.arange(len(wi))
    assert bad.size == 0, "%s ids differ for queries %s: want %s got %s" % (what, bad[:5], wi[bad[:1]], gi[bad[:1]])
    assert np.array_equal(gd, wd), what + " dists"
    if stats and got[3] is not None and want[3] is not None:
        assert np.array_equal(np.asarray(got[3])[:, :3], np.asarray(want[3])[:, :3]), \
            what + " n_dist/n_expand/n_neighbors"
