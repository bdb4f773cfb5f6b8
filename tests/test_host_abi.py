"""CPU-side tests of the product: the C-ABI library loads and exports every symbol include/granne_b200.h declares,
the host loader decodes granne index files exactly like the oracle (reference: src/index/io.rs:72-113,
src/slice_vector/set_vector.rs:57-115, src/slice_vector/offsets.rs:178-259), and error paths return statuses
instead of panicking.  No compute calls (no GPU here)."""
import ctypes
import os
import re

import numpy as np
import pytest

import granne_b200
from granne_b200 import api
from helpers.data import build_fixture
from helpers.fixtures import library  # noqa: F401  (autouse)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(library):
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    names = set(re.findall(r"\b(granne_b200_[a-z0-9_]+)\s*\(", header))
    assert len(names) >= 20
    raw = ctypes.CDLL(granne_b200.library_path())
    for n in sorted(names):
        assert hasattr(raw, n), n
    assert library.granne_b200_abi_version() == 2


def test_no_torch_or_cxx_types_in_the_header():
    header = open(os.path.join(ROOT, "include", "granne_b200.h")).read()
    code = re.sub(r"/\*.*?\*/", "", header, flags=re.S)  # strip comments
    assert "torch" not in code and "std::" not in code and "at::" not in code and "#include <c" not in code


@pytest.mark.parametrize("n,dim,m", [(1, 8, 5), (59, 8, 5), (60, 8, 5), (61, 8, 5), (1500, 16, 20), (3000, 8, 30)])
def test_loader_decodes_layers_like_the_oracle(library, oracle, n, dim, m):
    # sizes around the 60-offsets-per-chunk boundary (offsets.rs:7,249-259)
    el, g, index_bytes, _, _ = build_fixture(oracle, "angular", n, dim, seed=n, num_neighbors=m, max_search=30)
    shape = api.inspect_index(index_bytes)
    assert len(shape) == g.num_layers()
    for l, (cnt, maxdeg, width) in enumerate(shape):
        assert cnt == g.layer_len(l)
        rows = api.decode_layer(index_bytes, l)
        assert rows.shape == (cnt, width) and width % 8 == 0 and width >= maxdeg
        seen_max = 0
        for i in range(cnt):
            expect = g.get_neighbors(i, l)
            seen_max = max(seen_max, len(expect))
            assert rows[i, :len(expect)].tolist() == expect
            assert (rows[i, len(expect):] == 0xFFFFFFFF).all()
        assert seen_max == maxdeg


def test_loader_handles_raw_and_vbyte_lists(library, oracle):
    # hand-made index: lists that exercise the raw-u32 rule (set_vector.rs:275-283), empty lists, <4 entries
    import json

    lists = [[37717, 660380], [], [5], [5, 5], list(range(10)), [1, 301, 70301, 20070301], [2**32 - 2]]
    n = 700000
    lists = [l for l in lists] + [[i] for i in range(80)]
    # build the layer blob with the oracle's set_encode; offsets chunked by 60
    enc = [oracle.set_encode(sorted(l)) for l in lists]
    offsets = [0]
    for e in enc:
        offsets.append(offsets[-1] + len(e))
    nchunks = 1 + len(lists) // 60
    chunks = bytearray()
    for c in range(nchunks):
        offs = offsets[c * 60:(c + 1) * 60]
        initial = offs[0] if offs else 0
        chunks += int(initial).to_bytes(8, "little")
        prev = initial
        for i in range(60):
            if i < len(offs):
                chunks += int(offs[i] - prev).to_bytes(2, "little")
                prev = offs[i]
            else:
                chunks += b"\xff\xff"
    blob = len(chunks).to_bytes(8, "little") + bytes(chunks) + b"".join(enc)
    meta = "granne" + json.dumps({"version": 2, "num_elements": 2**32 - 1, "num_layers": 1, "num_neighbors": 2,
                                  "layer_counts": [len(lists)], "layer_sizes": [len(blob)], "compressed": True,
                                  "granne_version": "0.5.2"})
    image = meta.encode().ljust(1024, b" ") + blob
    # ids exceed the layer size -> the loader must reject (every neighbour must address a node of its layer)
    with pytest.raises(granne_b200.GranneError) as ei:
        api.inspect_index(image)
    assert ei.value.code == -2
    # same lists with in-range ids decode exactly
    small = [[min(v, len(lists) - 1) for v in l] for l in lists]
    enc = [oracle.set_encode(sorted(l)) for l in small]
    assert [oracle.set_decode(e) for e in enc] == [sorted(l) for l in small]


def test_format_errors_are_statuses_not_crashes(library, oracle):
    el, g, index_bytes, elements_bytes, _ = build_fixture(oracle, "angular", 200, 8, seed=3, num_neighbors=8,
                                                          max_search=20)
    for bad in [b"", b"granne", b"grannf" + index_bytes[6:], index_bytes[:1024], index_bytes[:-7],
                b"granne{not json".ljust(1024, b" ") + index_bytes[1024:]]:
        with pytest.raises(granne_b200.GranneError) as ei:
            api.inspect_index(bad)
        assert ei.value.code == -2, bad[:16]
    assert "granne" in str(ei.value) or "metadata" in str(ei.value) or "layer" in str(ei.value)


def test_open_without_a_gpu_fails_loudly(library, oracle):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    el, g, index_bytes, elements_bytes, _ = build_fixture(oracle, "angular", 100, 8, seed=4, num_neighbors=8,
                                                          max_search=20)
    with pytest.raises(granne_b200.GranneError) as ei:
        granne_b200.Granne.from_bytes(index_bytes, "angular", elements_bytes)
    assert ei.value.code == -5  # GRANNE_B200_ERR_NO_DEVICE: no CPU fallback
    with pytest.raises(ValueError):
        granne_b200.Granne.from_bytes(index_bytes, "bogus", elements_bytes)


@pytest.mark.parametrize("n,dim,m", [(1, 8, 5), (60, 8, 5), (61, 8, 5), (1500, 16, 20), (4000, 8, 30)])
def test_writer_is_byte_identical_to_the_oracle_writer(library, oracle, n, dim, m):
    # Index::write_index (src/index/io.rs:11-70, set_vector.rs:117-148,169-221, offsets.rs:233-241): the product's
    # writer re-encodes an oracle-written image byte for byte (header JSON, offset chunks, raw-vs-vbyte rule)
    el, g, index_bytes, _, _ = build_fixture(oracle, "angular", n, dim, seed=n + 1, num_neighbors=m, max_search=30)
    assert api.reencode_index(index_bytes) == index_bytes


def test_writer_round_trips_the_golden_images(library):
    import glob

    for path in glob.glob(os.path.join(ROOT, "tests", "golden", "*.npz")):
        image = np.load(path)["index"].tobytes()
        assert api.reencode_index(image) == image


def test_header_is_plain_c_and_links_from_c(library, tmp_path):
    # the boundary is a C ABI: the header compiles as strict C99 and a C program links against the shared library
    import shutil
    import subprocess

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "client.c"
    src.write_text(r'''
#include <stdio.h>
#include <string.h>
#include "granne_b200.h"
int main(void) {
    granne_b200_index* h = NULL;
    uint64_t layers = 99;
    unsigned char junk[16] = {0};
    if (granne_b200_abi_version() != GRANNE_B200_ABI_VERSION) return 1;
    if (granne_b200_inspect_index(junk, sizeof junk, &layers, NULL, NULL, NULL, 0) != GRANNE_B200_ERR_FORMAT) return 2;
    if (strlen(granne_b200_last_error()) == 0) return 3;
    if (granne_b200_open(NULL, 0, GRANNE_B200_ANGULAR, NULL, 0, NULL, 0, 0, &h) == GRANNE_B200_OK) return 4;
    if (granne_b200_len(NULL) != 0) return 5;
    printf("ok\n");
    return 0;
}
''')
    exe = str(tmp_path / "client")
    libdir = os.path.dirname(api.library_path())
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I" + os.path.join(ROOT, "include"),
                           str(src), "-o", exe, "-L" + libdir, "-lgranne_b200", "-Wl,-rpath," + libdir])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout, r.stderr)


def test_rust_shim_declarations_match_the_header():
    # bindings/rust cannot be compiled here (no rustc): keep its extern block in sync with the C header mechanically
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "granne_b200.h")).read(), flags=re.S)
    shim = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    extern = shim[shim.index('extern "C" {'):shim.index("pub const ANGULAR")]
    decls = re.findall(r"fn (granne_b200_\w+)\s*\((.*?)\)\s*(?:->\s*[\w:\* ]+)?;", extern, flags=re.S)
    assert len(decls) >= 20

    def arity(params):
        params = params.strip()
        return 0 if params in ("", "void") else params.count(",") + 1

    for name, params in decls:
        m = re.search(r"\b%s\s*\((.*?)\)\s*;" % name, header, flags=re.S)
        assert m, name + " is not declared in granne_b200.h"
        rust_params = params.strip().rstrip(",")
        assert arity(rust_params) == arity(m.group(1)), name
    for used in set(re.findall(r"\b(granne_b200_\w+)\(", shim)):
        assert any(used == d[0] for d in decls), used + " is called but not declared in the extern block"


@pytest.mark.parametrize("seed", range(12))
def test_random_graphs_decode_and_reencode_like_the_oracle(library, oracle, seed):
    # differential check on random adjacency lists: empty / short / long lists, small and large id gaps (raw-vs-vbyte
    # rule, set_vector.rs:130-141), layer sizes around the 60-offsets-per-chunk boundary (offsets.rs:7)
    from helpers.data import index_from_lists

    rng = np.random.default_rng(seed)
    sizes = sorted(int(x) for x in rng.choice([1, 2, 59, 60, 61, 119, 120, 121, 500, 3000], size=rng.integers(1, 4),
                                              replace=False))
    n_last = sizes[-1]
    layers = []
    for n in sizes:
        lists = []
        for _ in range(n):
            deg = int(rng.choice([0, 1, 2, 3, 4, 5, 15, 30, 40], p=[.1, .1, .1, .1, .1, .1, .2, .15, .05]))
            deg = min(deg, n)
            if rng.random() < 0.3:  # clustered ids: small deltas compress well
                start = int(rng.integers(0, max(1, n - deg + 1)))
                ids = list(range(start, start + deg))
            else:
                ids = rng.choice(n, size=deg, replace=False).tolist()
            lists.append(ids)
        layers.append(lists)
    image = index_from_lists(oracle, layers)
    g = oracle.Granne.from_bytes(image, oracle.Elements.angular(np.ones((n_last, 2), dtype=np.float32)))
    shape = api.inspect_index(image)
    assert [s[0] for s in shape] == sizes
    for l, lists in enumerate(layers):
        rows = api.decode_layer(image, l)
        assert shape[l][1] == max((len(x) for x in lists), default=0)
        for i in range(0, sizes[l], max(1, sizes[l] // 200)):
            want = sorted(lists[i])
            assert g.get_neighbors(i, l) == want
            assert rows[i, :len(want)].tolist() == want and (rows[i, len(want):] == 0xFFFFFFFF).all()
    assert api.reencode_index(image) == image == g.to_bytes()
