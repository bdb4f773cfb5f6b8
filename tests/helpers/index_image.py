"""Comparison of two index images that names the first neighbour list where they differ."""
import pytest


def assert_same_index(oracle, image, ref, el, what=""):
    """image (GPU builder) == ref (oracle Granne) byte for byte; on a mismatch name the first differing list."""
    want = ref.to_bytes()
    if image == want:
        return
    # compare both as loaded from their files (sorted lists; a built index keeps insertion order)
    got, ref = oracle.Granne.from_bytes(image, el), oracle.Granne.from_bytes(want, el)
    assert got.num_layers() == ref.num_layers(), "%s: %d layers, oracle %d" % (what, got.num_layers(), ref.num_layers())
    for layer in range(ref.num_layers()):
        assert got.layer_len(layer) == ref.layer_len(layer), "%s: layer %d length" % (what, layer)
        for i in range(ref.layer_len(layer)):
            a, b = got.get_neighbors(i, layer), ref.get_neighbors(i, layer)
            assert a == b, "%s: layer %d node %d: gpu %s, oracle %s" % (what, layer, i, a, b)
    pytest.fail("%s: every neighbour list agrees but the index images differ (%d vs %d bytes)"
                % (what, len(image), len(want)))
