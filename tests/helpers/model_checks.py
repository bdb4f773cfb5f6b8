"""Assertions that hold a query call's outputs to the NumPy model (ref_model.py): bit for bit, and against float64."""
import numpy as np

from helpers import ref_model as M


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def assert_same(got, want, k, what="", id_dtype=np.uint32):
    """got: a call's (ids, dists, counts[, stats]); want: model results [[(id, dist)]] and, optionally, stats."""
    want_res, want_stats = want if isinstance(want, tuple) else (want, None)
    ids, dists, counts = (np.asarray(x) for x in got[:3])
    wi, wd, wc = M.as_arrays(want_res, k, id_dtype)
    assert np.array_equal(counts.view(np.uint32), wc), "%s: counts %s, model %s" % (what, counts, wc)
    assert np.array_equal(ids.view(id_dtype), wi), "%s: ids" % what
    assert np.array_equal(bits(dists), bits(wd)), "%s: distance bits" % what
    if want_stats is not None:
        assert np.array_equal(np.asarray(got[3])[:, :3].astype(np.uint64), np.asarray(want_stats, dtype=np.uint64)), \
            "%s: stats" % what


def assert_within_f64_bound(rows, queries, results):
    """Each returned f32 distance lies within (dim + 64) 2^-24 sum|x_i y_i| + 2^-24 of the float64 distance.  rows:
    the element rows, or anything indexed by element id that gives them (a row gather of a large container)."""
    y = np.asarray(queries, dtype=np.float64)
    dim = y.shape[1]
    ids, dists, counts = results[:3]
    for q in range(y.shape[0]):
        c = int(counts[q])
        sel = np.asarray(ids[q, :c], dtype=np.int64)
        prod = np.asarray(rows[sel], dtype=np.float64).reshape(c, dim) * y[q]
        exact = np.maximum(0.0, 1.0 - prod.sum(1))
        bound = (dim + 64) * 2.0 ** -24 * np.abs(prod).sum(1) + 2.0 ** -24
        assert (np.abs(np.asarray(dists[q, :c], dtype=np.float64) - exact) <= bound).all(), "query %d" % q
