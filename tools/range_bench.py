"""Time of the exact range search (Granne.exact_range_count_device / exact_range_search_device) per batch of queries, next
to exact_search_batch_device(k = 10) on the same data and card, and the time of range_graph.  The data are clustered
vectors this tool generates itself (1M x 128-d angular f32 and 10M x 100-d angular_int with the defaults), indexed by a
single-layer index: the exact calls read no graph.  For each target median range size the radius is found by bisection
on the counts of the timed batch.  Every time is the median of --reps CUDA-event timings, with their min and max.
Prints one JSON line per configuration; the card's name and power limit are read in the same run.

    python tools/range_bench.py --nq 1024 --targets 10,1000,100000
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import granne_b200  # noqa: E402
from granne_b200 import build  # noqa: E402


def _card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception:  # noqa: BLE001 - reported as unknown
        return "unknown"


def _times(fn, reps):
    """(median, min, max) seconds of fn over reps CUDA-event timings, after one warm-up call."""
    import torch

    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / 1e3)
    return [round(float(np.median(out)) * 1e3, 3), round(min(out) * 1e3, 3), round(max(out) * 1e3, 3)]


def _radius_for(g, q, target):
    """A radius whose median count over the queries q is about target (bisection on the device counts)."""
    lo, hi = 0.0, 2.0
    for _ in range(24):
        mid = (lo + hi) / 2
        med = float(np.median(g.exact_range_count_device(q, mid).cpu().numpy()))
        if med < target:
            lo = mid
        else:
            hi = mid
    return hi


def _config(name, g, q, targets, reps):
    import torch

    dev = q.device
    rows = {"config": name, "n": len(g), "dim": g.dim, "nq": q.shape[0], "card": _card(),
            "exact_k10_ms": _times(lambda: g.exact_search_batch_device(q, 10), reps), "ranges": []}
    for target in targets:
        r = _radius_for(g, q, target)
        counts = g.exact_range_count_device(q, r)
        off = torch.zeros(q.shape[0] + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=off[1:])
        total = int(off[-1])
        out = (torch.empty(total, dtype=torch.int32, device=dev), torch.empty(total, dtype=torch.float32, device=dev))
        c = counts.cpu().numpy()
        rows["ranges"].append({
            "radius": r, "median_count": int(np.median(c)), "min_count": int(c.min()), "max_count": int(c.max()),
            "count_ms": _times(lambda: g.exact_range_count_device(q, r, out=counts), reps),
            "fill_ms": _times(lambda: g.exact_range_search_device(q, r, off, out=out), reps)})
        del out
        g.stream_status()
    print(json.dumps(rows), flush=True)


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--targets", default="10,1000,100000", help="median range sizes")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--f32-n", type=int, default=1000000)
    ap.add_argument("--i8-n", type=int, default=10000000)
    ap.add_argument("--graph-n", type=int, default=1000000, help="elements of the range_graph run (0: skip)")
    ap.add_argument("--graph-radius", type=float, default=0.01, help="a near-duplicate radius")
    args = ap.parse_args()
    build.build()
    from oracle import granne_oracle as go
    from helpers.data import clustered_vectors
    from helpers.exact_oracle import single_layer_index

    go.build_lib()
    targets = [int(t) for t in args.targets.split(",") if t]
    dev = torch.device("cuda", 0)

    raw = torch.from_numpy(clustered_vectors(args.f32_n, 128, seed=1)).to(dev)
    g = granne_b200.Granne.from_device_elements(single_layer_index(go, args.f32_n), "angular",
                                                granne_b200.elements_from_raw_device("angular", raw))
    del raw
    q = torch.from_numpy(clustered_vectors(args.nq, 128, seed=2)).to(dev)
    _config("f32_1m_128", g, q, targets, args.reps)
    if args.graph_n:
        n = min(args.graph_n, len(g))
        if n < len(g):
            g.close()
            raw = torch.from_numpy(clustered_vectors(n, 128, seed=1)).to(dev)
            g = granne_b200.Granne.from_device_elements(single_layer_index(go, n), "angular",
                                                        granne_b200.elements_from_raw_device("angular", raw))
        torch.cuda.synchronize()
        t0 = time.time()
        off, _, _ = g.range_graph(args.graph_radius, out="device")
        torch.cuda.synchronize()
        s = time.time() - t0
        deg = torch.diff(off).cpu().numpy()
        print(json.dumps({"config": "range_graph_f32_128", "n": n, "radius": args.graph_radius, "card": _card(),
                          "seconds": round(s, 2), "edges": int(deg.sum()), "median_degree": int(np.median(deg)),
                          "max_degree": int(deg.max())}), flush=True)
    g.close()

    raw = torch.from_numpy(clustered_vectors(args.i8_n, 100, seed=3)).to(dev)
    el = granne_b200.elements_from_raw_device("angular_int", raw)
    del raw
    g = granne_b200.Granne.from_device_elements(single_layer_index(go, args.i8_n), "angular_int", el)
    q = torch.from_numpy(clustered_vectors(args.nq, 100, seed=4)).to(dev)
    _config("i8_10m_100", g, q, targets, args.reps)
    g.close()


if __name__ == "__main__":
    main()
