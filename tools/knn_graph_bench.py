"""Throughput of the k-NN graph (Granne.knn_graph) and of queries by element id against the same queries as ELEMENT
rows, on an index of clustered vectors that this tool generates and builds itself (with the defaults it has C2's
shape, 1M x 128-d angular, but it is not bench.py's C2 data or index); recall@k of the graph against
knn_graph(exact=True) on a sample of ids.  Prints one JSON line.  CUDA events time the device calls; the card's name and power limit are printed with
the numbers they belong to.

    python tools/knn_graph_bench.py --n 1000000 --dim 128 --k 10 --max-search 200
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import granne_b200  # noqa: E402
from granne_b200 import build  # noqa: E402


def _card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception:  # noqa: BLE001 - reported as unknown
        return "unknown"


def _timed(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--max-search", type=int, default=200)
    ap.add_argument("--nq", type=int, default=65536, help="queries per timed id / element call")
    ap.add_argument("--sample", type=int, default=2000, help="ids whose graph rows are checked against exact")
    args = ap.parse_args()
    build.build()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from helpers.data import clustered_vectors

    t0 = time.time()
    raw = clustered_vectors(args.n, args.dim, seed=1)
    b = granne_b200.GranneBuilder("angular", granne_b200.elements_from_raw("angular", raw), max_search=args.max_search)
    b.build()
    g = b.get_index()
    build_s = time.time() - t0
    dev = torch.device("cuda", g.device)
    nq = min(args.nq, len(g))
    ids = torch.randint(0, len(g), (nq,), dtype=torch.int64, device=dev).to(torch.int32)
    rows = g.get_elements_device(ids)
    t_id = _timed(lambda: g.search_batch_device(ids, args.max_search, args.k, by_id=True), 5)
    t_ex = _timed(lambda: g.search_batch_device(ids, args.max_search, args.k, exclude_self=True), 5)
    t_el = _timed(lambda: g.search_batch_device(rows, args.max_search, args.k, already_element=True), 5)
    torch.cuda.synchronize()
    t0 = time.time()
    gi, _, _ = g.knn_graph(args.max_search, args.k)
    graph_s = time.time() - t0
    rng = np.random.default_rng(0)
    sample = rng.choice(len(g), size=min(args.sample, len(g)), replace=False).astype(np.uint32)
    xi, _, xc = g.exact_search_batch(sample, args.k, exclude_self=True)
    hits = sum(len(set(gi[s].tolist()) & set(xi[j, :xc[j]].tolist())) for j, s in enumerate(sample))
    print(json.dumps({
        "card": _card(), "n": len(g), "dim": args.dim, "k": args.k, "max_search": args.max_search,
        "build_s": round(build_s, 1), "graph_s": round(graph_s, 2), "graph_elements_per_s": round(len(g) / graph_s),
        "id_qps": round(nq / t_id), "id_excluding_qps": round(nq / t_ex), "element_qps": round(nq / t_el),
        "recall_at_k_vs_exact": round(hits / float(max(1, int(xc.sum()))), 4),
    }))


if __name__ == "__main__":
    main()
