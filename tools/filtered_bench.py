"""Measures filtered search (Granne.search_batch_filtered_device) against unfiltered search and the exact filtered
search over the same bitmap, on one H100.

Data: bench.py's clustered 10M x 128 f32 rows (rerank_bench.generate) with a GPU-built index (M = 30, max_search 200);
1024 raw queries in one device batch, k = 10, max_search 200 and 800.  Filters: one random filter admitting 100 %, 50 %,
10 % and 1 % of n.  Per (max_search, share):
  * QPS of search_batch_device and search_batch_filtered_device, timed by CUDA events over --windows windows of
    --calls calls each, the two calls alternating window by window; median, min and max of the windows;
  * recall@10 of the filtered search over the whole batch against the exact filtered answer (one
    exact_search_filtered_device call over the same bitmap), also over its first 64 queries, and the share of the
    1024 queries that returned fewer than k;
  * the time of that exact_search_filtered_device call on the 1024 queries, as queries per second: where the exact
    path and the graph path cross over.
Prints the card name and power limit read in the same run, then one JSON line per (max_search, share).

    python tools/filtered_bench.py [--elements 10000000] [--windows 7] [--calls 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exact_bench import card  # noqa: E402
from rerank_bench import generate  # noqa: E402


def window(torch, s, fn, calls):
    """Device seconds of `calls` back-to-back calls of fn(s), from CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(calls):
        fn(s)
    e1.record(s)
    s.synchronize()
    return e0.elapsed_time(e1) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=10_000_000)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=5)
    a = ap.parse_args()
    import torch

    import granne_b200

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    dev = torch.device("cuda", 0)
    n, dim, k, nq = a.elements, 128, 10, 1024
    rows, q = generate(torch, granne_b200, n, dim, 1234, ("angular",), nq)
    t0 = time.perf_counter()
    b = granne_b200.GranneBuilder.from_device_elements("angular", rows["angular"], num_neighbors=30, max_search=200)
    b.build()
    index = b.index_bytes().tobytes()
    b.close()
    torch.cuda.empty_cache()
    print(json.dumps({"n": n, "dim": dim, "build_s": time.perf_counter() - t0}), flush=True)
    g = granne_b200.Granne.from_device_elements(index, "angular", rows["angular"])
    rng = np.random.default_rng(7)
    s = torch.cuda.Stream()
    for share in (1.0, 0.5, 0.1, 0.01):
        mask = np.ones(n, bool) if share == 1.0 else rng.random(n) < share
        admitted = int(mask.sum())
        words = granne_b200.api._filter_words(mask, n)
        dw = torch.from_numpy(words.view(np.int32)).to(dev)
        # the exact filtered answer for the whole batch, and the exact path's time on it
        with torch.cuda.stream(s):
            def exact(st):
                return g.exact_search_filtered_device(q, dw, None, k, stream=st)

            exact(s)
            ex_t = [window(torch, s, exact, 1) for _ in range(3)]
            truth = exact(s)[0]
            s.synchronize()
            truth = truth.cpu().numpy().view(np.uint32)
        g.stream_status()
        for ef in (200, 800):
            with torch.cuda.stream(s):
                def plain(st):
                    return g.search_batch_device(q, ef, k, stream=st)

                def filt(st):
                    return g.search_batch_filtered_device(q, dw, None, ef, k, stream=st)

                for fn in (plain, filt):  # warm-up: modules, workspaces, visited-table scale
                    for _ in range(3):
                        fn(s)
                s.synchronize()
                tp, tf = [], []
                for _ in range(a.windows):
                    tp.append(window(torch, s, plain, a.calls))
                    tf.append(window(torch, s, filt, a.calls))
                fi, _, fc = filt(s)
                s.synchronize()
            g.stream_status()
            fi, fc = fi.cpu().numpy().view(np.uint32), fc.cpu().numpy()
            hits = [len(set(fi[i, :fc[i]].tolist()) & set(truth[i][truth[i] != 0xFFFFFFFF].tolist()))
                    for i in range(nq)]
            want = [min(k, int((truth[i] != 0xFFFFFFFF).sum())) for i in range(nq)]
            qps_p = [nq * a.calls / t for t in tp]
            qps_f = [nq * a.calls / t for t in tf]
            print(json.dumps({
                "max_search": ef, "admitted_share": share, "admitted": admitted, "nq": nq, "k": k,
                "search_qps": float(np.median(qps_p)), "search_qps_min": min(qps_p), "search_qps_max": max(qps_p),
                "filtered_qps": float(np.median(qps_f)), "filtered_qps_min": min(qps_f),
                "filtered_qps_max": max(qps_f), "filtered_over_search": float(np.median(qps_f) / np.median(qps_p)),
                "recall_at_10": float(sum(hits) / max(1, sum(want))), "recall_queries": nq,
                "recall_at_10_first_64": float(sum(hits[:64]) / max(1, sum(want[:64]))),
                "share_fewer_than_k": float((fc < k).mean()),
                "exact_qps": nq / float(np.median(ex_t)), "exact_qps_min": nq / max(ex_t),
                "exact_qps_max": nq / min(ex_t), "exact_path": "exact_search_filtered",
            }), flush=True)
        del dw
        torch.cuda.empty_cache()
    g.close()


if __name__ == "__main__":
    main()
