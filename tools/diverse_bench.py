"""Measures the diverse search (Granne.search_batch_diverse_device) against the plain search it starts from, and the
exact diverse path (exact_search_batch_device + select_neighbors_device), on one H100.

Data: filtered_bench.py's setup, bench.py's clustered 10M x 128 f32 rows (rerank_bench.generate) with a GPU-built index
(M = 30, max_search 200); 1024 raw queries in one device batch.  Per (max_search C in 200, 800; k in 10, 30):
  * QPS of search_batch_device(q, C, k) and search_batch_diverse_device(q, C, k), timed by CUDA events over --windows
    windows of --calls calls each, the two calls alternating window by window; median, min and max of the windows;
  * the time of stage 2 alone: select_neighbors_device over the stage-1 lists search_batch_device(q, C, C), which is
    the diverse call's second kernel (plus its list check), by CUDA events over the same windows;
  * pair distances per query: a float32 torch replay of the elimination on the first 64 queries (each kept
    candidate's distance to the later candidates still alive), next to the k * C bound;
  * the share of the 1024 queries that returned fewer than k;
  * the exact diverse path on the same queries, exact_search_batch_device(q, C) then select_neighbors_device(k): its
    QPS, and the recall of the graph version against it (|graph ∩ exact| / |exact| over the batch).
Prints the card name and power limit read in the same run, then one JSON line per (C, k).

    python tools/diverse_bench.py [--elements 10000000] [--windows 7] [--calls 5]
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
from filtered_bench import window  # noqa: E402
from rerank_bench import generate  # noqa: E402


def pair_distances(torch, rows, ids, dists, counts, k, nq):
    """Pair distances the elimination computes for the first nq lists: every round keeps the first alive candidate
    and computes its distance to each later alive one, which dies when it is closer to the kept one than to the query
    (float32 torch arithmetic: a tie may go the other way than on the device)."""
    out = []
    for q in range(nq):
        c = int(counts[q])
        if c <= k:
            out.append(0)
            continue
        cid = torch.from_numpy(ids[q, :c].astype(np.int64)).to(rows.device)
        cd = torch.from_numpy(dists[q, :c]).to(rows.device)
        x = rows[cid]
        alive = torch.ones(c, dtype=torch.bool, device=rows.device)
        kept, pairs = 0, 0
        while kept < k:
            idx = torch.nonzero(alive).flatten()
            if idx.numel() == 0:
                break
            s = int(idx[0])
            kept += 1
            alive[s] = False
            later = idx[1:]
            if kept == k or later.numel() == 0:
                break
            pairs += int(later.numel())
            ds = torch.clamp(1.0 - x[later] @ x[s], min=0.0)
            alive[later] = cd[later] <= ds
        out.append(pairs)
    return out


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
    n, dim, nq = a.elements, 128, 1024
    rows, q = generate(torch, granne_b200, n, dim, 1234, ("angular",), nq)
    t0 = time.perf_counter()
    b = granne_b200.GranneBuilder.from_device_elements("angular", rows["angular"], num_neighbors=30, max_search=200)
    b.build()
    index = b.index_bytes().tobytes()
    b.close()
    torch.cuda.empty_cache()
    print(json.dumps({"n": n, "dim": dim, "build_s": time.perf_counter() - t0}), flush=True)
    g = granne_b200.Granne.from_device_elements(index, "angular", rows["angular"])
    s = torch.cuda.Stream()
    for C in (200, 800):
        with torch.cuda.stream(s):
            li, ld, lc = g.search_batch_device(q, C, C, stream=s)
            ei, ed, ec = g.exact_search_batch_device(q, C, stream=s)
            s.synchronize()
        g.stream_status()
        for k in (10, 30):
            with torch.cuda.stream(s):
                def plain(st):
                    return g.search_batch_device(q, C, k, stream=st)

                def diverse(st):
                    return g.search_batch_diverse_device(q, C, k, stream=st)

                def stage2(st):
                    return g.select_neighbors_device(li, ld, lc, k, stream=st)

                def exact_div(st):
                    i, d, c = g.exact_search_batch_device(q, C, stream=st)
                    return g.select_neighbors_device(i, d, c, k, stream=st)

                for fn in (plain, diverse, stage2, exact_div):  # warm-up: modules, workspaces, visited-table scale
                    for _ in range(3):
                        fn(s)
                s.synchronize()
                tp, td, t2 = [], [], []
                for _ in range(a.windows):
                    tp.append(window(torch, s, plain, a.calls))
                    td.append(window(torch, s, diverse, a.calls))
                    t2.append(window(torch, s, stage2, a.calls))
                te = [window(torch, s, exact_div, 1) for _ in range(3)]
                di, dd, dc = diverse(s)
                xi, xd, xc = g.select_neighbors_device(ei, ed, ec, k, stream=s)
                s.synchronize()
            g.stream_status()
            di, dc = di.cpu().numpy().view(np.uint32), dc.cpu().numpy()
            xi, xc = xi.cpu().numpy().view(np.uint32), xc.cpu().numpy()
            hits = sum(len(set(di[i, :dc[i]].tolist()) & set(xi[i, :xc[i]].tolist())) for i in range(nq))
            pairs = pair_distances(torch, rows["angular"], li.cpu().numpy().view(np.uint32), ld.cpu().numpy(),
                                   lc.cpu().numpy(), k, 64)
            qps_p = [nq * a.calls / t for t in tp]
            qps_d = [nq * a.calls / t for t in td]
            print(json.dumps({
                "max_search": C, "k": k, "nq": nq,
                "search_qps": float(np.median(qps_p)), "search_qps_min": min(qps_p), "search_qps_max": max(qps_p),
                "diverse_qps": float(np.median(qps_d)), "diverse_qps_min": min(qps_d),
                "diverse_qps_max": max(qps_d), "diverse_over_search": float(np.median(qps_d) / np.median(qps_p)),
                "stage2_ms_per_call": float(np.median(t2)) * 1e3 / a.calls,
                "stage2_ms_min": min(t2) * 1e3 / a.calls, "stage2_ms_max": max(t2) * 1e3 / a.calls,
                "pair_distances_per_query_first_64": float(np.mean(pairs)), "pair_distances_max": max(pairs),
                "pair_distance_bound_k_times_C": k * C,
                "share_fewer_than_k": float((dc < k).mean()), "mean_count": float(dc.mean()),
                "exact_diverse_qps": nq / float(np.median(te)), "exact_diverse_qps_min": nq / max(te),
                "exact_diverse_qps_max": nq / min(te),
                "recall_vs_exact_diverse": float(hits / max(1, int(xc.sum()))),
            }), flush=True)
    g.close()


if __name__ == "__main__":
    main()
