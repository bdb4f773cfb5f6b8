"""Measures the two-stage search (Granne.search_batch_rerank_device) against plain f32 and i8 search on one graph.

Clustered vectors are generated on the GPU from fixed seeds with bench.py's generator.  One index is built with the
GPU builder over the f32 rows; the index file does not depend on the element type, so it is opened twice: over the
angular rows, and over the angular_int rows with the angular rows attached for the re-rank.  Every arm is device
resident, 1024-query batches, max_search 200, k = 10:
    f32       search_batch_device on the angular handle
    i8        search_batch_device on the angular_int handle
    rerank_C  search_batch_rerank_device with C candidates, for each C in --candidates
Per arm: QPS as the median (and min, max) of --rounds windows of --iters batches (about a second each at the default),
each timed with CUDA events after --warmup batches, the arms of one handle alternating window by window; recall@10
against exact_search_batch on the f32
handle, the algorithmic bytes gathered per query (n_dist x row stride of the traversed rows, plus C x the f32 row
stride for the re-rank) and, for the re-rank arms, the stage-2 kernel time from torch.profiler in a separate pass.
Prints the card name and power limit and one JSON line per arm.

    python tools/rerank_bench.py [--elements 10000000] [--candidates 10,50,100,200]
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exact_bench import card  # noqa: E402


def generate(torch, granne_b200, n, dim, seed, kinds, nq=0):
    """Element rows of each kind in `kinds` (CUDA tensors), chunk by chunk from bench.py's seeded mixture; with nq,
    raw queries from the next seed."""
    from bench import CHUNK, device_tables, raw_chunk_device

    dev = torch.device("cuda", 0)
    a = types.SimpleNamespace(dist="clustered", dim=dim)
    tables = device_tables(torch, dev, a, n)
    out = {k: torch.empty((n, dim), dtype=torch.int8 if k == "angular_int" else torch.float32, device=dev)
           for k in kinds}
    for ci, s in enumerate(range(0, n, CHUNK)):
        m = min(CHUNK, n - s)
        raw = raw_chunk_device(torch, dev, a, tables, seed, ci, m)
        for k, t in out.items():
            granne_b200.elements_from_raw_device(k, raw, out=t[s:s + m])
    q = raw_chunk_device(torch, dev, a, tables, seed + 1, 0, nq) if nq else None
    torch.cuda.synchronize()
    return out, q


def timed(torch, fn, warmup, iters):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn(s)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(iters):
            out = fn(s)
        e1.record(s)
    s.synchronize()
    return e0.elapsed_time(e1) / 1e3 / iters, out


def kernel_seconds(torch, fn, name, reps=5):
    """Mean device time per call of the kernels whose name contains `name` (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile

    s = torch.cuda.Stream()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(s):
            for _ in range(reps):
                fn(s)
        s.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if name in e.key:
            total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return total / 1e6 / reps


def recall(ids, truth):
    ids = ids.cpu().numpy().view(np.uint32)
    return float(np.mean([len(set(ids[i].tolist()) & set(truth[i].tolist())) / truth.shape[1]
                          for i in range(truth.shape[0])]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--num-neighbors", type=int, default=30)
    ap.add_argument("--max-search", type=int, default=200)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--candidates", default="10,50,100,200")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--iters", type=int, default=1500, help="batches per timed window (about a second each)")
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per arm, the arms alternating")
    a = ap.parse_args()
    import torch

    import granne_b200
    from granne_b200 import api

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    n, dim, ms, k = a.elements, a.dim, a.max_search, 10
    rows, q = generate(torch, granne_b200, n, dim, 1234, ("angular", "angular_int"), a.nq)
    t0 = time.perf_counter()
    b = granne_b200.GranneBuilder.from_device_elements("angular", rows["angular"], num_neighbors=a.num_neighbors,
                                                       max_search=200)
    b.build()
    index = b.index_bytes().tobytes()
    b.close()
    torch.cuda.empty_cache()
    print(json.dumps({"n": n, "dim": dim, "num_neighbors": a.num_neighbors,
                      "build_s": time.perf_counter() - t0}), flush=True)
    f32_stride = ((dim + 3) // 4 * 4) * 4
    i8_stride = (dim + 31) // 32 * 32
    stats = torch.zeros((a.nq, api.STATS_PER_QUERY), dtype=torch.int64, device="cuda")

    def run_arms(handle, arms):
        """arms: name -> (fn, traversed row stride, extra bytes per query, extra fields).  --rounds windows per arm,
        the arms of one handle alternating window by window; one JSON line per arm."""
        qps = {arm: [] for arm in arms}
        outs = {}
        for _ in range(a.rounds):
            for arm, (fn, _, _, _) in arms.items():
                sec, outs[arm] = timed(torch, fn, a.warmup, a.iters)
                qps[arm].append(a.nq / sec)
        handle.stream_status()
        for arm, (fn, stride, extra_bytes, kw) in arms.items():
            fn(torch.cuda.current_stream(), stats)
            torch.cuda.synchronize()
            n_dist = float(stats[:, 0].double().mean())
            res = {"arm": arm, "n": n, "dim": dim, "nq": a.nq, "max_search": ms, "k": k,
                   "window_queries": a.nq * a.iters, "qps": float(np.median(qps[arm])), "qps_min": min(qps[arm]),
                   "qps_max": max(qps[arm]), "qps_windows": qps[arm], "recall_at_10": recall(outs[arm][0], truth),
                   "stage1_n_dist": n_dist, "bytes_per_query": n_dist * stride + extra_bytes}
            res.update(kw)
            print(json.dumps(res), flush=True)

    # The f32 and angular_int handles are timed one after the other: at 50M the f32 handle, the source rows and the
    # attached re-rank rows (three f32 copies) do not fit in 80 GB together.
    f = granne_b200.Granne.from_device_elements(index, "angular", rows["angular"])
    truth = f.exact_search_batch(q.cpu().numpy(), k)[0]
    run_arms(f, {"f32": (lambda s, st=None: f.search_batch_device(q, ms, k, stats=st, stream=s.cuda_stream),
                         f32_stride, 0, {})})
    f.close()
    torch.cuda.empty_cache()

    g = granne_b200.Granne.from_device_elements(index, "angular_int", rows["angular_int"])
    g.set_rerank_elements_device(rows["angular"])
    rows = None
    torch.cuda.empty_cache()
    arms = {"i8": (lambda s, st=None: g.search_batch_device(q, ms, k, stats=st, stream=s.cuda_stream), i8_stride, 0,
                   {})}
    for c in [int(x) for x in a.candidates.split(",")]:
        def fn(s, st=None, c=c):
            return g.search_batch_rerank_device(q, c, max_search=ms, num_elements=k, stats=st, stream=s.cuda_stream)

        try:
            stage2 = kernel_seconds(torch, fn, "rerank_kernel")
        except Exception as e:  # the profiler is optional: the QPS and recall stand without it
            stage2 = "not measured (%s)" % type(e).__name__
        arms["rerank_%d" % c] = (fn, i8_stride, c * f32_stride, {"candidates": c, "stage2_kernel_s": stage2})
    run_arms(g, arms)
    g.close()


if __name__ == "__main__":
    main()
