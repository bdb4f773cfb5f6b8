"""Measures the two-stage search re-ranked by a SumEmbeddings container against the other ways to search the same
embeddings data.

The data is bench.py's `emb` distribution (a SumEmbeddings container: elements of 2..9 terms over n/5 embeddings of
width 100), generated from fixed seeds.  As granne's own pipeline does, compute_embeddings turns the container into
angular_int rows and the GPU builder builds one index over them.  The index file does not depend on the element type,
so it is opened several times.  Every arm is device resident, 1024-query batches, max_search 200, k = 10:
    emb        search_batch_device on the "embeddings" handle (DistSum search)
    i8         search_batch_device on the angular_int handle
    f32_C      search_batch_rerank_device with C candidates, compute_embeddings("angular") rows attached
    sum_C      search_batch_rerank_device with C candidates, the SumEmbeddings container attached
Per arm: QPS as the median (and min, max) of --rounds windows of --iters batches, each timed with CUDA events after
--warmup batches, the arms of one handle alternating window by window; recall@10 against exact_search_batch on the
"embeddings" handle; the handle's device_bytes including the attached container; and, for the re-rank arms, the
stage-2 kernel time from torch.profiler in a separate pass.  Prints the card name and power limit and one JSON line
per arm.

    python tools/sum_rerank_bench.py [--elements 1000000] [--candidates 10,50,100,200]
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
from rerank_bench import kernel_seconds, recall, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=100)
    ap.add_argument("--num-neighbors", type=int, default=30)
    ap.add_argument("--max-search", type=int, default=200)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--candidates", default="10,50,100,200")
    ap.add_argument("--f32-candidates", default="50")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--iters", type=int, default=1000, help="batches per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per arm, the arms alternating")
    a = ap.parse_args()
    import torch

    import granne_b200
    from bench import DATA_SEED, QUERY_SEED, SumContainer

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    n, dim, ms, k = a.elements, a.dim, a.max_search, 10
    dev = torch.device("cuda", 0)
    cont = SumContainer(torch, granne_b200, dev, types.SimpleNamespace(dim=dim, num_neighbors=a.num_neighbors), n,
                        DATA_SEED)
    ei, ti = cont.elements_image.tobytes(), cont.embeddings_image.tobytes()
    q_host = np.ascontiguousarray(cont.queries(a.nq, QUERY_SEED), dtype=np.float32)
    q = torch.from_numpy(q_host).to(dev)

    t0 = time.perf_counter()
    i8_rows = granne_b200.compute_embeddings_device("angular_int", ei, ti, device=0)
    torch.cuda.synchronize()
    b = granne_b200.GranneBuilder.from_device_elements("angular_int", i8_rows, num_neighbors=a.num_neighbors,
                                                       max_search=200)
    b.build()
    index = b.index_bytes().tobytes()
    b.close()
    torch.cuda.empty_cache()
    print(json.dumps({"n": n, "dim": dim, "num_neighbors": a.num_neighbors,
                      "terms_per_element": cont.terms_per_element, "table_rows": int(cont.emb.shape[0]),
                      "build_s": time.perf_counter() - t0}), flush=True)

    e = granne_b200.Granne.from_bytes(index, "embeddings", ei, ti)
    truth = e.exact_search_batch(q_host, k)[0]

    def run_arms(handle, arms):
        """arms: name -> (fn, extra fields).  --rounds windows per arm, the arms of one handle alternating window by
        window; one JSON line per arm."""
        qps = {arm: [] for arm in arms}
        outs = {}
        for _ in range(a.rounds):
            for arm, (fn, _) in arms.items():
                sec, outs[arm] = timed(torch, fn, a.warmup, a.iters)
                qps[arm].append(a.nq / sec)
        handle.stream_status()
        for arm, (fn, kw) in arms.items():
            res = {"arm": arm, "n": n, "dim": dim, "nq": a.nq, "max_search": ms, "k": k,
                   "window_queries": a.nq * a.iters, "qps": float(np.median(qps[arm])), "qps_min": min(qps[arm]),
                   "qps_max": max(qps[arm]), "qps_windows": qps[arm], "recall_at_10": recall(outs[arm][0], truth),
                   "device_bytes": handle.device_bytes()}
            res.update(kw)
            print(json.dumps(res), flush=True)

    def stage2(fn):
        try:
            return kernel_seconds(torch, fn, "rerank_kernel")
        except Exception as ex:  # the profiler is optional: the QPS and recall stand without it
            return "not measured (%s)" % type(ex).__name__

    run_arms(e, {"emb": (lambda s: e.search_batch_device(q, ms, k, stream=s.cuda_stream), {})})
    e.close()
    torch.cuda.empty_cache()

    # the f32 re-rank: the normalised sums materialised as angular rows
    f = granne_b200.Granne.from_device_elements(index, "angular_int", i8_rows)
    f32_rows = granne_b200.compute_embeddings_device("angular", ei, ti, device=0)
    f.set_rerank_elements_device(f32_rows)
    f32_rows = None
    torch.cuda.empty_cache()
    arms = {}
    for c in [int(x) for x in a.f32_candidates.split(",") if x]:
        def fn(s, c=c):
            return f.search_batch_rerank_device(q, c, max_search=ms, num_elements=k, stream=s.cuda_stream)

        arms["f32_%d" % c] = (fn, {"candidates": c, "stage2_kernel_s": stage2(fn)})
    run_arms(f, arms)
    f.close()
    torch.cuda.empty_cache()

    g = granne_b200.Granne.from_device_elements(index, "angular_int", i8_rows)
    i8_bytes = g.device_bytes()
    g.set_rerank_embeddings(ei, ti)
    i8_rows = None
    torch.cuda.empty_cache()
    arms = {"i8": (lambda s: g.search_batch_device(q, ms, k, stream=s.cuda_stream), {"device_bytes_i8": i8_bytes})}
    for c in [int(x) for x in a.candidates.split(",")]:
        def fn(s, c=c):
            return g.search_batch_rerank_device(q, c, max_search=ms, num_elements=k, stream=s.cuda_stream)

        arms["sum_%d" % c] = (fn, {"candidates": c, "stage2_kernel_s": stage2(fn)})
    run_arms(g, arms)
    g.close()


if __name__ == "__main__":
    main()
