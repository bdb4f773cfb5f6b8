"""Measures exact search within candidate lists (Granne.exact_search_within_device) on one H100.

Workloads (k = 10), each a device-resident call on CUDA tensors:
    f32 container   bench.py's clustered 10M x 128 rows, with a GPU-built index
      rerank_100 / hybrid_1000   1024 queries x 100 random ids, and 1024 x 1000
      long_1m                    16 queries x 1M random ids (one long list each: ~1000 segments per query)
      admitted_<p>               1024 queries sharing one random admitted set of p of n, next to exact_search_batch on
                                 the same queries: where the two cross over
      vs_rerank_<C>              the lists stage 1 of the two-stage search produces (C = 100, 1000 per query), ranked
                                 by this call on the f32 handle
    i8 container    10M x 100 angular_int rows: hybrid_1000
    emb container   bench.py's `emb` SumEmbeddings container at 1M elements: hybrid_1000
    --rerank-profile, a run of its own: the kernel times of within_kernel and of rerank_kernel on those same lists and
    rows, from torch.profiler (CUDA activity), --profile-rounds rounds of 5 calls per kernel, the two alternating round
    by round; median, min and max of the rounds' means.  Nothing else runs in that process.
Per workload: the device time of the call from CUDA events (median of --reps after --warmup calls, with min and max),
candidates per second, and the algorithmic bytes (sum |L_q| x row bytes + 4 bytes per id) over that time as a share
of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth.  Prints the card name and power limit read in the same run,
then one JSON line per workload.

    python tools/within_bench.py [--elements 10000000] [--reps 7] [--skip i8,emb]
    python tools/within_bench.py --rerank-profile [--profile-rounds 7]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from exact_bench import card  # noqa: E402
from rerank_bench import generate, kernel_seconds  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, HBM3 bytes/s


def event_times(torch, fn, warmup, reps):
    """Device seconds of fn(stream) per call: CUDA events around each of `reps` calls after `warmup`."""
    s = torch.cuda.Stream()
    out = None
    times = []
    with torch.cuda.stream(s):
        for _ in range(warmup):
            out = fn(s)
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            out = fn(s)
            e1.record(s)
            s.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
    return times, out


def device_lists(torch, lists_np, dev):
    offsets = np.zeros(len(lists_np) + 1, np.int64)
    np.cumsum([len(x) for x in lists_np], out=offsets[1:])
    ids = np.concatenate(lists_np).astype(np.uint32)
    return torch.from_numpy(offsets).to(dev), torch.from_numpy(ids.view(np.int32)).to(dev)


def report(name, times, total_ids, row_bytes, **kw):
    t = float(np.median(times))
    algo = total_ids * (row_bytes + 4)
    res = {"workload": name, "call_s": t, "call_s_min": min(times), "call_s_max": max(times), "reps": len(times),
           "candidates": int(total_ids), "candidates_per_s": total_ids / t, "algorithmic_bytes": int(algo),
           "algorithmic_bytes_per_s": algo / t, "share_of_hbm_datasheet_peak": algo / t / HBM_PEAK}
    res.update(kw)
    print(json.dumps(res), flush=True)


def stage1_lists(torch, g, q, dev):
    """(C, device lists) for C = 100, 1000: the candidate lists stage 1 of the two-stage search gives rerank_kernel,
    search_batch(q, max(200, C), C) on the angular_int handle g."""
    out = []
    for c in (100, 1000):
        si, _, sc = g.search_batch(q.cpu().numpy(), max(200, c), c)
        out.append((c, device_lists(torch, [si[i, :sc[i]] for i in range(len(si))], dev)))
    return out


def rerank_profile(torch, granne_b200, a, f, index, rows, q, dev, k):
    """Kernel times of within_kernel (on the angular handle f) and rerank_kernel (two-stage search on an angular_int
    handle with f's rows attached) on the same lists: --profile-rounds rounds, alternating, one JSON line per C."""
    g = granne_b200.Granne.from_device_elements(index, "angular_int", rows["angular_int"])
    g.set_rerank_elements_device(rows["angular"])
    for c, (offsets, ids) in stage1_lists(torch, g, q, dev):
        def wf(s, o=offsets, i=ids):
            return f.exact_search_within_device(q, o, i, k, stream=s)

        def rf(s, c=c):
            return g.search_batch_rerank_device(q, c, max_search=max(200, c), num_elements=k, stream=s)

        for fn in (wf, rf):  # warm-up outside the profiled rounds
            event_times(torch, fn, 3, 1)
        w, r = [], []
        for _ in range(a.profile_rounds):
            w.append(kernel_seconds(torch, wf, "within_kernel"))
            r.append(kernel_seconds(torch, rf, "rerank_kernel"))
        f.stream_status()
        g.stream_status()
        print(json.dumps({"workload": "kernel_within_vs_rerank_%d" % c, "nq": len(q), "k": k,
                          "candidates": int(offsets[-1]), "rounds": a.profile_rounds, "calls_per_round": 5,
                          "within_kernel_s": float(np.median(w)), "within_kernel_s_min": min(w),
                          "within_kernel_s_max": max(w), "rerank_kernel_s": float(np.median(r)),
                          "rerank_kernel_s_min": min(r), "rerank_kernel_s_max": max(r),
                          "within_over_rerank": float(np.median(w)) / float(np.median(r))}), flush=True)
    g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=10_000_000)
    ap.add_argument("--emb-elements", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip", default="", help="comma list of containers to skip: f32, i8, emb")
    ap.add_argument("--rerank-profile", action="store_true",
                    help="only the profiler comparison of within_kernel and rerank_kernel on identical lists")
    ap.add_argument("--profile-rounds", type=int, default=7)
    a = ap.parse_args()
    skip = set(x for x in a.skip.split(",") if x)
    import torch

    import granne_b200

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    dev = torch.device("cuda", 0)
    n, k, nq = a.elements, 10, 1024
    rng = np.random.default_rng(5)

    def run(handle, name, q, lists_np, row_bytes, **kw):
        offsets, ids = device_lists(torch, lists_np, dev)
        times, _ = event_times(torch, lambda s: handle.exact_search_within_device(q, offsets, ids, k, stream=s),
                               a.warmup, a.reps)
        handle.stream_status()
        report(name, times, int(offsets[-1]), row_bytes, nq=len(lists_np), k=k, **kw)

    if "f32" not in skip:
        dim = 128
        rows, q = generate(torch, granne_b200, n, dim, 1234, ("angular", "angular_int"), nq)
        t0 = time.perf_counter()
        b = granne_b200.GranneBuilder.from_device_elements("angular", rows["angular"], num_neighbors=30,
                                                           max_search=200)
        b.build()
        index = b.index_bytes().tobytes()
        b.close()
        torch.cuda.empty_cache()
        print(json.dumps({"container": "f32", "n": n, "dim": dim, "build_s": time.perf_counter() - t0}), flush=True)
        f = granne_b200.Granne.from_device_elements(index, "angular", rows["angular"])
        rb = dim * 4
        if a.rerank_profile:
            rerank_profile(torch, granne_b200, a, f, index, rows, q, dev, k)
            return
        run(f, "f32_rerank_100", q, [rng.integers(0, n, 100) for _ in range(nq)], rb)
        run(f, "f32_hybrid_1000", q, [rng.integers(0, n, 1000) for _ in range(nq)], rb)
        run(f, "f32_long_1m", q[:16], [rng.integers(0, n, 1_000_000) for _ in range(16)], rb)
        ex_times, _ = event_times(torch, lambda s: f.exact_search_batch_device(q, k, stream=s), 1, 5)
        for p in (0.0001, 0.001, 0.01, 0.1):
            admitted = rng.choice(n, int(n * p), replace=False)
            run(f, "f32_admitted_%g" % p, q, [admitted] * nq, rb, admitted_share=p,
                exact_search_batch_s=float(np.median(ex_times)), exact_search_batch_s_min=min(ex_times),
                exact_search_batch_s_max=max(ex_times))
        g = granne_b200.Granne.from_device_elements(index, "angular_int", rows["angular_int"])
        for c, (offsets, ids) in stage1_lists(torch, g, q, dev):
            times, _ = event_times(torch, lambda s: f.exact_search_within_device(q, offsets, ids, k, stream=s),
                                   a.warmup, a.reps)
            f.stream_status()
            report("f32_vs_rerank_%d" % c, times, int(offsets[-1]), rb, nq=nq, k=k)
        g.close()
        f.close()
        rows = None
        torch.cuda.empty_cache()

    if "i8" not in skip:
        from oracle import granne_oracle as go
        from helpers import composed_oracle as co

        dim = 100
        rows, q = generate(torch, granne_b200, n, dim, 4321, ("angular_int",), nq)
        h = granne_b200.Granne.from_device_elements(co.single_layer_index(go, n), "angular_int", rows["angular_int"])
        run(h, "i8_hybrid_1000", q, [rng.integers(0, n, 1000) for _ in range(nq)], (dim + 15) // 16 * 16)
        h.close()
        rows = None
        torch.cuda.empty_cache()

    if "emb" not in skip:
        from bench import DATA_SEED, QUERY_SEED, SumContainer
        from oracle import granne_oracle as go
        from helpers import composed_oracle as co

        ne, dim = a.emb_elements, 100
        cont = SumContainer(torch, granne_b200, dev, types.SimpleNamespace(dim=dim, num_neighbors=30), ne, DATA_SEED)
        e = granne_b200.Granne.from_bytes(co.single_layer_index(go, ne), "embeddings",
                                          cont.elements_image.tobytes(), cont.embeddings_image.tobytes())
        q = torch.from_numpy(np.ascontiguousarray(cont.queries(nq, QUERY_SEED), dtype=np.float32)).to(dev)
        # row bytes: the element's terms (mean terms_per_element table rows of dim f32) and its 5-byte offset
        rb = cont.terms_per_element * dim * 4 + 5
        run(e, "emb_hybrid_1000", q, [rng.integers(0, ne, 1000) for _ in range(nq)], rb, n=ne)
        e.close()


if __name__ == "__main__":
    main()
