"""Measures the exact filtered k-NN scan (Granne.exact_search_filtered_device) against the unfiltered exact scan and
exact search within one shared list of the admitted ids.

Data: tools/exact_bench.py's random elements (1M x 128 f32, 10M x 100 i8) and 10M x 128 f32, the size of DESIGN's
filtered-search table.  1024 queries, k = 10.  Filters: one filter admitting 0.1, 1, 10, 50 and 100 % of n, and 16
per-query filters of 1 % each (query q uses filter q % 16, so every query chunk names all 16).  Per (workload, filter):
  * exact_search_filtered_device;
  * exact_search_batch_device (the same for every filter: the full scan);
  * exact_search_within_device with a CSR in which every query lists its filter's admitted ids, and the CSR's size in
    bytes; only up to 10 %, since it ranks every query's list on its own.
Each is timed by CUDA events over --windows windows of one call, the calls alternating window by window, after one
warm-up call each; median, min and max.  The filtered result is checked against the within-list result (at 100 %:
against exact_search_batch; at 50 %: not checked here).  Prints the
card name and power limit read in the same run, then one JSON line per (workload, filter).

    python tools/exact_filtered_bench.py [--workloads f32_1m,i8_10m,f32_10m] [--windows 5]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from exact_bench import card, make  # noqa: E402
from filtered_bench import window  # noqa: E402


def stats(ts):
    return {"median_ms": float(np.median(ts)) * 1e3, "min_ms": min(ts) * 1e3, "max_ms": max(ts) * 1e3}


def run(name, kind, n, dim, windows, nq=1024, k=10):
    import torch

    import granne_b200

    dev = torch.device("cuda", 0)
    h, rows = make(kind, n, dim, 1)
    del rows
    torch.cuda.empty_cache()
    q = (torch.rand((nq, dim), generator=torch.Generator(device="cuda").manual_seed(2), device="cuda") - 0.5)
    s = torch.cuda.Stream()
    rng = np.random.default_rng(3)
    cases = [("%g%%" % (share * 100), [share], None) for share in (0.001, 0.01, 0.1, 0.5, 1.0)]
    cases.append(("16x1%", [0.01] * 16, np.arange(nq, dtype=np.int32) % 16))
    for label, shares, qf in cases:
        masks = np.stack([np.ones(n, bool) if sh == 1.0 else rng.random(n) < sh for sh in shares])
        words = granne_b200.api._filter_words(masks, n)
        dw = torch.from_numpy(words.view(np.int32)).to(dev)
        dqf = torch.from_numpy(qf).to(dev) if qf is not None else None
        lists = [np.nonzero(m)[0].astype(np.uint32) for m in masks]
        # the within call's CSR: every query lists its filter's admitted ids (made on the device)
        per = [lists[0]] * nq if qf is None else [lists[f] for f in qf]
        offsets = np.zeros(nq + 1, np.int64)
        np.cumsum([x.size for x in per], out=offsets[1:])
        d_off = torch.from_numpy(offsets).to(dev)
        if qf is None:
            d_ids = torch.from_numpy(lists[0].view(np.int32)).to(dev).repeat(nq)
        else:
            d_ids = torch.from_numpy(np.concatenate(per).view(np.int32)).to(dev)
        with torch.cuda.stream(s):
            def filt(st):
                return h.exact_search_filtered_device(q, dw, dqf, k, stream=st)

            def full(st):
                return h.exact_search_batch_device(q, k, stream=st)

            def within(st):
                return h.exact_search_within_device(q, d_off, d_ids, k, stream=st)

            # a list of half or all of n per query ranks 1024 x |A| pairs one query at a time: not timed
            fns = (filt, full, within) if max(shares) <= 0.1 else (filt, full)
            for fn in fns:
                fn(s)
            s.synchronize()
            t = {fn.__name__: [] for fn in fns}
            for _ in range(windows):
                for fn in fns:
                    t[fn.__name__].append(window(torch, s, fn, 1))
            got, want = filt(s), (within(s) if within in fns else full(s))
            s.synchronize()
        h.stream_status()
        equal = all(torch.equal(a, b) for a, b in zip(got, want)) if within in fns or shares == [1.0] else None
        print(json.dumps({"workload": name, "n": n, "dim": dim, "nq": nq, "k": k, "filter": label,
                          "admitted_per_filter": [int(x.size) for x in lists],
                          "exact_search_filtered": stats(t["filt"]), "exact_search_batch": stats(t["full"]),
                          "exact_search_within": stats(t["within"]) if "within" in t else None,
                          "within_list_bytes": int(offsets[-1]) * 4, "filtered_equals_exact": equal}), flush=True)
        del dw, dqf, d_off, d_ids
        torch.cuda.empty_cache()
    h.close()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="f32_1m,i8_10m,f32_10m")
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    import granne_b200

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    w = {"f32_1m": ("angular", 1_000_000, 128), "i8_10m": ("angular_int", 10_000_000, 100),
         "f32_10m": ("angular", 10_000_000, 128)}
    for key in a.workloads.split(","):
        kind, n, dim = w[key]
        run(key, kind, n, dim, a.windows)


if __name__ == "__main__":
    main()
