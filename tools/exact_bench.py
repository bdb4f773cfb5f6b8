"""Measures the exact k-NN scan (Granne.exact_search_batch*) and the ground truth it replaces.

For each workload (1024 queries, k = 10): kernel time of the device call (CUDA events, median of --reps), pairs/s and
the share of the data-sheet peak that bounds it (FP32: 67 TFLOP/s counting 2*dim + 31 flops per pair; the i8 scan is
reported against the same CUDA-core issue rate in int ops, 2*dim per pair), the end-to-end host call, the CPU oracle's
brute force on 16 threads over a query subset, and the torch FP32 matmul + topk ground truth: its time and the
fraction of queries whose top-10 differs from the exact answer.  Prints one JSON line per workload and the card name
and power limit read in the same run.

    python tools/exact_bench.py [--workloads f32_1m,i8_10m,f32_50m] [--reps 5]
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

PEAK_FP32 = 67e12  # H100 SXM data sheet, FP32 (non-tensor) FLOP/s


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def make(kind, n, dim, seed):
    """(handle, host rows or None) for n random elements; rows are made on the device, one slab at a time."""
    import torch
    import granne_b200
    from oracle import granne_oracle as go
    from helpers import composed_oracle as co

    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.float32 if kind == "angular" else torch.int8
    rows = torch.empty((n, dim), dtype=dt, device="cuda")
    for r0 in range(0, n, 1 << 22):
        r1 = min(n, r0 + (1 << 22))
        x = torch.rand((r1 - r0, dim), generator=g, device="cuda") - 0.5
        if kind == "angular":
            rows[r0:r1] = x / x.norm(dim=1, keepdim=True)
        else:
            rows[r0:r1] = (x * 255).to(torch.int8)
    h = granne_b200.Granne.from_device_elements(co.single_layer_index(go, n), kind, rows)
    return h, rows


def run(name, kind, n, dim, reps, oracle_q, nq=1024, k=10):
    import torch
    from helpers import composed_oracle as co

    h, rows = make(kind, n, dim, 1)
    q = (torch.rand((nq, dim), generator=torch.Generator(device="cuda").manual_seed(2), device="cuda") - 0.5)
    s = torch.cuda.Stream()
    out = None
    times = []
    for _ in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s):
            e0.record(s)
            out = h.exact_search_batch_device(q, k, stream=s.cuda_stream)
            e1.record(s)
        s.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    h.stream_status()
    kt = float(np.median(times[1:]))
    pairs = n * nq
    ops = 2 * dim + 31 if kind == "angular" else 2 * dim
    qh = q.cpu().numpy()
    t0 = time.perf_counter()
    ids, dists, _ = h.exact_search_batch(qh, k)
    host_s = time.perf_counter() - t0
    res = {"workload": name, "n": n, "dim": dim, "nq": nq, "k": k, "kernel_s": kt, "pairs_per_s": pairs / kt,
           "ops_per_pair": ops, "tops": pairs * ops / kt / 1e12, "share_fp32_peak": pairs * ops / kt / PEAK_FP32,
           "host_call_s": host_s}
    assert np.array_equal(ids.view(np.int32), out[0].cpu().numpy())
    if kind == "angular":
        # the ground truth the bench and tools compute today: FP32 matmul (no TF32) + topk
        torch.backends.cuda.matmul.allow_tf32 = False
        qn = q / q.norm(dim=1, keepdim=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        top = torch.cat([torch.topk(qn[i:i + 64] @ rows.T, k, dim=1).indices for i in range(0, nq, 64)])
        torch.cuda.synchronize()
        res["torch_topk_s"] = time.perf_counter() - t0
        res["torch_top10_differs"] = float((top.cpu().numpy() != ids.astype(np.int64)).any(axis=1).mean())
    if oracle_q and n <= 10_000_000:
        host = rows.cpu().numpy()
        c = co.Container(kind, np.uint64(dim).tobytes() + host.tobytes())
        t0 = time.perf_counter()
        wi, wd, _ = c.exact_search(qh[:oracle_q] if kind == "angular" else qh[:oracle_q], k, threads=16)
        res["oracle_16t_s"] = time.perf_counter() - t0
        res["oracle_queries"] = oracle_q
        res["oracle_equal"] = bool(np.array_equal(wi, ids[:oracle_q]) and
                                   np.array_equal(wd.view(np.uint32), dists[:oracle_q].view(np.uint32)))
    del h, rows
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="f32_1m,i8_10m,f32_50m")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-queries", type=int, default=16)
    a = ap.parse_args()
    import granne_b200

    granne_b200.load_library()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl}), flush=True)
    w = {"f32_1m": ("angular", 1_000_000, 128), "i8_10m": ("angular_int", 10_000_000, 100),
         "f32_50m": ("angular", 50_000_000, 128)}
    for key in a.workloads.split(","):
        kind, n, dim = w[key]
        print(json.dumps(run(key, kind, n, dim, a.reps, a.oracle_queries)), flush=True)


if __name__ == "__main__":
    main()
