"""Measures compute_embeddings (granne's compute_embeddings_and_save_to_disk, src/elements/embeddings/parsing.rs:102-152)
on one GPU and what the materialised rows buy at search time.  Prints one JSON line.

Data: bench.py's `emb` distribution (a clustered table of n/5 embeddings of width 100; element i holds 2 + i % 8 terms
drawn from one cluster), generated from a seed.

  materialisation (n = --n, 10M by default): the device variant (warmed up, --calls timed calls), the host variant end
  to end (image in host memory), and the CPU oracle on every host thread — a C++ restatement used as the tests'
  checker, not the reference's Rust binary.  Algorithmic bytes: the table rows read (terms x dim x 4), the term ids
  (4 bytes each on the device), the offsets (8 bytes each), the raw rows written and read back (2 x n x dim x 4) and
  the output rows; over the two kernels' time (torch.profiler, a run of its own), and as a fraction of the H100 SXM
  data-sheet HBM3 bandwidth of 3.35 TB/s.

  search (n = --search-n, 1M): one index built on the GPU over the SumEmbeddings container; batches of 1024 queries on
  --streams concurrent host threads (one stream each) against the SumEmbeddings container, the materialised angular
  rows (results asserted identical) and the materialised angular_int rows (recall@10 against exact neighbours).

    python tools/embeddings_bench.py [--n 10000000] [--search-n 1000000]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_DATASHEET = 3.35e12  # B/s, H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, power = (out[0].split(", ") + ["?"])[:2] if out else ("?", "?")
    return name, power


def container(torch, gb, dev, n, seed):
    import bench

    return bench.SumContainer(torch, gb, dev, SimpleNamespace(dim=100, num_neighbors=20), n, seed)


def materialise(torch, gb, c, calls):
    from helpers import composed_oracle as co

    el, emb = c.elements_image, c.embeddings_image
    n, dim, terms = c.n, 100, int(c.offsets[-1])
    res = {"n": n, "dim": dim, "terms": terms}
    for kind, esz in (("angular_int", 1), ("angular", 4)):
        out = torch.empty((n, dim), dtype=torch.int8 if esz == 1 else torch.float32, device="cuda")
        for _ in range(2):
            gb.compute_embeddings_device(kind, el, emb, out=out)
        times = []
        for _ in range(calls):
            t0 = time.perf_counter()
            gb.compute_embeddings_device(kind, el, emb, out=out)  # returns after a stream synchronise
            times.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                gb.compute_embeddings_device(kind, el, emb, out=out)
        kern = {}
        for e in prof.key_averages():
            for name in ("sum_embeddings_kernel", "make_elements_kernel"):
                if name in e.key:
                    kern[name] = kern.get(name, 0.0) + e.device_time_total / 3 / 1e6  # s per call
        del out
        torch.cuda.empty_cache()
        host_img = np.empty(8 + n * dim * esz, dtype=np.uint8)
        gb.compute_embeddings(kind, el, emb, out=host_img)
        t0 = time.perf_counter()
        gb.compute_embeddings(kind, el, emb, out=host_img)
        host_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        ref = co.compute_embeddings(kind, el.tobytes(), emb.tobytes(), threads=os.cpu_count())
        oracle_s = time.perf_counter() - t0
        assert np.array_equal(ref, host_img), kind + ": the host variant's image differs from the oracle's"
        del ref, host_img
        nbytes = terms * dim * 4 + terms * 4 + (n + 1) * 8 + 2 * n * dim * 4 + n * dim * esz
        kt = sum(kern.values())
        res[kind] = {
            "device_call_s": {"median": float(np.median(times)), "min": float(min(times)), "calls": calls},
            "kernel_s": kern,
            "kernel_s_total": kt,
            "fused_pass_share": kern.get("make_elements_kernel", 0.0) / kt if kt else None,
            "host_call_s": host_s,
            "oracle_port_all_threads_s": oracle_s,
            "oracle_threads": os.cpu_count(),
            "algorithmic_bytes": nbytes,
            "bytes_per_s_over_kernel_time": nbytes / kt if kt else None,
            "fraction_of_datasheet_3.35TBps": nbytes / kt / HBM_DATASHEET if kt else None,
        }
    return res


def qps(index, queries, max_search, k, streams, reps):
    batches = [queries[i:i + 1024] for i in range(0, len(queries), 1024)]
    index.search_batch(batches[0], max_search, k)

    def work(t):
        for _ in range(reps):
            for b in batches[t::streams]:
                index.search_batch(b, max_search, k)

    th = [threading.Thread(target=work, args=(t,)) for t in range(streams)]
    t0 = time.perf_counter()
    for t in th:
        t.start()
    for t in th:
        t.join()
    return reps * len(queries) / (time.perf_counter() - t0)


def search(torch, gb, c, streams, max_search):
    os.environ.pop("GRANNE_B200_BUILD_MAX_BATCH", None)
    t0 = time.perf_counter()
    b = c.builder()
    b.build()
    index = bytes(b.index_bytes())
    b.close()
    build_s = time.perf_counter() - t0
    el, emb = c.elements_image, c.embeddings_image
    q = c.queries(16384, seed=99)
    summed = gb.Granne.from_bytes(index, "embeddings", el, emb)
    ang = gb.Granne.from_device_elements(index, "angular", gb.compute_embeddings_device("angular", el, emb))
    i8 = gb.Granne.from_device_elements(index, "angular_int", gb.compute_embeddings_device("angular_int", el, emb))
    a, s = summed.search_batch(q, max_search, 10, with_stats=True), ang.search_batch(q, max_search, 10, with_stats=True)
    same = all(np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)) for x, y in zip(a[:3], s[:3]))
    assert same and np.array_equal(a[3][:, :3], s[3][:, :3]), "angular rows must search like the SumEmbeddings container"
    # exact neighbours by cosine over the normalised sums
    rows = c.ground_truth_block(0, c.n)
    qt = torch.nn.functional.normalize(torch.from_numpy(q).cuda(), dim=1)
    truth = torch.cat([torch.topk(qt[i:i + 1024] @ rows.T, 10, dim=1).indices for i in range(0, len(q), 1024)]).cpu()
    c.free()

    def recall(ids):
        ids = torch.from_numpy(np.asarray(ids).astype(np.int64))
        return float((ids[:, :, None] == truth[:, None, :]).any(dim=2).float().mean())

    ids8 = i8.search_batch(q, max_search, 10)[0]
    out = {"n": c.n, "build_s_gpu": build_s, "max_search": max_search, "k": 10, "batch": 1024, "streams": streams,
           "queries": len(q), "angular_identical_to_sum_embeddings": True,
           "recall@10": {"embeddings": recall(a[0]), "angular": recall(s[0]), "angular_int": recall(ids8)}}
    rates = {}
    for _ in range(2):  # alternate the three containers, twice
        for name, ix in (("embeddings", summed), ("angular", ang), ("angular_int", i8)):
            rates.setdefault(name, []).append(qps(ix, q, max_search, 10, streams, 3))
    out["qps"] = {k: {"runs": v, "max": max(v)} for k, v in rates.items()}
    for ix in (summed, ang, i8):
        ix.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--search-n", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--max-search", type=int, default=200)
    a = ap.parse_args()
    import torch

    import granne_b200 as gb
    from granne_b200 import build

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    build.build()
    name, power = card()
    dev = torch.device("cuda", 0)
    res = {"tool": "embeddings_bench", "gpu": name, "power_limit": power}
    res["materialise"] = materialise(torch, gb, container(torch, gb, dev, a.n, 1234), a.calls)
    res["search"] = search(torch, gb, container(torch, gb, dev, a.search_n, 1234), a.streams, a.max_search)
    name2, power2 = card()
    res["gpu_after"], res["power_limit_after"] = name2, power2
    print(json.dumps(res))


if __name__ == "__main__":
    main()
