"""What resuming a GPU build saves: a full build of n elements against a build checkpointed at a fraction of n, loaded
back into a builder (GranneBuilder index_bytes=..., i.e. GranneBuilder::from_bytes) and finished, with the reinsertion
pass on and off.  Reports wall times (host clock around calls that end in a device synchronise) and recall@10 of each
index against exact neighbours for held-out queries, with the card's name and power limit read in the same run.

    python tools/resume_bench.py [--n 4000000] [--dim 100] [--kind angular_int] [--fraction 0.9] [--queries 1000]
                                 [--dist clustered|uniform]

clustered: a Gaussian mixture on a low-dimensional subspace (easy: recall saturates); uniform: the reference's test
distribution (every component uniform in [-0.5, 0.5): hard in 100 dimensions, so recall differences show).

Elements live on the device (GranneBuilder.from_device_elements), so the times are the builder's, not a host upload's.
Prints a table and one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import granne_b200  # noqa: E402
from helpers.data import clustered_vectors, random_vectors  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def exact_top10(rows, q_el):
    """The 10 nearest elements of every query by cosine of the stored elements (what the angular distances order by)."""
    base = rows.float()
    base = base / base.norm(dim=1, keepdim=True).clamp_min(1e-30)
    qf = q_el.float()
    qf = qf / qf.norm(dim=1, keepdim=True).clamp_min(1e-30)
    out = []
    for s in range(0, qf.shape[0], 256):
        best_v, best_i = None, None
        for c in range(0, base.shape[0], 1 << 20):
            sim = qf[s:s + 256] @ base[c:c + (1 << 20)].T
            v, i = sim.topk(10, dim=1)
            i = i + c
            if best_v is None:
                best_v, best_i = v, i
            else:
                v = torch.cat([best_v, v], 1)
                i = torch.cat([best_i, i], 1)
                best_v, sel = v.topk(10, dim=1)
                best_i = i.gather(1, sel)
        out.append(best_i)
    return torch.cat(out).cpu().numpy()


def recall(builder, queries, exact, ef):
    index = builder.get_index()
    ids, _, _ = index.search_batch(queries, ef, 10)
    index.close()
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / 10.0 for a, b in zip(ids, exact)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=100)
    ap.add_argument("--kind", default="angular_int", choices=["angular", "angular_int"])
    ap.add_argument("--fraction", type=float, default=0.9)
    ap.add_argument("--num-neighbors", type=int, default=30)
    ap.add_argument("--max-search", type=int, default=200)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--search-ef", type=int, default=200)
    ap.add_argument("--dist", default="clustered", choices=["clustered", "uniform"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("resume_bench: no CUDA device (the builder has no CPU path)")
    from granne_b200 import build

    build.build()
    name, limit = card()
    n1 = int(a.n * a.fraction)
    raw = (clustered_vectors if a.dist == "clustered" else random_vectors)(a.n + a.queries, a.dim, seed=5)
    rows = granne_b200.elements_from_raw_device(a.kind, torch.from_numpy(raw[:a.n]).cuda())
    queries = raw[a.n:]
    q_el = granne_b200.elements_from_raw_device(a.kind, torch.from_numpy(queries).cuda())
    exact = exact_top10(rows, q_el)
    cfg = dict(num_neighbors=a.num_neighbors, max_search=a.max_search)

    # warm-up: module load and first launches of every kernel the timed builds use
    head = rows[:20000].contiguous()
    warm = granne_b200.GranneBuilder.from_device_elements(a.kind, head, **cfg)
    warm.build(10000)
    again = granne_b200.GranneBuilder.from_device_elements(a.kind, head, index_bytes=warm.index_bytes(), **cfg)
    again.build()
    warm.close()
    again.close()

    res = {}
    full = granne_b200.GranneBuilder.from_device_elements(a.kind, rows, **cfg)
    _, res["full_build_s"] = timed(full.build)
    res["full_recall10"] = recall(full, queries, exact, a.search_ef)
    full.close()

    part = granne_b200.GranneBuilder.from_device_elements(a.kind, rows, **cfg)
    _, res["partial_build_s"] = timed(lambda: part.build(n1))
    image, res["write_index_s"] = timed(part.index_bytes)
    image = image.tobytes()
    part.close()
    res["image_mb"] = len(image) / 1e6
    for reinsert in (True, False):
        tag = "reinsert_on" if reinsert else "reinsert_off"
        b, res["load_s"] = timed(lambda: granne_b200.GranneBuilder.from_device_elements(
            a.kind, rows, index_bytes=image, reinsert_elements=reinsert, **cfg))
        _, res["resume_%s_s" % tag] = timed(b.build)
        res["resume_%s_recall10" % tag] = recall(b, queries, exact, a.search_ef)
        b.close()

    print("card: %s, power limit %s" % (name, limit))
    print("%s %s n=%d dim=%d M=%d build max_search=%d; checkpoint at %d (%.0f%%), image %.1f MB; recall@10 of %d "
          "held-out queries at max_search=%d" % (a.dist, a.kind, a.n, a.dim, a.num_neighbors, a.max_search, n1,
                                                 100 * a.fraction, res["image_mb"], a.queries, a.search_ef))
    print("%-44s %10s %10s" % ("step", "seconds", "recall@10"))
    print("%-44s %10.2f %10.4f" % ("full build of n", res["full_build_s"], res["full_recall10"]))
    print("%-44s %10.2f" % ("build_partial(%d)" % n1, res["partial_build_s"]))
    print("%-44s %10.2f" % ("write_index", res["write_index_s"]))
    print("%-44s %10.2f" % ("load the image into a builder (last run)", res["load_s"]))
    for tag in ("reinsert_on", "reinsert_off"):
        print("%-44s %10.2f %10.4f" % ("resumed build() to n, %s" % tag.replace("_", " "), res["resume_%s_s" % tag],
                                       res["resume_%s_recall10" % tag]))
    print(json.dumps(dict(res, card=name, power_limit=limit, kind=a.kind, dist=a.dist, n=a.n, dim=a.dim, checkpoint=n1)))


if __name__ == "__main__":
    main()
