#!/usr/bin/env python
"""multi_scan_bench.py -- the batched multi-index scan (sptag_b200_multi_scan) against the reference's MultiIndexScan.

Builds two views of the same --n items with tools/gpu_index_builder.py (an L2 view of --dims[0] and a Cosine view of
--dims[1] floats, random projections of one latent space), saves them to a temporary directory and loads them on the
device.  Then for each batch size of --batches:
  device     capi.multi_scan over the first `batch` queries after one untimed warm-up call of that shape, --repeats
             times; the host clock around each call, which returns after its outputs are copied back (a synchronise);
             results/s of the median call, rounds, launches per call and per round
  reference  tests/cpp/multi_scan_ref (MultiIndexScan::Init + Next until false per query, the unmodified reference) with
             --threads host threads on the same folders and queries: one timed pass
Every timed device call's counts, ids and score bits are compared with the reference's.  The card's name and power
limit are read in the same call.  One JSON line per batch size.

    python tools/multi_scan_bench.py --n 1000000 --dims 64,32 --batches 1000,10000
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from spann_bench import card  # noqa: E402

DRIVER = os.path.join(ROOT, "tests", "cpp", "multi_scan_ref")


def views(n, nq, dims, seed=5):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((max(16, n // 500), 16)).astype(np.float32) * 3.0
    z = centres[rng.integers(0, len(centres), n + nq)] + rng.standard_normal((n + nq, 16), dtype=np.float32)
    out = []
    for i, d in enumerate(dims):
        x = z @ rng.standard_normal((16, d)).astype(np.float32) + 0.1 * rng.standard_normal((n + nq, d), dtype=np.float32)
        if i % 2 == 1:  # the Cosine views: unit rows
            x /= np.linalg.norm(x, axis=1, keepdims=True)
        out.append((np.ascontiguousarray(x[:n], np.float32), np.ascontiguousarray(x[n:], np.float32)))
    return out


def reference(folders, queries, k, term, limit, threads, tmp):
    nq = queries[0].shape[0]
    pre = os.path.join(tmp, "ref")
    args = [DRIVER, str(nq), pre, str(k), str(term), str(limit), "sum", "0", str(threads)]
    for i, (f, q) in enumerate(zip(folders, queries)):
        qf = os.path.join(tmp, "q%d.bin" % i)
        q.tofile(qf)
        args += [f, qf]
    subprocess.check_call(args, stdout=subprocess.DEVNULL)
    ids = np.fromfile(pre + ".ids", np.int32).reshape(nq, k)
    scores = np.fromfile(pre + ".scores", np.float32).reshape(nq, k)
    counts = np.fromfile(pre + ".counts", np.int32)
    ms = float(np.fromfile(pre + ".ms", np.float64)[0])
    return ids, scores, counts, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--dims", default="64,32")
    ap.add_argument("--batches", default="1000,10000")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--term", type=int, default=20, help="termCondVal: consecutive drops that end a query")
    ap.add_argument("--limit", type=int, default=1000, help="searchLimit: ids seen that end a query")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    import torch
    from gpu_index_builder import build_index, save_index_folder
    from sptag_b200 import capi
    if not os.path.exists(DRIVER):
        sys.exit("%s is missing: __graft_entry__.build() makes it where the reference was compiled" % DRIVER)
    dims = [int(x) for x in a.dims.split(",")]
    batches = [int(x) for x in a.batches.split(",")]
    nq = max(batches)
    data = views(a.n, nq, dims)
    gpu = card()
    with tempfile.TemporaryDirectory() as tmp:
        folders, handles = [], []
        for i, (x, _) in enumerate(data):
            metric = "Cosine" if i % 2 == 1 else "L2"
            t0 = time.time()
            nodes, starts, graph = build_index(torch.from_numpy(x).cuda(), metric=metric)
            folder = os.path.join(tmp, "view%d" % i)
            save_index_folder(folder, x, graph, nodes, starts, metric)
            print("view %d: %d x %d %s built in %.0f s" % (i, a.n, x.shape[1], metric, time.time() - t0), file=sys.stderr)
            folders.append(folder)
            handles.append(capi.B200Index.load(folder, 0))
        torch.cuda.empty_cache()
        for b in batches:
            qs = [np.ascontiguousarray(q[:b]) for _, q in data]
            capi.multi_scan(handles, qs, a.k, term_cond=a.term, search_limit=a.limit)  # warm-up of this shape
            times, launches, outs = [], [], []
            for _ in range(a.repeats):
                l0 = capi.launch_count()
                t0 = time.perf_counter()
                out = capi.multi_scan(handles, qs, a.k, term_cond=a.term, search_limit=a.limit, want_stats=True)
                times.append(time.perf_counter() - t0)
                launches.append(capi.launch_count() - l0)
                outs.append(out)
            r_ids, r_scores, r_counts, r_ms = reference(folders, qs, a.k, a.term, a.limit, a.threads, tmp)
            same = all(np.array_equal(o[2], r_counts) and np.array_equal(o[0], r_ids) and
                       np.array_equal(o[1].view(np.int32), r_scores.view(np.int32)) for o in outs)
            rounds = int(outs[0][3][:, capi.MS_ROUNDS].max())
            med = float(np.median(times))
            print(json.dumps({
                "workload": "multi_scan", "n": a.n, "views": ["%dd %s" % (d, "Cosine" if i % 2 else "L2")
                                                              for i, d in enumerate(dims)],
                "batch": b, "k": a.k, "term_cond": a.term, "search_limit": a.limit, "weights": "sum",
                "device_ms": [round(t * 1e3, 2) for t in times], "device_results_per_s": float(outs[0][2].sum()) / med,
                "device_queries_per_s": b / med, "rounds": rounds, "launches_per_call": launches[0],
                "launches_per_round": launches[0] / rounds,
                "mean_rounds": float(outs[0][3][:, capi.MS_ROUNDS].mean()),
                "reference_ms": round(r_ms, 1), "reference_threads": a.threads,
                "reference_queries_per_s": b / (r_ms / 1e3), "reference_results_per_s": float(r_counts.sum()) / (r_ms / 1e3), "identical_to_reference": same, "gpu": gpu}))
            if not same:
                sys.exit("device outputs differ from the reference's")
        for h in handles:
            h.close()


if __name__ == "__main__":
    main()
