#!/usr/bin/env python
"""spann_cache_bench.py -- SPANN search with the posting lists in pinned host memory and an HBM cache of the hottest
lists (sptag_b200_spann_cache_warm), against the same index with every list in HBM.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, built by __graft_entry__.build() where
/root/reference exists; it links oracle/_ref only) and loads it twice: posting_placement "device" and "host".  On the
host handle a cache is installed for each budget (--budgets, in % of B200.PostingHostBytes) by cache_warm with --nwarm
warm-up queries drawn with another seed than the --nq timed ones; each cache is then re-installed by cache_lists from the
ids cache_warm returned, so that every configuration is timed in one call.  sptag_b200_spann_search (batch --nq, K = --k)
is timed on the device handle and on every cache configuration, alternated for --repeats rounds of --steps blocking calls
(host buffers, H2D and D2H included) after --warmup calls each; the median and the spread are reported.  Also reported
per configuration: the bytes gathered over the host link per batch (B200.LastGatherBytes) and the rounds, the cached
lists and bytes (B200.PostingCacheLists / PostingCacheBytes), how much less is gathered than without a cache, and
whether ids and distance bits equal the device handle's for all queries.  After the timing, each configuration
searches the batch once more with a stage that holds every list (one round), so that its gathered bytes are the
batch's union of uncached lists: with the uncached handle's figure, the batch's whole union, that gives the share of
the union the cache serves from HBM.  The card's name and power limit are read in the same call.  At 200k x 128 the
lists fit in HBM, so the host placement with a cache stands in for an index whose lists do not.  Data: tools/spann_bench.py's clustered float32 rows.  Writes nothing in the tree: the
index goes to a temporary directory.

    python tools/spann_cache_bench.py --n 200000 --dim 128 --nq 10000 --nwarm 10000 --k 10
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
from spann_bench import DRIVER, card, data  # noqa: E402


def warm_queries(x, nq, seed=11):
    """Queries of the timed set's two kinds (perturbed rows, points near a row) from their own seed"""
    rng = np.random.default_rng(seed)
    n, dim = x.shape
    near = x[rng.choice(n, nq // 2, replace=False)] + 0.05 * rng.standard_normal((nq // 2, dim), dtype=np.float32)
    fresh = x[rng.choice(n, nq - nq // 2, replace=False)] + rng.standard_normal((nq - nq // 2, dim), dtype=np.float32)
    return np.ascontiguousarray(np.concatenate([near, fresh]), np.float32)


def timed(s, q, k, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        s.search(q, k)
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--nwarm", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--budgets", type=int, nargs="+", default=[0, 10, 25, 50, 100])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_ref is missing: run __graft_entry__.build() where the reference sources exist")
    from sptag_b200 import capi
    x, q = data(a.n, a.dim, a.nq)
    qw = warm_queries(x, a.nwarm)
    res = {"card": card(), "n": a.n, "dim": a.dim, "k": a.k, "nq": a.nq, "nwarm": a.nwarm, "metric": "L2", "dtype": "f32",
           "steps": a.steps, "repeats": a.repeats, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        xf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        t0 = time.perf_counter()
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1", str(a.threads)])
        res["reference_build_s"] = round(time.perf_counter() - t0, 1)
        dev = capi.B200SpannIndex.load(folder, 0, posting_placement="device")
        host = capi.B200SpannIndex.load(folder, 0, posting_placement="host")
        host_bytes = int(host.get_param("B200.PostingHostBytes"))
        res["host_posting_bytes"] = host_bytes
        res["stage_bytes"] = int(host.get_param("B200.PostingStageBytes"))
        ids_d, dists_d = dev.search(q, a.k)
        configs = []  # (name, budget %, list ids or None for the device handle)
        for pct in a.budgets:
            t0 = time.perf_counter()
            lists = host.cache_warm(qw, host_bytes * pct // 100)
            configs.append(("host_cache_%d" % pct, pct, lists, round(time.perf_counter() - t0, 3)))
        runs = {"device": {"name": "device"}}
        base_gathered = None
        for name, pct, lists, warm_s in configs:
            host.cache_lists(lists)
            ids_h, dists_h = host.search(q, a.k)
            gathered = int(host.get_param("B200.LastGatherBytes"))
            if pct == 0:
                base_gathered = gathered
            runs[name] = {
                "name": name, "budget_pct": pct, "warm_s": warm_s,
                "cached_lists": int(host.get_param("B200.PostingCacheLists")),
                "cached_bytes": int(host.get_param("B200.PostingCacheBytes")),
                "gathered_bytes_per_batch": gathered, "gather_rounds": int(host.get_param("B200.LastGatherRounds")),
                "ids_equal": bool(np.array_equal(ids_d, ids_h)),
                "dist_bits_equal": bool(np.array_equal(dists_d.view(np.int32), dists_h.view(np.int32))),
            }
        for r in runs.values():
            if "gathered_bytes_per_batch" in r and base_gathered:
                r["gathered_reduction"] = round(1 - r["gathered_bytes_per_batch"] / base_gathered, 4)
        for _ in range(a.warmup):
            dev.search(q, a.k)
            for name, _, lists, _ in configs:
                host.cache_lists(lists)
                host.search(q, a.k)
        times = {name: [] for name in runs}
        for _ in range(a.repeats):  # alternated, so that every configuration sees the same host and card conditions
            times["device"].append(timed(dev, q, a.k, a.steps))
            for name, _, lists, _ in configs:
                host.cache_lists(lists)
                host.search(q, a.k)
                times[name].append(timed(host, q, a.k, a.steps))
        # one round per batch: the gathered bytes are the batch's union of uncached lists, counted once
        stage = res["stage_bytes"]
        host.set_param("B200.PostingStageBytes", host_bytes)
        union = {}
        for name, pct, lists, _ in configs:
            host.cache_lists(lists)
            host.search(q, a.k)
            assert int(host.get_param("B200.LastGatherRounds")) == 1
            union[name] = int(host.get_param("B200.LastGatherBytes"))
        host.set_param("B200.PostingStageBytes", stage)
        whole = union.get("host_cache_0")
        res["union_bytes_per_batch"] = whole
        for name in union:
            runs[name]["uncached_union_bytes"] = union[name]
            if whole:
                runs[name]["union_share_from_hbm"] = round(1 - union[name] / whole, 4)
        for name, t in times.items():
            m = float(np.median(t))
            runs[name].update({"qps": round(a.nq / m, 1), "qps_min_max": [round(a.nq / max(t), 1), round(a.nq / min(t), 1)],
                               "ms_per_batch": round(m * 1000, 3)})
            res["runs"].append(runs[name])
        dev.close()
        host.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
