#!/usr/bin/env python
"""spann_bench.py -- SPANN search with the posting lists in HBM against the reference's SPANN::Index::SearchIndex.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, built by __graft_entry__.build() where
/root/reference exists; it links oracle/_ref only) on the host and records the build time.  Then, on the same folder and
the same queries:
  device     sptag_b200_spann_search, batch --nq, K = --k: wall time of --steps blocking calls after --warmup calls
             (host buffers, H2D and D2H included), repeated --repeats times; the median and the spread are reported
  reference  SPANN::Index::SearchIndex(QueryResult&) for every query, OpenMP over all host threads (one timed pass)
and compares ids and distance bits on the first --sample queries.  The card's name and power limit are read in the same
call.  Data: clustered float32 rows (seeded), queries are perturbed rows and fresh points.  Writes nothing in the tree:
the index goes to a temporary directory.

    python tools/spann_bench.py --n 200000 --dim 128 --nq 10000 --k 10
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
DRIVER = os.path.join(ROOT, "tests", "cpp", "spann_ref")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def data(n, dim, nq, seed=7):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((max(16, n // 500), dim)).astype(np.float32) * 3.0
    x = centres[rng.integers(0, len(centres), n)] + rng.standard_normal((n, dim), dtype=np.float32)
    q = np.concatenate([x[rng.choice(n, nq // 2, replace=False)] + 0.05 * rng.standard_normal((nq // 2, dim), dtype=np.float32),
                        centres[rng.integers(0, len(centres), nq - nq // 2)] + rng.standard_normal((nq - nq // 2, dim),
                                                                                                 dtype=np.float32)])
    return np.ascontiguousarray(x, np.float32), np.ascontiguousarray(q, np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=1000)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_ref is missing: run __graft_entry__.build() where the reference sources exist")
    from sptag_b200 import capi
    x, q = data(a.n, a.dim, a.nq)
    res = {"card": card(), "n": a.n, "dim": a.dim, "nq": a.nq, "k": a.k, "metric": "L2", "dtype": "f32",
           "host_threads": a.threads}
    with tempfile.TemporaryDirectory() as tmp:
        xf, qf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "q.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        q.tofile(qf)
        t0 = time.perf_counter()
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1", str(a.threads)])
        res["reference_build_s"] = round(time.perf_counter() - t0, 1)
        pre = os.path.join(tmp, "r")
        subprocess.check_call([DRIVER, "search", folder, qf, str(a.nq), str(a.k), pre, str(a.threads)])
        ref_ms = float(np.fromfile(pre + ".ms", np.float64)[0])
        ref_ids = np.fromfile(pre + ".ids", np.int32).reshape(a.nq, a.k)
        ref_dists = np.fromfile(pre + ".dists", np.float32).reshape(a.nq, a.k)
        s = capi.B200SpannIndex.load(folder, 0)
        res["posting_bytes"] = int(s.get_param("PostingBytes"))
        for _ in range(a.warmup):
            ids, dists = s.search(q, a.k)
        per_batch = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            for _ in range(a.steps):
                ids, dists = s.search(q, a.k)
            per_batch.append((time.perf_counter() - t0) / a.steps)
        dev_s = float(np.median(per_batch))
        _, _, stats = s.search(q, a.k, want_stats=True)
        s.close()
    m = min(a.sample, a.nq)
    res.update({
        "device_qps": round(a.nq / dev_s, 1),
        "device_ms_per_batch": round(dev_s * 1000, 2),
        "device_qps_min_max": [round(a.nq / max(per_batch), 1), round(a.nq / min(per_batch), 1)],
        "window_s": round(a.steps * dev_s, 2), "repeats": a.repeats,
        "reference_qps": round(a.nq / (ref_ms / 1000), 1),
        "mean_postings": float(stats[:, 0].mean()), "mean_list_elements": float(stats[:, 1].mean()),
        "mean_distances": float(stats[:, 2].mean()),
        "sample": m,
        "ids_equal": bool(np.array_equal(ids[:m], ref_ids[:m])),
        "dist_bits_equal": bool(np.array_equal(dists[:m].view(np.int32), ref_dists[:m].view(np.int32))),
    })
    print(json.dumps(res))


if __name__ == "__main__":
    main()
