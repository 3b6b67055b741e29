#!/usr/bin/env python
"""spann_iterator_bench.py -- SPANN iterators with the posting lists in HBM against the reference's GetIterator + Next.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, as tools/spann_bench.py does; the index goes to
a temporary directory).  Then, on the same folder and queries, for each --iterators count:
  device     sptag_b200_spann_iterator_open over that many queries, then --calls x Next(--batch): wall time of the calls
             (host buffers and every per-round synchronisation included; the open is timed apart), --repeats times on
             fresh iterators; results/s of the median repeat, B200.LastIteratorRounds of the last call and the dedup
             table bytes
  reference  tests/cpp/spann_iter_ref with --threads host threads on the same queries and schedule (one timed pass)
and compares counts, ids and distance bits of every call on the first --sample queries.  The card's name and power limit
are read in the same call.

    python tools/spann_iterator_bench.py --n 200000 --dim 128 --iterators 10000,100 --calls 8 --batch 10
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

ITER_DRIVER = os.path.join(ROOT, "tests", "cpp", "spann_iter_ref")


def device_run(s, q, calls, batch):
    t0 = time.perf_counter()
    it = s.iterators(q)
    t_open = time.perf_counter() - t0
    out, rounds = [], []
    t0 = time.perf_counter()
    for _ in range(calls):
        out.append(it.next(batch))
        rounds.append(int(s.get_param("B200.LastIteratorRounds")))
    t_next = time.perf_counter() - t0
    dedup = int(s.get_param("B200.LastIteratorDedupBytes"))
    it.close()
    return t_open, t_next, out, rounds, dedup


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--iterators", default="10000,100")
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sample", type=int, default=500)
    ap.add_argument("--threads", type=int, default=16)
    a = ap.parse_args()
    if not (os.path.exists(DRIVER) and os.path.exists(ITER_DRIVER)):
        sys.exit("tests/cpp/spann_ref or spann_iter_ref is missing: run __graft_entry__.build() where the reference "
                 "sources exist")
    from sptag_b200 import capi
    counts_list = [int(v) for v in a.iterators.split(",")]
    x, q_all = data(a.n, a.dim, max(counts_list))
    res = {"card": card(), "n": a.n, "dim": a.dim, "metric": "L2", "dtype": "f32", "calls": a.calls, "batch": a.batch,
           "reference_threads": a.threads, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        xf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        t0 = time.perf_counter()
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1",
                               str(os.cpu_count() or 1)])
        res["reference_build_s"] = round(time.perf_counter() - t0, 1)
        s = capi.B200SpannIndex.load(folder, 0)
        res["head_batch"] = int(s.get_param("IterativeSearchHeadBatch"))
        device_run(s, q_all[:min(100, len(q_all))], a.calls, a.batch)  # warm-up: module loads, allocations
        for nit in counts_list:
            q = np.ascontiguousarray(q_all[:nit])
            runs = [device_run(s, q, a.calls, a.batch) for _ in range(a.repeats)]
            t_next = [r[1] for r in runs]
            med = runs[int(np.argsort(t_next)[len(t_next) // 2])]
            results = sum(int(c[0].sum()) for c in med[2])
            qf, pre = os.path.join(tmp, "q.bin"), os.path.join(tmp, "r")
            q.tofile(qf)
            subprocess.check_call([ITER_DRIVER, folder, qf, str(nit), pre, ",".join([str(a.batch)] * a.calls),
                                   str(a.threads)])
            ref_ms = float(np.fromfile(pre + ".ms", np.float64)[0])
            ref_counts = np.fromfile(pre + ".counts", np.int32).reshape(a.calls, nit)
            ref_ids = np.fromfile(pre + ".ids", np.int32).reshape(a.calls, nit, a.batch)
            ref_dists = np.fromfile(pre + ".dists", np.float32).reshape(a.calls, nit, a.batch)
            m = min(a.sample, nit)
            equal = all(np.array_equal(c[0][:m], ref_counts[i, :m]) and np.array_equal(c[1][:m], ref_ids[i, :m]) and
                        np.array_equal(c[2][:m].view(np.int32), ref_dists[i, :m].view(np.int32))
                        for i, c in enumerate(med[2]))
            res["runs"].append({
                "iterators": nit,
                "device_results_per_s": round(results / float(np.median(t_next)), 1),
                "device_next_ms_median": round(float(np.median(t_next)) * 1000 / a.calls, 3),
                "device_next_ms_min_max": [round(min(t_next) * 1000 / a.calls, 3), round(max(t_next) * 1000 / a.calls, 3)],
                "device_open_ms": round(med[0] * 1000, 2),
                "rounds_per_call": med[3],
                "dedup_bytes": med[4],
                "results": results,
                "reference_results_per_s": round(int(ref_counts.sum()) / (ref_ms / 1000), 1),
                "reference_ms_per_call": round(ref_ms / a.calls, 3),
                "sample": m,
                "counts_ids_dist_bits_equal": bool(equal),
            })
        s.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
