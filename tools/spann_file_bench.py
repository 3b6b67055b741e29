#!/usr/bin/env python
"""spann_file_bench.py -- SPANN search with the posting lists left in their files, against the same index in HBM and in
pinned host memory.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, built by __graft_entry__.build() where
/root/reference exists; it links oracle/_ref only) and loads it as posting_placement "device", "host" and "file", and once
more as "file" with an HBM cache installed by cache_warm for each budget (--budgets, in % of the lists' bytes; --nwarm
warm-up queries drawn with another seed than the --nq timed ones).  sptag_b200_spann_search (batch --nq, K = --k) is
timed on every handle, alternated for --repeats rounds of --steps blocking calls (host buffers, H2D and D2H included)
after --warmup calls each; the median and the spread are reported.  Also reported per handle: the posting-file bytes read
per batch (B200.LastReadBytes), the bytes staged into HBM and the rounds (B200.LastGatherBytes / LastGatherRounds), the
effective read rate of a file handle (read bytes over its extra time per batch relative to the device handle), and
whether ids and distance bits equal the device handle's.  The card's name and power limit are read in the same call.

Page cache: the posting files were just written, so by default every read is served from the host's page cache; the
result says so ("page_cache": "warm").  Dropping the host's caches would change a host setting, which this tool never
does.  --cold instead calls posix_fadvise(POSIX_FADV_DONTNEED) on the posting files this tool wrote in its temporary
directory before each timed call (one call per step, the advice's time outside the timing), and says "cold" (the kernel
may still keep pages that are in use elsewhere).  Data: tools/spann_bench.py's clustered float32 rows.  Writes nothing in
the tree: the index goes to a temporary directory.

    python tools/spann_file_bench.py --n 200000 --dim 128 --nq 10000 --k 10
"""
import argparse
import glob
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
from spann_cache_bench import warm_queries  # noqa: E402


def drop(paths):
    for p in paths:
        fd = os.open(p, os.O_RDONLY)
        try:
            os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
        finally:
            os.close(fd)


def timed(s, q, k, steps, cold):
    total = 0.0
    for _ in range(steps):
        if cold:
            drop(cold)
        t0 = time.perf_counter()
        s.search(q, k)
        total += time.perf_counter() - t0
    return total / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--nwarm", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--budgets", type=float, nargs="*", default=[10.0, 50.0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--cold", action="store_true")
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_ref is missing: run __graft_entry__.build() where the reference sources exist")
    from sptag_b200 import capi
    x, q_all = data(a.n, a.dim, a.nq)
    q = q_all[:a.nq]
    res = {"card": card(), "n": a.n, "dim": a.dim, "nq": a.nq, "k": a.k, "metric": "L2", "dtype": "f32",
           "steps": a.steps, "repeats": a.repeats, "page_cache": "cold" if a.cold else "warm", "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        xf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1", str(a.threads)])
        os.remove(xf)
        posting = sorted(glob.glob(os.path.join(folder, "SPTAGFullList.bin*")))
        res["posting_file_bytes"] = sum(os.path.getsize(p) for p in posting)
        handles = {}
        for name in ("device", "host", "file"):
            t0 = time.perf_counter()
            handles[name] = capi.B200SpannIndex.load(folder, 0, posting_placement=name)
            res[name + "_load_s"] = round(time.perf_counter() - t0, 2)
        list_bytes = int(handles["host"].get_param("B200.PostingHostBytes"))
        warm = warm_queries(x, a.nwarm)
        for pct in a.budgets:
            s = capi.B200SpannIndex.load(folder, 0, posting_placement="file")
            lists = s.cache_warm(warm, int(list_bytes * pct / 100))
            handles["file_cache_%g%%" % pct] = s
            res["file_cache_%g%%_lists" % pct] = len(lists)
        ids_d, dists_d = handles["device"].search(q, a.k)
        counters, same = {}, {}
        for name, s in handles.items():
            ids, dists = s.search(q, a.k)
            counters[name] = {p: int(s.get_param("B200." + p)) for p in ("LastReadBytes", "LastGatherBytes", "LastGatherRounds")}
            same[name] = (bool(np.array_equal(ids, ids_d)), bool(np.array_equal(dists.view(np.int32), dists_d.view(np.int32))))
            for _ in range(a.warmup):
                s.search(q, a.k)
        times = {name: [] for name in handles}
        for _ in range(a.repeats):  # alternated, so that every handle sees the same host and card conditions
            for name, s in handles.items():
                times[name].append(timed(s, q, a.k, a.steps, posting if a.cold and name.startswith("file") else None))
        md = float(np.median(times["device"]))
        for name in handles:
            t = times[name]
            m = float(np.median(t))
            read = counters[name]["LastReadBytes"]
            res["runs"].append({
                "handle": name, "qps": round(a.nq / m, 1), "qps_min_max": [round(a.nq / max(t), 1), round(a.nq / min(t), 1)],
                "ms_per_batch": round(m * 1000, 3),
                "read_bytes_per_batch": read, "staged_bytes_per_batch": counters[name]["LastGatherBytes"],
                "rounds_per_batch": counters[name]["LastGatherRounds"],
                "read_gb_s_effective": round(read / (m - md) / 1e9, 2) if read and m > md else None,
                "ids_equal": same[name][0], "dist_bits_equal": same[name][1],
            })
        for s in handles.values():
            s.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
