#!/usr/bin/env python
"""spann_host_bench.py -- SPANN search with the posting lists in pinned host memory against the same index in HBM.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, built by __graft_entry__.build() where
/root/reference exists; it links oracle/_ref only) and loads it twice: posting_placement "device" (the lists in HBM) and
"host" (the lists in pinned host memory, each batch's chosen lists gathered into HBM).  On the same queries,
sptag_b200_spann_search (batch --nq, K = --k) is timed on both handles, alternating them for --repeats rounds of --steps
blocking calls (host buffers, H2D and D2H included) after --warmup calls each; the median and the spread are reported.
Also reported: the bytes the host placement gathered per batch (B200.LastGatherBytes) and its rounds, the bytes of every
query's chosen lists before the union (list elements read x (row stride + 4)), the effective host-link rate of the
gather (gathered bytes over the extra time per batch of the host placement over the device placement), and whether ids
and distance bits of the two placements are identical.  The card's name and power limit are read in the same call.
Data: tools/spann_bench.py's clustered float32 rows.  Writes nothing in the tree: the index goes to a temporary directory.

    python tools/spann_host_bench.py --n 200000 --dim 128 --nq 10000 --k 10
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


def timed(s, q, k, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        s.search(q, k)
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, nargs="+", default=[10000, 1000])
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_ref is missing: run __graft_entry__.build() where the reference sources exist")
    from sptag_b200 import capi
    x, q_all = data(a.n, a.dim, max(a.nq))
    res = {"card": card(), "n": a.n, "dim": a.dim, "k": a.k, "metric": "L2", "dtype": "f32", "steps": a.steps,
           "repeats": a.repeats, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        xf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        t0 = time.perf_counter()
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1", str(a.threads)])
        res["reference_build_s"] = round(time.perf_counter() - t0, 1)
        t0 = time.perf_counter()
        dev = capi.B200SpannIndex.load(folder, 0, posting_placement="device")
        res["device_load_s"] = round(time.perf_counter() - t0, 2)
        t0 = time.perf_counter()
        host = capi.B200SpannIndex.load(folder, 0, posting_placement="host")
        res["host_load_s"] = round(time.perf_counter() - t0, 2)
        res["device_posting_bytes"] = int(dev.get_param("PostingBytes"))
        res["host_posting_bytes"] = {"hbm": int(host.get_param("PostingBytes")),
                                     "pinned": int(host.get_param("B200.PostingHostBytes"))}
        res["stage_bytes"] = int(host.get_param("B200.PostingStageBytes"))
        elem_bytes = (a.dim * 4 + 15) // 16 * 16 + 4
        for nq in a.nq:
            q = q_all[:nq]
            ids_d, dists_d, stats = dev.search(q, a.k, want_stats=True)
            ids_h, dists_h = host.search(q, a.k)
            gathered = int(host.get_param("B200.LastGatherBytes"))
            rounds = int(host.get_param("B200.LastGatherRounds"))
            for _ in range(a.warmup):
                dev.search(q, a.k)
                host.search(q, a.k)
            t_dev, t_host = [], []
            for _ in range(a.repeats):  # alternated, so that both see the same host and card conditions
                t_dev.append(timed(dev, q, a.k, a.steps))
                t_host.append(timed(host, q, a.k, a.steps))
            md, mh = float(np.median(t_dev)), float(np.median(t_host))
            chosen = int(stats[:, 1].astype(np.int64).sum()) * elem_bytes
            res["runs"].append({
                "nq": nq,
                "device_qps": round(nq / md, 1), "device_qps_min_max": [round(nq / max(t_dev), 1), round(nq / min(t_dev), 1)],
                "host_qps": round(nq / mh, 1), "host_qps_min_max": [round(nq / max(t_host), 1), round(nq / min(t_host), 1)],
                "device_ms_per_batch": round(md * 1000, 3), "host_ms_per_batch": round(mh * 1000, 3),
                "gathered_bytes_per_batch": gathered, "gather_rounds": rounds,
                "chosen_list_bytes_per_batch": chosen,
                "union_share_of_chosen": round(gathered / max(chosen, 1), 4),
                "host_link_gb_s_effective": round(gathered / max(mh - md, 1e-9) / 1e9, 2) if mh > md else None,
                "ids_equal": bool(np.array_equal(ids_d, ids_h)),
                "dist_bits_equal": bool(np.array_equal(dists_d.view(np.int32), dists_h.view(np.int32))),
            })
        dev.close()
        host.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
