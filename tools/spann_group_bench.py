#!/usr/bin/env python
"""spann_group_bench.py -- a SPANN group (sptag_b200_spann_group_*: one pinned copy of the posting lists, one member per
GPU, an HBM cache spread over the members and read by peers) against one host-placed handle with the same cache budget,
and against the lists in HBM.

Builds one SPANN index with the unmodified reference (tests/cpp/spann_ref, built by __graft_entry__.build() where
/root/reference exists; it links oracle/_ref only), tools/spann_bench.py's 200 000 x 128 clustered float32 L2 rows, and
loads it three ways: posting_placement "device" on GPU 0 (the ceiling), "host" on GPU 0 with cache_warm at --budget % of
B200.PostingHostBytes, and a group over every visible GPU with group cache_warm at that budget per member.  With one
visible GPU the group has two members on it (--members overrides), and the run says that several GPUs were not measured.
Warm-up queries come from another seed than the --nq timed ones.  The three are timed alternately for --repeats rounds
of --steps blocking batch searches (K = --k, host buffers, H2D and D2H included) after --warmup calls; the median and the
min-max QPS are reported.  Per configuration also: the bytes copied over the host link per batch (B200.LastGatherBytes
less B200.LastPeerGatherBytes, summed over members), the bytes copied from peers' HBM, the distinct cached lists, and
whether ids and distance bits equal the device handle's.  The card's name and power limit, the device count and which
device pairs have peer access are read in the same call.  Writes nothing in the tree: the index goes to a temporary
directory.

    python tools/spann_group_bench.py
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
from spann_cache_bench import timed, warm_queries  # noqa: E402


def link_bytes(handles):
    """(host-link bytes, peer bytes) of the last search on each handle, summed"""
    host = peer = 0
    for h in handles:
        gathered, p = int(h.get_param("B200.LastGatherBytes")), int(h.get_param("B200.LastPeerGatherBytes"))
        host += gathered - p
        peer += p
    return host, peer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--nwarm", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--budget", type=int, default=25, help="cache budget per handle / member, %% of the lists' bytes")
    ap.add_argument("--members", type=int, default=0, help="group members (0: every visible GPU, 2 with one GPU)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_ref is missing: run __graft_entry__.build() where the reference sources exist")
    import torch
    from sptag_b200 import capi
    ndev = torch.cuda.device_count()
    if ndev < 1:
        sys.exit("no CUDA device")
    members = a.members or (ndev if ndev > 1 else 2)
    devices = [i % ndev for i in range(members)]
    peer = {"%d-%d" % (i, j): bool(torch.cuda.can_device_access_peer(i, j)) for i in range(ndev) for j in range(ndev)
            if i != j}
    x, q = data(a.n, a.dim, a.nq)
    qw = warm_queries(x, a.nwarm)
    res = {"card": card(), "device_count": ndev, "peer_access": peer, "group_devices": devices,
           "multi_gpu_measured": len(set(devices)) > 1, "n": a.n, "dim": a.dim, "k": a.k, "nq": a.nq, "nwarm": a.nwarm,
           "metric": "L2", "dtype": "f32", "budget_pct": a.budget, "steps": a.steps, "repeats": a.repeats, "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        xf, folder = os.path.join(tmp, "x.bin"), os.path.join(tmp, "spann")
        x.tofile(xf)
        subprocess.check_call([DRIVER, "build", folder, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1",
                               str(a.threads)])
        dev = capi.B200SpannIndex.load(folder, 0, posting_placement="device")
        host = capi.B200SpannIndex.load(folder, 0, posting_placement="host")
        group = capi.B200SpannGroup.load(folder, devices)
        host_bytes = int(host.get_param("B200.PostingHostBytes"))
        budget = host_bytes * a.budget // 100
        res["host_posting_bytes"] = host_bytes
        res["budget_bytes"] = budget
        single_lists = host.cache_warm(qw, budget)
        group_lists, owners = group.cache_warm(qw, budget)
        res["owners_per_member"] = np.bincount(owners, minlength=members).tolist()
        ids_d, dists_d = dev.search(q, a.k)
        configs = {"device": (dev, [], 0), "host": (host, [host], len(single_lists)),
                   "group": (group, group.members, len(set(group_lists.tolist())))}
        runs = {}
        for name, (h, parts, cached) in configs.items():
            ids, dists = h.search(q, a.k)
            host_link, from_peers = link_bytes(parts)
            runs[name] = {"name": name, "distinct_cached_lists": cached, "host_link_bytes_per_batch": host_link,
                          "peer_bytes_per_batch": from_peers, "ids_equal": bool(np.array_equal(ids, ids_d)),
                          "dist_bits_equal": bool(np.array_equal(dists.view(np.int32), dists_d.view(np.int32)))}
        for _ in range(a.warmup):
            for h, _, _ in configs.values():
                h.search(q, a.k)
        times = {name: [] for name in configs}
        for _ in range(a.repeats):  # alternated, so that every configuration sees the same host and card conditions
            for name, (h, _, _) in configs.items():
                times[name].append(timed(h, q, a.k, a.steps))
        for name, t in times.items():
            m = float(np.median(t))
            runs[name].update({"qps": round(a.nq / m, 1), "qps_min_max": [round(a.nq / max(t), 1), round(a.nq / min(t), 1)],
                               "ms_per_batch": round(m * 1000, 3)})
            res["runs"].append(runs[name])
        group.close()
        host.close()
        dev.close()
    if not res["multi_gpu_measured"]:
        res["note"] = "one visible GPU: the group's members share it; several GPUs and NVLink are not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
