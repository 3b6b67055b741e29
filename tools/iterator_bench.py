#!/usr/bin/env python
"""ResultIterator scans on the device vs the reference (SURVEY.md 8 row f3): open one iterator per query, call
Next(batch) `rounds` times, report results/s through the C ABI (host buffers) next to the unmodified reference's
ResultIterator on the host cores (a bounded sample of the same queries), and check the two agree call by call.

    python tools/iterator_bench.py --num-vectors 1000000 --dim 128 --nq 4096 --batch 10 --rounds 8

--visited picks the iterators' visited set (B200.IteratorVisitedSet): a bitmap per query, a growing hash table per
query, or both, timed in alternating repeats on two handles of one index and checked to return the same calls.  Per
mode the report gives results/s, the open time, the visited-set bytes held after the scan, and the table growths and
suspensions of the last call; with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

VISITED = {"bitmap": 0, "hashed": 1}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def scan(idx, qh, batch, rounds):
    """Open one iterator per query, Next(batch) `rounds` times: outputs, seconds per call, open seconds, visited-set stats."""
    t0 = time.time()
    its = idx.iterators(qh)
    t_open = time.time() - t0
    outs, secs, kms, growths, susp = [], [], [], 0, [0, 0]
    for _ in range(rounds):
        t = time.time()
        outs.append(its.next(batch))
        secs.append(time.time() - t)
        kms.append(idx.last_kernel_ms())
        growths += int(idx.get_param("B200.LastIteratorGrowths"))
        s = [int(v) for v in idx.get_param("B200.LastIteratorSuspensions").split(",")]
        susp = [susp[0] + s[0], susp[1] + s[1]]
    vbytes = int(idx.get_param("B200.LastIteratorVisitedBytes"))
    its.close()
    return outs, secs, t_open, kms, {"visited_bytes": vbytes, "growths": growths, "suspensions_step": susp[0],
                                     "suspensions_trees": susp[1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num-vectors", type=int, default=1000000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--metric", default="L2", choices=["L2", "Cosine"])
    ap.add_argument("--data", default="lowrank", choices=["lowrank", "iid"])
    ap.add_argument("--rank-dim", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--nq", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--maxcheck", type=int, default=2048)
    ap.add_argument("--cpu-sample", type=int, default=256)
    ap.add_argument("--visited", default="bitmap", choices=["bitmap", "hashed", "both"])
    ap.add_argument("--repeats", type=int, default=1, help="timed scans per mode (alternating with --visited both)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    a.raw_type = "float"
    a.n = a.num_vectors
    a.algo = "bkt"
    if a.rank_dim <= 0:
        a.rank_dim = 32 if a.dim >= 512 else 16

    import numpy as np
    import torch
    import bench
    import reflib
    from tools import gpu_index_builder as B
    from sptag_b200 import B200Index, capi

    dev = torch.device("cuda", 0)
    log = bench.log
    x = bench.gen_data(a, a.n, a.seed + 1000, dev)
    q = bench.gen_data(a, a.nq, a.seed + 7, dev)
    torch.backends.cuda.matmul.allow_tf32 = True
    nodes, starts, graph = B.build_index(x, a.metric, seed=a.seed, log=log, algo="BKT")
    torch.backends.cuda.matmul.allow_tf32 = False
    xh, qh = x.cpu().numpy(), q.cpu().numpy()
    del x, q
    torch.cuda.empty_cache()
    modes = ["bitmap", "hashed"] if a.visited == "both" else [a.visited]
    handles = {}
    for m in modes:
        handles[m] = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT,
                                      metric=capi.METRIC_COSINE if a.metric == "Cosine" else capi.METRIC_L2, vectors=xh,
                                      graph=graph, tree_starts=starts, tree_nodes=nodes)
        handles[m].set_param("MaxCheck", a.maxcheck)
        handles[m].set_param("B200.IteratorVisitedSet", VISITED[m])
        # warm-up on a few queries
        w = handles[m].iterators(qh[:64])
        w.next(a.batch)
        w.close()

    # the timed scans, modes alternating
    runs = {m: [] for m in modes}
    for _ in range(max(1, a.repeats)):
        for m in modes:
            runs[m].append(scan(handles[m], qh, a.batch, a.rounds))
    outs = runs[modes[0]][0][0]
    report = {"n": a.n, "dim": a.dim, "metric": a.metric, "max_check": a.maxcheck, "iterators": a.nq, "batch": a.batch,
              "rounds": a.rounds, "repeats": max(1, a.repeats), "card": card(), "modes": {}}
    for m in modes:
        rates, opens = [], []
        for o, secs, t_open, kms, st in runs[m]:
            total = int(sum(int(c[0].sum()) for c in o))
            rates.append(total / sum(secs))
            opens.append(t_open)
            log("%s: %d iterators x %d x Next(%d): %d results in %.3f s (+ open %.3f s) = %.0f results/s; kernel ms per "
                "call %s; %s" % (m, a.nq, a.rounds, a.batch, total, sum(secs), t_open, rates[-1],
                                 ["%.1f" % k for k in kms], st))
        report["modes"][m] = {"results": total, "device_results_per_second": [round(r, 1) for r in rates],
                              "open_seconds": [round(t, 4) for t in opens],
                              "kernel_ms_per_call": [round(k, 2) for k in runs[m][-1][3]], **runs[m][-1][4]}
    if len(modes) == 2:
        same = True
        for x, y in zip(runs["bitmap"][0][0], runs["hashed"][0][0]):
            same &= bool(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and
                         np.array_equal(x[2].view(np.int32), y[2].view(np.int32)) and np.array_equal(x[3], y[3]))
        report["hashed_equals_bitmap"] = same
        log("hashed equals bitmap: %s" % same)
    for m in modes[1:]:
        handles[m].close()
    idx = handles[modes[0]]
    if a.cpu_sample > 0 and reflib.have_ref():
        ns = min(a.cpu_sample, a.nq)
        with tempfile.TemporaryDirectory() as tmp:
            B.save_index_folder(tmp, xh, graph, nodes, starts, a.metric, algo="BKT")
            r = reflib.RefIndex.load(tmp)
            r.set_param("MaxCheck", a.maxcheck)
            same = True
            t = time.time()
            n_res = 0
            for i in range(ns):
                it = r.iterator(qh[i])
                for rd in range(a.rounds):
                    c, ids, dists, rm = it.next(a.batch)
                    n_res += c
                    o = outs[rd]
                    same &= bool(c == o[0][i] and np.array_equal(ids, o[1][i]) and
                                 np.array_equal(dists.view(np.int32), o[2][i].view(np.int32)) and rm == bool(o[3][i]))
                it.close()
            cpu_s = time.time() - t
            # all host threads, no Python in the loop: the CPU baseline proper
            threads = os.cpu_count() or 1
            nb = min(a.nq, max(ns, 2048))
            r.iterator_scan(qh[:min(nb, 256)], a.batch, a.rounds, threads)
            n_all, s_all = r.iterator_scan(qh[:nb], a.batch, a.rounds, threads)
        report["cpu_reference"] = {"results_per_second": round(n_all / s_all, 1), "threads": threads,
                                   "sample_iterators": nb,
                                   "kind": "reference (oracle/_ref ResultIterator, OpenMP over queries)"}
        log("reference, %d threads: %d iterators, %d results in %.3f s = %.0f results/s" % (threads, nb, n_all, s_all, n_all / s_all))
        report["parity_vs_reference"] = {"iterators": ns, "calls": ns * a.rounds, "bit_exact": same}
        log("reference: %d iterators, %d results in %.2f s = %.0f results/s on one thread; parity %s"
            % (ns, n_res, cpu_s, n_res / cpu_s, same))
    idx.close()
    line = json.dumps(report)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
