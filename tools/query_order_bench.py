#!/usr/bin/env python
"""query_order_bench.py -- does the order of a batch's queries change how fast the device searches it?

For each shape one handle is loaded and the same batch is searched in three orders, alternating within every round:
    (a) generation order;
    (b) sorted by a tree key (a stable sort), one setting per key depth in --levels;
    (c) a seeded random shuffle.
The key of a query is the path of child indices of a greedy descent of tree 0 (nearest child centre at each level, the
metric's fp32 distance, 5 bits per level, a leaf or duplicate-group head reached early padded with zeros), computed
with torch.  The idea under test: queries with equal keys read mostly the same rows, so running them at the same time
could serve part of those reads from L2 (DESIGN.md §7b records the outcome).

Reported per setting: median / min / max QPS (CUDA events around --steps batches of search_device) and kernel ms (the
handle's last launch), and whether the results of (b) and (c), put back into batch order, have the same ids and
distance bits as (a).  The card's name and power limit are read in the same call.

Shapes (indexes built and cached by bench.py's builder, under --cache):
    c2     BKT 1M x 768 float32 cosine (BASELINE config 2, bench.py's default)
    1m128  BKT 1M x 128 float32 L2

    python tools/query_order_bench.py --shapes c2,1m128 --levels 2,3
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = {
    "c2": ["--n", "1000000", "--dim", "768", "--metric", "Cosine"],
    "1m128": ["--n", "1000000", "--dim", "128", "--metric", "L2"],
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def bench_args(shape, a):
    import bench
    argv = sys.argv
    sys.argv = ["bench.py"] + SHAPES[shape] + ["--nq", str(a.nq), "--k", str(a.k), "--cache", a.cache]
    try:
        return bench.parse_args()
    finally:
        sys.argv = argv


def bkt_keys(x, nodes, root, q, levels, cosine, chunk=1024):
    """Greedy descent of one BKT tree: key = child indices along the path, 5 bits per level"""
    import torch
    keys = []
    j = torch.arange(32, device=q.device)
    for s in range(0, q.shape[0], chunk):
        qq = q[s:s + chunk]
        node = torch.full((qq.shape[0],), root, dtype=torch.long, device=q.device)
        alive = torch.ones(qq.shape[0], dtype=torch.bool, device=q.device)
        key = torch.zeros(qq.shape[0], dtype=torch.long, device=q.device)
        for _ in range(levels):
            cs, ce = nodes[node, 1].long(), nodes[node, 2].long()
            alive &= cs >= 0
            cnt = torch.where(alive, (ce - cs).clamp(0, 32), torch.zeros_like(cs))
            valid = j[None, :] < cnt[:, None]
            child = (cs[:, None] + j[None, :]).clamp(0, nodes.shape[0] - 1)
            centre = nodes[child, 0].long().clamp(0, x.shape[0] - 1)
            v = x[centre]                                     # [chunk, 32, dim]
            if cosine:
                d = -(v @ qq[:, :, None]).squeeze(2)
            else:
                d = ((v - qq[:, None, :]) ** 2).sum(2)
            d = torch.where(valid, d, torch.full_like(d, float("inf")))
            best = d.argmin(1)
            key = key * 32 + torch.where(alive, best, torch.zeros_like(best))
            node = torch.where(alive, cs + best, node)
        keys.append(key)
    return torch.cat(keys)


def run_shape(shape, a):
    import numpy as np
    import torch
    import bench
    import reflib
    from sptag_b200 import B200Index

    dev = torch.device("cuda", 0)
    args = bench_args(shape, a)
    folder = bench.ensure_index(args, 0, dev)
    d_q = bench.gen_data(args, args.nq, args.seed + 7, dev).to(torch.float32).contiguous()
    files = reflib.IndexFiles(folder)
    if files.algo != "BKT":
        raise SystemExit("query_order_bench.py: BKT indexes only")
    x = torch.from_numpy(np.ascontiguousarray(files.vectors)).to(dev).float()
    nodes = torch.from_numpy(np.ascontiguousarray(files.nodes)).to(dev)
    root = int(files.tree_starts[0])
    orders = {"a_batch": torch.arange(args.nq, device=dev)}
    distinct = {}
    for lv in a.levels:
        key = bkt_keys(x, nodes, root, d_q, lv, args.metric == "Cosine")
        orders["b_tree%d" % lv] = torch.sort(key, stable=True).indices
        distinct["b_tree%d" % lv] = int(torch.unique(key).numel())
    g = torch.Generator(device="cpu")
    g.manual_seed(a.shuffle_seed)
    orders["c_shuffle"] = torch.randperm(args.nq, generator=g).to(dev)
    del x, nodes
    torch.cuda.empty_cache()

    idx = B200Index.load(folder, device=0)
    idx.set_param("MaxCheck", args.maxcheck)
    stream = torch.cuda.current_stream()
    bufs = {}
    for name, perm in orders.items():
        bufs[name] = (d_q[perm].contiguous(), torch.empty((args.nq, args.k), dtype=torch.int32, device=dev),
                      torch.empty((args.nq, args.k), dtype=torch.float32, device=dev))

    def step(name):
        q, ids, dists = bufs[name]
        idx.search_device(q.data_ptr(), args.nq, args.k, ids.data_ptr(), dists.data_ptr(), 0, stream.cuda_stream)

    names = list(orders)
    for name in names:
        for _ in range(a.warmup):
            step(name)
    torch.cuda.synchronize()
    res = {n: {"qps": [], "kernel_ms": []} for n in names}
    for r in range(a.rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                step(name)
            e1.record(stream)
            e1.synchronize()
            res[name]["qps"].append(args.nq * a.steps / (e0.elapsed_time(e1) / 1000.0))
            res[name]["kernel_ms"].append(idx.last_kernel_ms())

    # results back in batch order: the same ids and distance bits as the batch-order search
    ref_ids, ref_d = bufs["a_batch"][1].cpu().numpy(), bufs["a_batch"][2].cpu().numpy()
    rows = []
    for name in names:
        perm = orders[name].cpu().numpy()
        ids = np.empty_like(ref_ids)
        dists = np.empty_like(ref_d)
        ids[perm] = bufs[name][1].cpu().numpy()
        dists[perm] = bufs[name][2].cpu().numpy()
        q = sorted(res[name]["qps"])
        km = sorted(res[name]["kernel_ms"])
        rows.append({"order": name, "qps_median": round(q[len(q) // 2], 1), "qps_min": round(q[0], 1),
                     "qps_max": round(q[-1], 1), "kernel_ms_median": round(km[len(km) // 2], 3),
                     "kernel_ms_min": round(km[0], 3), "kernel_ms_max": round(km[-1], 3),
                     "distinct_keys": distinct.get(name),
                     "identical_to_batch_order": bool(np.array_equal(ids, ref_ids) and
                                                      np.array_equal(dists.view(np.int32), ref_d.view(np.int32)))})
    idx.close()
    torch.cuda.empty_cache()
    return {"shape": shape, "workload": "%d x %d %s, batch %d, k=%d, MaxCheck %d" % (
        args.n, args.dim, args.metric, args.nq, args.k, args.maxcheck), "card": card(), "rounds": a.rounds,
        "steps_per_round": a.steps, "orders": rows}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="c2,1m128")
    ap.add_argument("--levels", default="2,3", help="key depths of the tree-ordered settings")
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4, help="timed rounds, the order of the settings reversed every other round")
    ap.add_argument("--steps", type=int, default=3, help="batches per timed round")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shuffle-seed", type=int, default=99)
    ap.add_argument("--cache", default=os.environ.get("SPTAG_B200_CACHE", "/tmp/sptag_b200_cache"))
    a = ap.parse_args()
    a.levels = [int(v) for v in a.levels.split(",")]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("query_order_bench.py needs a GPU")
    for shape in a.shapes.split(","):
        if shape not in SHAPES:
            raise SystemExit("unknown shape %s (%s)" % (shape, ", ".join(SHAPES)))
        t0 = time.time()
        line = run_shape(shape, a)
        line["wall_s"] = round(time.time() - t0, 1)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    sys.exit(main())
