#!/usr/bin/env python
"""bfs_bench.py -- what breadth-first tree seeding (EnableBfs, BKTree.h:703-758) costs and buys on the device.

For each shape one handle is loaded, and every EnableBfs x MaxCheck setting is timed in the same process, the settings'
order reversed on every other round: resident-query QPS (CUDA events around `--steps` batches of search_device) and
kernel time (the handle's last launch).  A blocking search per setting gives recall@k against exact search (the
builder's exact_topk), the mean distance evaluations (ST_NDIST) and the mean checked leaves (ST_CHECKED).  Where
oracle/_ref is built, the unmodified reference searches a sample of the queries at the same EnableBfs and MaxCheck and
ids and distance bits are compared.  The card's name and power limit are read in the same call.

EnableBfs != 0 runs the generic-dimension kernels (the 128- and 768-d specialisations are built without it), so part
of any gap to EnableBfs = 0 is that routing, not the seeding.

Shapes (indexes built and cached by bench.py's builder, under --cache):
    1m128  BKT 1M x 128 float32 L2
    c2     BKT 1M x 768 float32 cosine (BASELINE config 2, bench.py's default)

    python tools/bfs_bench.py --shapes 1m128,c2 --bfs 0,1,2,4 --maxchecks 2048,8192
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
    "1m128": ["--n", "1000000", "--dim", "128", "--metric", "L2"],
    "c2": ["--n", "1000000", "--dim", "768", "--metric", "Cosine"],
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


def reference_check(folder, h_q, ids, dists, bfs, mc, k, sample):
    """ids / distance bits of the reference on the first `sample` queries at the same settings; None without oracle/_ref"""
    import numpy as np
    import reflib
    if not reflib.have_ref():
        return None
    r = reference_check.cache.get(folder)
    if r is None:
        r = reference_check.cache[folder] = reflib.RefIndex.load(folder)
    r.set_param("EnableBfs", bfs)
    r.set_param("MaxCheck", mc)
    ri, rd, _ = r.search(np.ascontiguousarray(h_q[:sample]), k)
    return bool(np.array_equal(ri, ids[:sample]) and np.array_equal(rd.view(np.int32), dists[:sample].view(np.int32)))


reference_check.cache = {}


def run_shape(shape, a):
    import numpy as np
    import torch
    import bench
    from sptag_b200 import B200Index, capi
    from tools import gpu_index_builder as gib

    dev = torch.device("cuda", 0)
    args = bench_args(shape, a)
    folder = bench.ensure_index(args, 0, dev)
    d_q = bench.gen_data(args, args.nq, args.seed + 7, dev).to(torch.float32).contiguous()
    h_q = d_q.cpu().numpy()
    # exact neighbours: the builder's exact top-k on the device (float32 scores)
    import reflib
    files = reflib.IndexFiles(folder)
    x = torch.from_numpy(np.ascontiguousarray(files.vectors)).to(dev)
    exact = gib.exact_topk(x, d_q, args.k, args.metric)
    del x
    torch.cuda.empty_cache()

    idx = B200Index.load(folder, device=0)
    d_ids = torch.empty((args.nq, args.k), dtype=torch.int32, device=dev)
    d_dists = torch.empty((args.nq, args.k), dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream()
    settings = [(b, m) for m in a.maxchecks for b in a.bfs]

    def use(s):
        idx.set_param("EnableBfs", s[0])
        idx.set_param("MaxCheck", s[1])

    def step():
        idx.search_device(d_q.data_ptr(), args.nq, args.k, d_ids.data_ptr(), d_dists.data_ptr(), 0, stream.cuda_stream)

    res = {s: {"qps": [], "kernel_ms": []} for s in settings}
    for s in settings:
        use(s)
        for _ in range(a.warmup):
            step()
    torch.cuda.synchronize()
    for r in range(a.rounds):
        for s in (settings if r % 2 == 0 else settings[::-1]):
            use(s)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                step()
            e1.record(stream)
            e1.synchronize()
            res[s]["qps"].append(args.nq * a.steps / (e0.elapsed_time(e1) / 1000.0))
            res[s]["kernel_ms"].append(idx.last_kernel_ms())

    rows = []
    for s in settings:
        use(s)
        ids, dists, stats = idx.search(h_q, args.k, want_stats=True)
        recall = float(np.mean([len(set(ids[i].tolist()) & set(exact[i].tolist())) for i in range(args.nq)]) / args.k)
        q = sorted(res[s]["qps"])
        rows.append({"enable_bfs": s[0], "max_check": s[1], "qps_median": q[len(q) // 2], "qps_min": q[0],
                     "qps_max": q[-1], "kernel_ms_median": sorted(res[s]["kernel_ms"])[len(q) // 2],
                     "recall_at_k": recall, "mean_ndist": float(stats[:, capi.ST_NDIST].mean()),
                     "mean_checked_leaves": float(stats[:, capi.ST_CHECKED].mean()),
                     "reference_identical": reference_check(folder, h_q, ids, dists, s[0], s[1], args.k, a.ref_sample)})
    idx.close()
    reference_check.cache.clear()
    torch.cuda.empty_cache()
    return {"shape": shape, "workload": "%d x %d %s, batch %d, k=%d" % (args.n, args.dim, args.metric, args.nq, args.k),
            "card": card(), "rounds": a.rounds, "steps_per_round": a.steps, "reference_sample": a.ref_sample,
            "settings": rows}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="1m128,c2")
    ap.add_argument("--bfs", default="0,1,2,4")
    ap.add_argument("--maxchecks", default="2048,8192")
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4, help="timed rounds per setting, the order reversed every other round")
    ap.add_argument("--steps", type=int, default=3, help="batches per timed round")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-sample", type=int, default=200, help="queries checked against oracle/_ref per setting")
    ap.add_argument("--cache", default=os.environ.get("SPTAG_B200_CACHE", "/tmp/sptag_b200_cache"))
    a = ap.parse_args()
    a.bfs = [int(v) for v in a.bfs.split(",")]
    a.maxchecks = [int(v) for v in a.maxchecks.split(",")]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bfs_bench.py needs a GPU")
    for shape in a.shapes.split(","):
        if shape not in SHAPES:
            raise SystemExit("unknown shape %s (%s)" % (shape, ", ".join(SHAPES)))
        t0 = time.time()
        line = run_shape(shape, a)
        line["wall_s"] = round(time.time() - t0, 1)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    sys.exit(main())
