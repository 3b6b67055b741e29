#!/usr/bin/env python
"""row_sketch_bench.py -- what the row sketches (B200.RowSketch) buy, measured on one handle in one process.

For each shape the same batch is searched with B200.RowSketch = 0 (every candidate's row is fetched) and with the
setting under test (--on: -1 auto, the default, or 1 forced), alternating within every round.  Reported per setting:
median / min / max QPS (CUDA events around --steps batches of search_device), kernel ms of the handle's last launch,
the share of distance computations whose row was not fetched (B200.RowsSkipped over ST_NDIST), the bytes a query really
requests (sketches + fetched rows; graph rows and tree nodes are the same in both settings and left out) with their
rate, and whether ids, distance bits and all eight per-query counters are identical in the two settings.
The card's name and power limit are read in the same call.

Shapes (indexes built and cached by bench.py's builder, under --cache):
    c2      BKT 1M x 768 float32 cosine (bench.py's default)    c2l2   the same rows, L2
    1m512   BKT 1M x 512 float32 L2 (2 KB rows: the edge of auto)
    1m128   BKT 1M x 128 float32 L2 (auto is off)

    python tools/row_sketch_bench.py --shapes c2,c2l2,1m512,1m128
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
    "c2l2": ["--n", "1000000", "--dim", "768", "--metric", "L2"],
    "1m512": ["--n", "1000000", "--dim", "512", "--metric", "L2"],
    "1m128": ["--n", "1000000", "--dim", "128", "--metric", "L2"],
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def run_shape(shape, a):
    import numpy as np
    import torch
    import bench
    from sptag_b200 import B200Index, capi

    argv = sys.argv
    sys.argv = ["bench.py"] + SHAPES[shape] + ["--nq", str(a.nq), "--k", str(a.k), "--cache", a.cache]
    try:
        args = bench.parse_args()
    finally:
        sys.argv = argv
    dev = torch.device("cuda", 0)
    folder = bench.ensure_index(args, 0, dev)
    d_q = bench.gen_data(args, args.nq, args.seed + 7, dev).to(torch.float32).contiguous()
    idx = B200Index.load(folder, device=0)
    idx.set_param("MaxCheck", args.maxcheck)
    stream = torch.cuda.current_stream()
    settings = {"off": 0, "on": a.on}
    out = {n: (torch.empty((args.nq, args.k), dtype=torch.int32, device=dev),
               torch.empty((args.nq, args.k), dtype=torch.float32, device=dev),
               torch.zeros((args.nq, 8), dtype=torch.int32, device=dev)) for n in settings}

    def step(name, stats=False):
        ids, dists, st = out[name]
        idx.set_param("B200.RowSketch", settings[name])
        idx.search_device(d_q.data_ptr(), args.nq, args.k, ids.data_ptr(), dists.data_ptr(), st.data_ptr() if stats else 0,
                          stream.cuda_stream)

    skipped = {}
    for name in settings:          # warm-up, with the counters
        before = int(idx.get_param("B200.RowsSkipped"))
        step(name, stats=True)
        skipped[name] = int(idx.get_param("B200.RowsSkipped")) - before
        for _ in range(a.warmup):
            step(name)
    torch.cuda.synchronize()
    res = {n: {"qps": [], "kernel_ms": []} for n in settings}
    names = list(settings)
    for r in range(a.rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            step(name)             # the parameter change (and, after "off", rebuilding the sketches) stays outside the window
            torch.cuda.synchronize()
            e0.record(stream)
            for _ in range(a.steps):
                step(name)
            e1.record(stream)
            e1.synchronize()
            res[name]["qps"].append(args.nq * a.steps / (e0.elapsed_time(e1) / 1000.0))
            res[name]["kernel_ms"].append(idx.last_kernel_ms())
    same = all(bool(torch.equal(out["off"][i].view(torch.int32), out["on"][i].view(torch.int32))) for i in range(3))
    ndist = float(out["off"][2][:, capi.ST_NDIST].sum().item())
    row_b = ((args.dim * 4 + 15) // 16) * 16
    sk_b = ((args.dim + 15) // 16) * 16 + 16
    rows = []
    for name in names:
        q = sorted(res[name]["qps"])
        km = sorted(res[name]["kernel_ms"])
        sk = skipped[name]
        bytes_q = (ndist - sk) * row_b / args.nq
        if sk:  # every graph candidate's sketch was read once m_Results was full; bounded above by all distances
            bytes_q += ndist * sk_b / args.nq
        med_ms = km[len(km) // 2]
        rows.append({"row_sketch": settings[name], "qps_median": round(q[len(q) // 2], 1), "qps_min": round(q[0], 1),
                     "qps_max": round(q[-1], 1), "kernel_ms_median": round(med_ms, 3), "kernel_ms_min": round(km[0], 3),
                     "kernel_ms_max": round(km[-1], 3), "skipped_share": round(sk / ndist, 4),
                     "row_and_sketch_bytes_per_query": round(bytes_q), "requested_GBps": round(bytes_q * args.nq / med_ms / 1e6, 1)})
    idx.close()
    torch.cuda.empty_cache()
    return {"shape": shape, "workload": "%d x %d %s, batch %d, k=%d, MaxCheck %d" % (
        args.n, args.dim, args.metric, args.nq, args.k, args.maxcheck), "card": card(), "rounds": a.rounds,
        "steps_per_round": a.steps, "identical_ids_dists_stats": same, "settings": rows}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="c2")
    ap.add_argument("--on", type=int, default=-1, choices=[-1, 1], help="the setting compared with 0")
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3, help="batches per timed round")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cache", default=os.environ.get("SPTAG_B200_CACHE", "/tmp/sptag_b200_cache"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("row_sketch_bench.py needs a GPU")
    for shape in a.shapes.split(","):
        if shape not in SHAPES:
            raise SystemExit("unknown shape %s (%s)" % (shape, ", ".join(SHAPES)))
        t0 = time.time()
        line = run_shape(shape, a)
        line["wall_s"] = round(time.time() - t0, 1)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    sys.exit(main())
