#!/usr/bin/env python
"""visited_bench.py -- the hashed visited set (B200.VisitedSet = 1) against the per-slot bitmap (B200.VisitedSet = 0).

For each shape, two handles are loaded on the same index folder, one per mode, and timed in alternating rounds in the
same process: resident-query QPS and kernel time (CUDA events; the hashed set's time includes its re-run launch),
B200.ScratchBytes, the overflow count of a blocking search, and the clearing work of the hashed set.  Both modes'
ids, distances and WorkSpace counters are written as .npy files and compared bit for bit.  The card's name and power
limit are read in the same call.

The clearing work is derived, not timed: a query clears one table position per id it inserted, reading the position
from its log (4 B) and storing a zero (4 B); every inserted id also had a distance computed, so the per-query count of
distances bounds it from above.

Shapes (indexes built and cached by bench.py's builder, under --cache):
    c2     BKT 1M x 768 float32 cosine        (BASELINE config 2, bench.py's default)
    1m128  BKT 1M x 128 float32 L2            (512-byte rows: the fast path)
    c4     BKT 50M x 100 int8 -> OPQ 50 codes (BASELINE config 4; the bitmap scratch is about 28 GB)

    python tools/visited_bench.py --shapes c2,1m128,c4 --out /tmp/visited_bench
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

SHAPES = {
    "c2": ["--n", "1000000", "--dim", "768", "--metric", "Cosine"],
    "1m128": ["--n", "1000000", "--dim", "128", "--metric", "L2"],
    "c4": ["--n", "50000000", "--dim", "100", "--metric", "L2", "--quantizer", "opq", "--pq-m", "50", "--raw-type", "int8"],
}
MODES = (("bitmap", 0), ("hash", 1))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def bench_args(shape, a):
    import bench
    argv = sys.argv
    sys.argv = ["bench.py"] + SHAPES[shape] + ["--nq", str(a.nq), "--k", str(a.k), "--maxcheck", str(a.maxcheck),
                                               "--cache", a.cache]
    try:
        return bench.parse_args()
    finally:
        sys.argv = argv


def run_shape(shape, a, out_dir):
    import numpy as np
    import torch
    import bench
    from sptag_b200 import B200Index, capi

    dev = torch.device("cuda", 0)
    args = bench_args(shape, a)
    folder = bench.ensure_index(args, 0, dev)
    qdtype = torch.int8 if args.raw_type == "int8" else torch.float32
    d_q = bench.gen_data(args, args.nq, args.seed + 7, dev).to(qdtype).contiguous()
    h_q = d_q.cpu().numpy()
    torch.cuda.empty_cache()

    idx = {}
    for mode, v in MODES:
        idx[mode] = B200Index.load(folder, device=0)
        idx[mode].set_param("MaxCheck", args.maxcheck)
        idx[mode].set_param("B200.VisitedSet", v)
    d_ids = torch.empty((args.nq, args.k), dtype=torch.int32, device=dev)
    d_dists = torch.empty((args.nq, args.k), dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream()

    def step(mode):
        idx[mode].search_device(d_q.data_ptr(), args.nq, args.k, d_ids.data_ptr(), d_dists.data_ptr(), 0,
                                stream.cuda_stream)

    res = {m: {"qps": [], "kernel_ms": []} for m, _ in MODES}
    for mode, _ in MODES:
        for _ in range(a.warmup):
            step(mode)
    torch.cuda.synchronize()
    for r in range(a.rounds):
        for mode, _ in (MODES if r % 2 == 0 else MODES[::-1]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            kms = []
            e0.record(stream)
            for _ in range(a.steps):
                step(mode)
            e1.record(stream)
            e1.synchronize()
            kms.append(idx[mode].last_kernel_ms())
            res[mode]["qps"].append(args.nq * a.steps / (e0.elapsed_time(e1) / 1000.0))
            res[mode]["kernel_ms"].append(kms[-1])

    # blocking searches: outputs, counters and the overflow count of each mode
    outs = {}
    for mode, _ in MODES:
        ids, dists, stats = idx[mode].search(h_q, args.k, want_stats=True)
        outs[mode] = (ids, dists, stats)
        res[mode]["overflows"] = int(idx[mode].get_param("B200.LastVisitedOverflows"))
        res[mode]["scratch_bytes"] = int(idx[mode].get_param("B200.ScratchBytes"))
        for name, arr in zip(("ids", "dists", "stats"), outs[mode]):
            np.save(os.path.join(out_dir, "%s_%s_%s.npy" % (shape, mode, name)), arr)
    b, h = outs["bitmap"], outs["hash"]
    identical = (np.array_equal(b[0], h[0]) and np.array_equal(b[1].view(np.int32), h[1].view(np.int32))
                 and np.array_equal(b[2], h[2]))

    ndist = float(h[2][:, capi.ST_NDIST].mean())
    for m in idx.values():
        m.close()
    torch.cuda.empty_cache()
    summary = {}
    for mode, _ in MODES:
        q = sorted(res[mode]["qps"])
        summary[mode] = {"qps_median": q[len(q) // 2], "qps_min": q[0], "qps_max": q[-1],
                         "kernel_ms_median": sorted(res[mode]["kernel_ms"])[len(q) // 2],
                         "scratch_bytes": res[mode]["scratch_bytes"], "overflows": res[mode]["overflows"]}
    return {"shape": shape, "workload": "%d x %d %s %s%s, batch %d, k=%d, MaxCheck=%d" % (
                args.n, args.dim, args.metric, args.raw_type,
                "" if args.quantizer == "none" else " -> %s %d codes" % (args.quantizer, args.pq_m),
                args.nq, args.k, args.maxcheck),
            "card": card(), "rounds": a.rounds, "steps_per_round": a.steps,
            "bitmap": summary["bitmap"], "hash": summary["hash"],
            "hash_over_bitmap_qps": summary["hash"]["qps_median"] / summary["bitmap"]["qps_median"],
            "identical_ids_dists_stats": bool(identical),
            "clear_bytes_per_query_upper_bound": 8.0 * ndist,
            "clear_bytes_per_batch_upper_bound": 8.0 * ndist * args.nq,
            "outputs": out_dir}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="c2,1m128,c4")
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--maxcheck", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=4, help="timed rounds per mode, alternating which mode goes first")
    ap.add_argument("--steps", type=int, default=5, help="batches per timed round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cache", default=os.environ.get("SPTAG_B200_CACHE", "/tmp/sptag_b200_cache"))
    ap.add_argument("--out", default=None, help="directory for the .npy outputs (default: a new temporary directory)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("visited_bench.py needs a GPU")
    out_dir = a.out or tempfile.mkdtemp(prefix="visited_bench_")
    os.makedirs(out_dir, exist_ok=True)
    for shape in a.shapes.split(","):
        if shape not in SHAPES:
            raise SystemExit("unknown shape %s (%s)" % (shape, ", ".join(SHAPES)))
        t0 = time.time()
        line = run_shape(shape, a, out_dir)
        line["wall_s"] = round(time.time() - t0, 1)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    sys.exit(main())
