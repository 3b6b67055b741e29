#!/usr/bin/env python
"""spann_pq_bench.py -- SPANN search on a PQ-quantized index (code rows in HBM, SDC / ADC look-ups) next to the same rows
unquantized.

Data: tools/spann_bench.py's clustered float32 rows and queries.  Two SPANN indexes are built with the unmodified
reference on the host (tests/cpp/spann_ref and tests/cpp/spann_pq_ref, built by __graft_entry__.build() where the
reference sources exist; they link oracle/_ref only): one over the raw rows, one over their PQ codes (M = --m
sub-vectors of 256 codewords, trained by tests/reflib.train_quantizer, codes by the reference's QuantizeVector).  Then,
in one call, with batch --nq, K = --k and SearchInternalResultNum --internal:
  device QPS   sptag_b200_spann_search on the raw handle, the PQ handle in SDC and the PQ handle in ADC, --steps blocking
               calls each (host buffers, H2D and D2H included) after --warmup calls, the three alternated --repeats times;
               the median and the spread per configuration
  PostingBytes of both handles
  recall@10    of every configuration against exact L2 search on the raw rows (numpy)
  parity       ids and distance bits of the first --sample queries against the reference searching the same folder
The card's name and power limit are read in the same call.  Writes nothing in the tree: the indexes go to --work (a
temporary directory unless given; folders already built there are reused).

    python tools/spann_pq_bench.py --n 200000 --dim 128 --m 32 --nq 10000 --k 10
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
RAW_DRIVER = os.path.join(ROOT, "tests", "cpp", "spann_ref")
PQ_DRIVER = os.path.join(ROOT, "tests", "cpp", "spann_pq_ref")


def set_internal(folder, internal):
    """SearchInternalResultNum in the folder's indexloader.ini (the reference and the device read it from there)"""
    path = os.path.join(folder, "indexloader.ini")
    with open(path) as fh:
        lines = fh.read().split("\n")
    lines = ["SearchInternalResultNum=%d" % internal if ln.startswith("SearchInternalResultNum=") else ln for ln in lines]
    with open(path, "w") as fh:
        fh.write("\n".join(lines))


def exact_top(x, q, k, chunk=1000):
    """exact L2 top-k ids on the raw rows"""
    xn = (x.astype(np.float64) ** 2).sum(1)
    out = np.empty((len(q), k), np.int64)
    for i in range(0, len(q), chunk):
        d = xn[None, :] - 2.0 * (q[i:i + chunk].astype(np.float64) @ x.T.astype(np.float64))
        part = np.argpartition(d, k, axis=1)[:, :k]
        order = np.argsort(np.take_along_axis(d, part, 1), axis=1)
        out[i:i + chunk] = np.take_along_axis(part, order, 1)
    return out


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / truth.shape[1] for a, b in zip(ids, truth)]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--internal", type=int, default=64)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=1000)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--work", default=None)
    a = ap.parse_args()
    for drv in (RAW_DRIVER, PQ_DRIVER):
        if not os.path.exists(drv):
            sys.exit("%s is missing: run __graft_entry__.build() where the reference sources exist" % drv)
    import reflib
    from spann_bench import card, data
    from sptag_b200 import capi
    x, q = data(a.n, a.dim, a.nq)
    res = {"card": card(), "n": a.n, "dim": a.dim, "m": a.m, "nq": a.nq, "k": a.k, "internal": a.internal,
           "metric": "L2", "dtype": "f32", "host_threads": a.threads}
    tmp = tempfile.TemporaryDirectory()
    work = a.work or tmp.name
    os.makedirs(work, exist_ok=True)
    raw_dir, pq_dir = os.path.join(work, "raw"), os.path.join(work, "pq_m%d" % a.m)
    xf, qf = os.path.join(work, "x.bin"), os.path.join(work, "q.bin")
    q.tofile(qf)
    if not os.path.exists(os.path.join(raw_dir, "indexloader.ini")):
        x.tofile(xf)
        t0 = time.perf_counter()
        subprocess.check_call([RAW_DRIVER, "build", raw_dir, "Float", "L2", "0", str(a.n), str(a.dim), xf, "1", "1",
                               str(a.threads)])
        res["reference_build_raw_s"] = round(time.perf_counter() - t0, 1)
    if not os.path.exists(os.path.join(pq_dir, "indexloader.ini")):
        qpath, cf = os.path.join(work, "quantizer_m%d.bin" % a.m), os.path.join(work, "codes_m%d.bin" % a.m)
        reflib.train_quantizer(x, m=a.m, ks=256, seed=7, iters=4).write(qpath)
        reflib.RefQuantizer(qpath).encode(x).tofile(cf)
        t0 = time.perf_counter()
        subprocess.check_call([PQ_DRIVER, "build", pq_dir, qpath, "0", str(a.n), str(a.m), cf, "1", str(a.threads)])
        res["reference_build_pq_s"] = round(time.perf_counter() - t0, 1)
    for folder in (raw_dir, pq_dir):
        set_internal(folder, a.internal)
    m = min(a.sample, a.nq)
    qs = os.path.join(work, "qs.bin")
    q[:m].tofile(qs)
    ref = {}
    pre = os.path.join(work, "r")
    subprocess.check_call([RAW_DRIVER, "search", raw_dir, qs, str(m), str(a.k), pre, str(a.threads)])
    ref["raw"] = (np.fromfile(pre + ".ids", np.int32).reshape(m, a.k), np.fromfile(pre + ".dists", np.int32).reshape(m, a.k))
    for adc, name in ((0, "sdc"), (1, "adc")):
        subprocess.check_call([PQ_DRIVER, "search", pq_dir, qs, str(m), str(a.k), str(adc), pre, str(a.threads)])
        ref[name] = (np.fromfile(pre + ".ids", np.int32).reshape(m, a.k), np.fromfile(pre + ".dists", np.int32).reshape(m, a.k))

    raw = capi.B200SpannIndex.load(raw_dir, 0)
    pq = capi.B200SpannIndex.load(pq_dir, 0)
    res["posting_bytes_raw"] = int(raw.get_param("PostingBytes"))
    res["posting_bytes_pq"] = int(pq.get_param("PostingBytes"))
    configs = (("raw", raw, None), ("sdc", pq, 0), ("adc", pq, 1))
    times = {name: [] for name, _, _ in configs}
    out = {}
    for _ in range(a.repeats):
        for name, h, adc in configs:
            if adc is not None:
                h.set_param("EnableADC", adc)
            for _ in range(a.warmup):
                h.search(q, a.k)
            t0 = time.perf_counter()
            for _ in range(a.steps):
                ids, dists = h.search(q, a.k)
            times[name].append((time.perf_counter() - t0) / a.steps)
            out[name] = (ids, dists)
    for name, h, adc in configs:
        if adc is not None:
            h.set_param("EnableADC", adc)
        _, _, stats = h.search(q, a.k, want_stats=True)
        res["mean_distances_" + name] = float(stats[:, 2].mean())
    raw.close()
    pq.close()
    tmp.cleanup()
    truth = exact_top(x, q, a.k)
    for name in times:
        t = times[name]
        ids, dists = out[name]
        res[name] = {
            "device_qps": round(a.nq / float(np.median(t)), 1),
            "device_qps_min_max": [round(a.nq / max(t), 1), round(a.nq / min(t), 1)],
            "recall_at_%d" % a.k: round(recall(ids, truth), 5),
            "sample": m,
            "ids_equal": bool(np.array_equal(ids[:m], ref[name][0])),
            "dist_bits_equal": bool(np.array_equal(dists[:m].view(np.int32), ref[name][1])),
        }
    res["repeats"], res["steps"] = a.repeats, a.steps
    print(json.dumps(res))


if __name__ == "__main__":
    main()
