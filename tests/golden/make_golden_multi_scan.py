"""Golden fixtures for the multi-index scan (MultiIndexScan, src/Core/MultiIndexScan.cpp) -- TEST INFRASTRUCTURE.

Builds small BKT index sets with the UNMODIFIED REFERENCE (oracle/_ref/libsptag_ref.so, one build thread, so that a
second run writes byte-identical files).  The indexes of a set are views of the same items, so they share one id space:

  views3   1500 items: float L2 16-d, float Cosine 24-d and int8 L2 12-d projections of one latent space
  dups     500 items, a fifth of them exact copies of another item in every view (equal scores), 10% tombstoned in
           the first index (the scan searches deleted vectors too); float L2 12-d + int8 L2 8-d
  bfs      600 items, float L2 16-d with EnableBfs 2 + float Cosine 20-d
  views5   300 items in 5 views and
  views9   300 items in 9 views (float L2 / float Cosine alternating, the last one int8 L2): the score's blocks of 4 and
           8 rounded products, which fewer than 4 indexes never reach

then runs tests/cpp/multi_scan_ref.cpp (MultiIndexScan::Init + Next until false per query) for every parameter set of
PARAMS that applies to the set, and records each index's own Next(1) stream (GetIterator(target, true)) as far as the
scans of the set read it (tests/oracle_multi_scan.py replays them), plus one entry more where a stream ends.

tests/golden/multi_scan/<set>.npz holds: n (indexes), file:<i>:<name> (the bytes of index i's folder), queries_<i>,
and per parameter set p: k_p, term_p, limit_p, weights_p (empty = NULL, rankFunc), ids_p / scores_p [nq x k],
counts_p [nq]; sids / sdists [n x nq x L] and slen [n x nq] (results in the stream; < L: the iterator returned nothing
after them).
Run (where oracle/_ref exists):  python tests/golden/make_golden_multi_scan.py
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(HERE, "multi_scan")
NQ = 16
BUILD = "NeighborhoodSize=16;RefineIterations=1;CEF=64;TPTNumber=4;BKTLeafSize=8"

# name: (k, term_cond, search_limit, weights or None); weights are per index of a 3- or 2-index set
W5 = (1.0, 0.5, 2.0, 0.25, 0.01)
W9 = (1.0, 0.5, 2.0, 0.25, 1.5, 0.75, 3.0, 0.125, 0.01)
PARAMS = {
    "drops": (10, 12, 100000, {3: (1.0, 2.0, 0.001), 2: (1.0, 0.01), 5: W5, 9: W9}),
    "sum": (10, 12, 100000, None),
    "limit": (8, -1, 90, {3: (0.5, 1.0, 0.002), 2: (2.0, 0.02), 5: W5[::-1], 9: W9[::-1]}),
    "term0": (5, 0, 1000, {3: (1.0, 1.0, 1.0), 2: (1.0, 1.0)}),
    "k1": (1, 25, 400, {3: (0.25, 4.0, 0.003), 2: (0.5, 0.05), 5: W5, 9: W9}),
    "k40": (40, 30, 600, {3: (1.0, 0.0, 0.001), 2: (0.0, 1.0)}),
    "int": (6, 150, 300, {3: (0.0, 0.0, 1.0), 2: (0.0, 1.0)}),  # int8 L2 alone: integer scores, ties at eviction
    "exhaust": (12, -1, -1, {3: (1.0, 2.0, 0.001), 2: (1.0, 0.01)}),
}
SET_PARAMS = {
    "views3": ("drops", "sum", "limit", "term0", "k1", "k40", "int"),
    "dups": ("drops", "sum", "limit", "term0", "k1", "k40", "int", "exhaust"),
    "bfs": ("drops", "sum", "limit", "k1", "exhaust"),
    "views5": ("drops", "sum", "limit", "k1"),
    "views9": ("drops", "sum", "limit", "k1"),
}


def views(n, seed, specs, dup_frac=0.0):
    """Items of a latent space seen through one projection per spec (dim, dtype); with dup_frac, that share of the items
    copies another item.  Also NQ query items.  -> ([rows per view], [queries per view])"""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n + NQ, 6)).astype(np.float32)
    if dup_frac:
        dst = rng.choice(np.arange(1, n), int(n * dup_frac), replace=False)
        z[dst] = z[rng.integers(0, n, dst.shape[0])]
    rows, qs = [], []
    for dim, dtype in specs:
        a = rng.standard_normal((6, dim)).astype(np.float32)
        x = z @ a + 0.05 * rng.standard_normal((n + NQ, dim)).astype(np.float32)
        if dtype == np.int8:
            x = np.clip(np.rint(x * 2.0), -127, 127).astype(np.int8)  # coarse: equal distances are common
        x = np.ascontiguousarray(x)
        rows.append(x[:n])
        qs.append(np.ascontiguousarray(x[n:]))
    return rows, qs


def sets():
    """-> {name: [(rows, queries, metric, extra ini params, tombstones)]}"""
    out = {}
    r, q = views(1500, 11, [(16, np.float32), (24, np.float32), (12, np.int8)])
    out["views3"] = [(r[0], q[0], "L2", {}, None), (r[1], q[1], "Cosine", {}, None), (r[2], q[2], "L2", {}, None)]
    r, q = views(500, 12, [(12, np.float32), (8, np.int8)], dup_frac=0.2)
    dead = np.random.default_rng(13).choice(500, 50, replace=False).astype(np.int32)
    out["dups"] = [(r[0], q[0], "L2", {}, dead), (r[1], q[1], "L2", {}, None)]
    r, q = views(600, 14, [(16, np.float32), (20, np.float32)])
    out["bfs"] = [(r[0], q[0], "L2", {"EnableBfs": 2}, None), (r[1], q[1], "Cosine", {}, None)]
    for n, seed in ((5, 15), (9, 16)):
        specs = [(8 + 2 * i, np.float32) for i in range(n - 1)] + [(8, np.int8)]
        r, q = views(300, seed, specs)
        out["views%d" % n] = [(r[i], q[i], "Cosine" if i % 2 else "L2", {}, None) for i in range(n - 1)] + \
            [(r[n - 1], q[n - 1], "L2", {}, None)]
    return out


def build_folder(rows, metric, extra, dead, folder):
    import reflib
    x = rows
    if metric == "Cosine":  # the reference expects normalised rows for Cosine
        x = reflib.normalize_rows(rows.astype(np.float32)).astype(np.float32)
    # the BKT tree draws its centres with std::rand, whose state the previous graph build seeded from clock()
    ctypes.CDLL(None).srand(7)
    idx = reflib.RefIndex.build("BKT", x, metric, threads=1, params=BUILD)
    for k, v in extra.items():
        idx.set_param(k, v)
    if dead is not None:
        idx.delete(dead)
    idx.save(folder)


def folder_files(folder):
    return {name: np.fromfile(os.path.join(folder, name), np.uint8) for name in sorted(os.listdir(folder))}


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "multi_scan_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def run(drv, folders, qfiles, nq, k, term, limit, weights, stream_len, tmp):
    pre = os.path.join(tmp, "ms")
    w = "sum" if weights is None else ",".join(repr(float(x)) for x in weights)
    args = [drv, str(nq), pre, str(k), str(term), str(limit), w, str(stream_len), "1"]
    for f, qf in zip(folders, qfiles):
        args += [f, qf]
    subprocess.check_call(args)
    out = dict(ids=np.fromfile(pre + ".ids", np.int32).reshape(nq, k),
               scores=np.fromfile(pre + ".scores", np.float32).reshape(nq, k),
               counts=np.fromfile(pre + ".counts", np.int32))
    if stream_len:
        n = len(folders)
        out["sids"] = np.fromfile(pre + ".sids", np.int32).reshape(n, nq, stream_len)
        out["sdists"] = np.fromfile(pre + ".sdists", np.float32).reshape(n, nq, stream_len)
        out["slen"] = np.fromfile(pre + ".slen", np.int32).reshape(n, nq)
    return out


def main():
    import oracle_multi_scan as oms
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "multi_scan_ref")
        build_driver(drv)
        for name, members in sets().items():
            out = {"n": np.int32(len(members))}
            folders, qfiles = [], []
            for i, (rows, q, metric, extra, dead) in enumerate(members):
                folder = os.path.join(tmp, "%s_%d" % (name, i))
                build_folder(rows, metric, extra, dead, folder)
                if metric == "Cosine":
                    import reflib
                    q = reflib.normalize_rows(q.astype(np.float32)).astype(np.float32)
                qf = os.path.join(tmp, "%s_%d.q" % (name, i))
                q.tofile(qf)
                folders.append(folder)
                qfiles.append(qf)
                out["queries_%d" % i] = q
                for fname, data in folder_files(folder).items():
                    out["file:%d:%s" % (i, fname)] = data
            n_items = members[0][0].shape[0]
            streams = run(drv, folders, qfiles, NQ, 1, 0, 0, [1.0] * len(members), n_items + 1, tmp)
            fx = oms.Fixture(out, streams)
            need = np.zeros((len(members), NQ), np.int64)
            for p in SET_PARAMS[name]:
                k, term, limit, wsets = PARAMS[p]
                weights = None if wsets is None else wsets[len(members)]
                r = run(drv, folders, qfiles, NQ, k, term, limit, weights, 0, tmp)
                out["k_" + p], out["term_" + p], out["limit_" + p] = np.int32(k), np.int32(term), np.int32(limit)
                out["weights_" + p] = np.array([] if weights is None else weights, np.float32)
                out["ids_" + p], out["scores_" + p], out["counts_" + p] = r["ids"], r["scores"], r["counts"]
                for q in range(NQ):
                    res = oms.scan(fx, q, k, term, limit, weights)
                    need[:, q] = np.maximum(need[:, q], res["used"])
            # keep each stream as far as a scan read it; where it ended there, one entry more shows the end
            length = int(need.max()) + 1
            out["sids"] = streams["sids"][:, :, :length]
            out["sdists"] = streams["sdists"][:, :, :length]
            out["slen"] = np.minimum(streams["slen"], length).astype(np.int32)
            path = os.path.join(OUT, name + ".npz")
            np.savez_compressed(path, **out)
            print("%s: %d bytes, streams of %d" % (path, os.path.getsize(path), length))


if __name__ == "__main__":
    sys.exit(main())
