#!/usr/bin/env python
"""row_sketch_model.py -- how many row fetches of the BKT graph step could an exact 1-byte-per-dimension bound avoid?

BKT search offers every new graph neighbour to m_Results (BKTIndex.cpp:338-344); a neighbour whose distance is above
m_Results.worst() leaves no trace but the counters, so its 4-byte-per-dimension row need not have been read if a cheaper
test proves `distance > worst`.  This script measures, on the CPU, what such a test could save:

  (a) the share of graph candidates with distance > worst (the ceiling of any such test);
  (b) the share caught by the int8 sketch bound restated below (sketch_rows / lower_bound);
  (c) the bytes per query that follow: every tree node's row, every graph candidate's sketch, and the rows of the
      candidates the bound does not catch, against every row as the search kernels fetch them today.

The search loop is a Python restatement of BKT::Index::Search with MaxCheck, K and the pivots of the index folder; its
count of distance computations per query is checked against the C oracle (tests/reflib.py OracleIndex) on the same
folder, so the logged candidates are the reference's.  `worst` is taken where a kernel would test it: before the
inserts of the candidate's own 32-wide chunk of the graph row (it only decreases, so this is the weaker test).

The sketch of a float32 vector v of `dim` elements (rows and queries alike):
    scale = max|v_i| / 127 (fp32 division; 0 for an all-zero vector)
    s_i   = clamp(rint(v_i / scale), -127, 127) as int8 (0 when scale is 0)
    err   = an upper bound of ||v - scale * s||_2, norm = an upper bound of ||v||_2, nsq = a lower bound of ||v||_2^2
    a vector with a NaN or an infinity has err = +inf and is never skipped
With q = scale_q t + e_q, x = scale_x s + e_x and the exact integer I = sum t_i s_i, Cauchy-Schwarz gives
    q.x <= scale_q scale_x I + norm_q err_x + err_q norm_x + err_q err_x
Cosine: distance = fl(1 - S), S the reference's fp32 sum; |S - q.x| and the last rounding stay below
`margin = REL(dim) * (1 + norm_q norm_x)`, so  1 - ub(q.x) - margin  is a lower bound of the returned distance.
L2: ||q - x||^2 >= nsq_q + nsq_x - 2 ub(q.x), and the reference's fp32 sum of squares is within REL(dim) (norm_q + norm_x)^2.
Every step rounds towards the safe side, as the device intrinsics (__fmul_ru, __fadd_ru, __fsub_rd) would.

    python tools/row_sketch_model.py --n 100000 --dim 768 --metric Cosine --nq 64
"""
import argparse
import heapq
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

F32, F64 = np.float32, np.float64
MAXDIST = F32(np.finfo(np.float32).max / F32(10))
SKETCH_PAD = 16          # bytes after the int8 elements of a sketch row: scale, err, norm, nsq
NORM_LIMIT = F32(1e15)   # above this the reference's own sum can overflow to NaN: never skip


def rel_margin(dim):
    """Relative bound of the reference's fp32 summation error in any of its three trees: dim/4 additions per accumulator in
    the narrowest (SSE) one, the folds, the tail, the product and the final subtraction, each 2^-24, doubled."""
    return F32(F32(dim // 4 + 24) * F32(2.0 ** -23))


# ---- fp32 arithmetic rounded towards one side, exact (the operands' double sum / product error is accounted) ----
def _to_f32(v64, err64, up):
    """float32 nearest to the real number v64 + err64 on the asked side (|err64| far below one ulp of v64)."""
    with np.errstate(over="ignore", invalid="ignore"):
        f = v64.astype(F32)
        f64 = f.astype(F64)
        if up:
            bump = (f64 < v64) | ((f64 == v64) & (err64 > 0))
            return np.where(bump, np.nextafter(f, F32(np.inf)), f)
        bump = (f64 > v64) | ((f64 == v64) & (err64 < 0))
        return np.where(bump, np.nextafter(f, F32(-np.inf)), f)


def _mul(a, b, up):
    v = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)   # exact: 24 x 24 bits
    return _to_f32(v, np.zeros_like(v), up)


def _add(a, b, up):
    a = np.asarray(a, F32).astype(F64)
    b = np.asarray(b, F32).astype(F64)
    with np.errstate(invalid="ignore"):
        s = a + b
        bb = s - a
        e = (a - (s - bb)) + (b - bb)                                     # TwoSum: s + e is the real sum
        e = np.where(np.isfinite(e), e, 0.0)
    return _to_f32(s, e, up)


def mul_ru(a, b): return _mul(a, b, True)
def mul_rd(a, b): return _mul(a, b, False)
def add_ru(a, b): return _add(a, b, True)
def add_rd(a, b): return _add(a, b, False)
def sub_rd(a, b): return _add(a, -np.asarray(b, F32), False)


def _sqrt_f32(v64, up):
    with np.errstate(over="ignore"):
        f = np.sqrt(v64).astype(F32)
    # one more step to the safe side covers the rounding of the double sum and of the square root
    return np.nextafter(f, F32(np.inf if up else -np.inf))


def sketch_rows(x):
    """x float32 [n, dim] -> (s int8 [n, dim], scale, err, norm, nsq float32 [n])."""
    x = np.ascontiguousarray(x, F32)
    finite = np.isfinite(x).all(axis=1)
    xz = np.where(finite[:, None], x, F32(0))
    amax = np.abs(xz).max(axis=1) if x.shape[1] else np.zeros(x.shape[0], F32)
    scale = (amax / F32(127)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(scale[:, None] > 0, xz / np.where(scale > 0, scale, F32(1))[:, None], F32(0)).astype(F32)
    s = np.clip(np.rint(r), -127, 127).astype(np.int8)
    x64 = xz.astype(F64)
    res = x64 - scale.astype(F64)[:, None] * s.astype(F64)
    err = _sqrt_f32((res * res).sum(axis=1), True)
    n2 = (x64 * x64).sum(axis=1)
    norm = _sqrt_f32(n2, True)
    with np.errstate(over="ignore"):
        nsq = np.maximum(np.nextafter(np.nextafter(n2.astype(F32), F32(-np.inf)), F32(-np.inf)), F32(0))
    err = np.where(finite, err, F32(np.inf)).astype(F32)
    return s, scale, err, norm.astype(F32), nsq.astype(F32)


def dot_upper(I, q, r):
    """Upper bound of q.x; I int32 [m], q = (scale, err, norm, nsq) scalars, r = the rows' four arrays [m]."""
    sq, eq, nq, _ = q
    sx, ex, nx, _ = r
    fi = I.astype(F32)                                   # exact below 2^24; larger |I| is rounded up just below
    fi = np.where(fi.astype(F64) < I.astype(F64), np.nextafter(fi, F32(np.inf)), fi)
    ss = np.where(I >= 0, mul_ru(sq, sx), mul_rd(sq, sx))
    ub = mul_ru(ss, fi)
    ub = add_ru(ub, mul_ru(nq, ex))
    ub = add_ru(ub, mul_ru(eq, nx))
    return add_ru(ub, mul_ru(eq, ex))


def lower_bound(I, q, r, cosine, dim):
    """A value the reference's float distance of the query to each row never falls below (-inf: no statement)."""
    sq, eq, nq, sqq = q
    sx, ex, nx, sqx = r
    ub = dot_upper(I, q, r)
    rel = rel_margin(dim)
    with np.errstate(invalid="ignore", over="ignore"):
        if cosine:
            margin = mul_ru(rel, add_ru(F32(1), mul_ru(nq, nx)))
            lb = sub_rd(sub_rd(F32(1), ub), margin)
        else:
            nsum = add_ru(nq, nx)
            margin = add_ru(mul_ru(rel, mul_ru(nsum, nsum)), F32(1e-30))
            lb = sub_rd(sub_rd(add_rd(sqq, sqx), mul_ru(F32(2), ub)), margin)
        safe = (mul_ru(nq, nx) < NORM_LIMIT) & (nq < NORM_LIMIT) & (nx < NORM_LIMIT) & np.isfinite(ex) & np.isfinite(eq)
        return np.where(safe & ~np.isnan(lb), lb, F32(-np.inf)).astype(F32)


# ---- BKT::Index::Search restated with a log of the graph candidates ----
def search_logged(f, q, k, max_check, initial_pivots, other_pivots, dist):
    """-> (ndist, ntree_rows, log) with log = list of (ids [c], dists [c], worst before the chunk)."""
    nodes, graph, n = f.nodes, f.graph, f.n
    visited = set()
    spt, ng = [], []
    seq = [0]

    def push(h, node, d):
        seq[0] += 1
        heapq.heappush(h, (d, seq[0], node))

    tree_rows = [0]

    def push_children(cs, ce):
        ids = nodes[cs:ce, 0]
        d = dist(q, ids)
        tree_rows[0] += ce - cs
        for c in range(cs, ce):
            push(spt, c, d[c - cs])

    checked = [0]

    def search_trees(limit):
        while spt:
            d, _, node = heapq.heappop(spt)
            cid, cs, ce = (int(v) for v in nodes[node])
            if cid not in visited:
                visited.add(cid)
                if cs < 0:
                    checked[0] += 1
                push(ng, cid, d)
            if cs < 0:
                if checked[0] >= limit:
                    break
            else:
                push_children(cs, ce)

    for start in f.tree_starts:
        cid, cs, ce = (int(v) for v in nodes[start])
        if cs < 0:
            tree_rows[0] += 1
            push(spt, int(start), dist(q, np.array([cid]))[0])
        else:
            push_children(cs, ce)
    search_trees(initial_pivots)

    cap = max(max_check // 16, k)
    mres = [-MAXDIST] * cap            # max-heap of the cap smallest distances
    topk = []                          # max-heap of (-(d), -id)
    log = []
    while ng:
        gd, _, node = heapq.heappop(ng)
        worst_d = -topk[0][0] if len(topk) == k else MAXDIST
        if gd <= worst_d:
            if len(topk) == k:
                heapq.heapreplace(topk, (-gd, -node))
            else:
                heapq.heappush(topk, (-gd, -node))
        elif gd > -mres[0] or checked[0] > max_check:
            break
        row = graph[node]
        neg = np.nonzero(row < 0)[0]
        row = row[:neg[0]] if neg.size else row
        fresh = []
        for v in row:
            v = int(v)
            if v not in visited:
                visited.add(v)
                fresh.append(v)
        for c0 in range(0, len(fresh), 32):
            ids = np.array(fresh[c0:c0 + 32], np.int64)
            d = dist(q, ids)
            log.append((ids, d, F32(-mres[0])))
            checked[0] += len(ids)
            for v, dv in zip(ids, d):
                if not dv > -mres[0]:
                    heapq.heapreplace(mres, -dv)
                    push(ng, int(v), dv)
        top_ng = ng[0][0] if ng else MAXDIST
        top_spt = spt[0][0] if spt else MAXDIST
        if top_ng > top_spt:
            search_trees(other_pivots + checked[0])
    nd = tree_rows[0] + sum(len(e[0]) for e in log)
    return nd, tree_rows[0], log


def build_folder(a, log):
    """The index folder of `a` (bench.py's generator and builder on the CPU), cached under a.cache."""
    import torch
    import bench
    from tools import gpu_index_builder as B
    argv = sys.argv
    sys.argv = ["bench.py", "--n", str(a.n), "--dim", str(a.dim), "--metric", a.metric, "--nq", str(a.nq), "--k", str(a.k),
                "--rank-dim", str(a.rank_dim), "--data", a.data, "--cache", a.cache]
    try:
        bargs = bench.parse_args()
    finally:
        sys.argv = argv
    folder = bench.index_folder(bargs, 0) + "_cpu"
    cpu = torch.device("cpu")
    queries = bench.gen_data(bargs, a.nq, bargs.seed + 7, cpu).numpy()
    if not os.path.exists(os.path.join(folder, "DONE")):
        t0 = time.time()
        x = bench.gen_data(bargs, a.n, bargs.seed + 1000, cpu)
        nodes, starts, graph = B.build_index(x, a.metric, seed=bargs.seed, log=log)
        B.save_index_folder(folder, x.numpy(), graph, nodes, starts, a.metric)
        with open(os.path.join(folder, "DONE"), "w") as fh:
            fh.write("ok\n")
        log("index built in %.0fs -> %s" % (time.time() - t0, folder))
    return folder, queries


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--metric", default="Cosine", choices=["Cosine", "L2"])
    ap.add_argument("--data", default="lowrank", choices=["lowrank", "iid"])
    ap.add_argument("--rank-dim", type=int, default=32)
    ap.add_argument("--nq", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--maxcheck", type=int, default=8192)
    ap.add_argument("--cache", default=os.path.join(tempfile.gettempdir(), "sptag_b200_cache"))
    a = ap.parse_args()

    def log(*m):
        print("[row_sketch_model]", *m, file=sys.stderr, flush=True)

    import reflib
    folder, queries = build_folder(a, log)
    f = reflib.IndexFiles(folder)
    cosine = a.metric == "Cosine"
    x = f.vectors

    def dist(q, ids):
        rows = x[ids]
        if cosine:
            return (F32(1) - rows @ q).astype(F32)
        dd = rows - q
        return (dd * dd).sum(axis=1).astype(F32)

    ora = reflib.OracleIndex(f)
    ora.max_check = a.maxcheck
    _, _, stats = ora.search(queries, a.k)

    t0 = time.time()
    s_rows, sc, er, nr, n2 = sketch_rows(x)
    log("sketches of %d rows in %.0fs; median err %.4g, median scale %.4g" % (f.n, time.time() - t0, np.median(er), np.median(sc)))
    tot = dict(cand=0, rejected=0, caught=0, tree=0, ndist=0, ndist_oracle=0, wrong=0)
    slack, gap = [], []
    for qi in range(a.nq):
        q = queries[qi]
        nd, ntree, lg = search_logged(f, q, a.k, a.maxcheck, ora.initial_pivots, ora.other_pivots, dist)
        t, qsc, qer, qnr, qn2 = sketch_rows(q[None, :])
        qs = (qsc[0], qer[0], qnr[0], qn2[0])
        t32 = t[0].astype(np.int32)
        for ids, d, worst in lg:
            I = s_rows[ids].astype(np.int32) @ t32
            lb = lower_bound(I, qs, (sc[ids], er[ids], nr[ids], n2[ids]), cosine, f.dim)
            rej = d > worst
            caught = lb > worst
            tot["wrong"] += int((lb > d).sum())
            tot["cand"] += len(ids)
            tot["rejected"] += int(rej.sum())
            tot["caught"] += int(caught.sum())
            slack.extend((d - lb)[np.isfinite(lb)].tolist())
            if worst < MAXDIST:
                gap.extend((d - worst)[rej].tolist())
        tot["tree"] += ntree
        tot["ndist"] += nd
        tot["ndist_oracle"] += int(stats[qi, reflib.ST_NDIST])
    nq = a.nq
    row_b = ((f.dim * 4 + 15) // 16) * 16
    sk_b = ((f.dim + 15) // 16) * 16 + SKETCH_PAD
    cand, tree = tot["cand"] / nq, tot["tree"] / nq
    now = (cand + tree) * row_b
    ceiling = tree * row_b + cand * sk_b + (cand - tot["rejected"] / nq) * row_b
    bound = tree * row_b + cand * sk_b + (cand - tot["caught"] / nq) * row_b
    out = {
        "index": "BKT %d x %d %s %s, MaxCheck %d, K %d, %d queries" % (f.n, f.dim, a.metric, a.data, a.maxcheck, a.k, nq),
        "distances_per_query": tot["ndist"] / nq, "distances_per_query_oracle": tot["ndist_oracle"] / nq,
        "graph_candidates_per_query": cand, "tree_rows_per_query": tree,
        "share_rejected": tot["rejected"] / tot["cand"], "share_caught_by_bound": tot["caught"] / tot["cand"],
        "bound_above_distance": tot["wrong"],
        "median_distance_minus_bound": float(np.median(slack)), "median_rejected_distance_minus_worst": float(np.median(gap)),
        "row_bytes_per_query_now": now, "row_bytes_per_query_perfect_test": ceiling, "row_bytes_per_query_bound": bound,
        "bytes_saved_perfect_test": 1 - ceiling / now, "bytes_saved_bound": 1 - bound / now,
    }
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
