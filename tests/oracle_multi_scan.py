"""Plain-Python restatement of the reference's MultiIndexScan (src/Core/MultiIndexScan.cpp:87-183) -- TEST
INFRASTRUCTURE.

The per-index iterators are not run here: their Next(1) streams are recorded from the reference
(tests/golden/make_golden_multi_scan.py) and replayed.  GetDistance(target_j, vid) is the C restatement's distance
(oracle/sptag_oracle.c, AVX-512 summation trees).  Everything else is restated:

* the round loop, the seen set and the unsigned termination tests (termCondVal is unsigned int, searchLimit is compared
  with seenSet.size() as size_t);
* std::priority_queue<pair<float, SizeType>> with a comparator on the score only, through libstdc++'s __push_heap /
  __pop_heap / __adjust_heap (bits/stl_heap.h, GCC 13), which decide which of equal scores is evicted and their output
  order;
* the score as GCC compiles WeightedRankFunc with -O3 -march=x86-64-v3 (MultiIndexScan.o): blocks of 8 and then 4 terms
  add their rounded products one after another (vmulps + vaddss), the last n % 4 terms are fused (vfmadd231ss).
  rankFunc's plain sum (std::accumulate, vaddss) equals that with unit weights bit for bit.
"""
import os
from fractions import Fraction

import numpy as np

import reflib

MAXDIST = np.float32(np.finfo(np.float32).max / np.float32(10))
END_DROPS, END_LIMIT, END_EXHAUSTED = 0, 1, 2


def _ini(text):
    params = {}
    for line in text.splitlines():
        line = line.strip()
        if "=" in line and not line.startswith("["):
            key, v = line.split("=", 1)
            params[key.strip()] = v.strip()
    return params


class Fixture:
    """One index set of a multi-scan fixture: its folders' files, queries and recorded iterator streams."""

    def __init__(self, g, streams=None):
        self.g = g
        self.n = int(g["n"])
        s = streams if streams is not None else g
        self.sids, self.sdists, self.slen = s["sids"], s["sdists"], s["slen"]
        self.length = self.sids.shape[2]
        self.metric, self.vt, self.rows, self.queries = [], [], [], []
        for i in range(self.n):
            p = _ini(bytes(g["file:%d:indexloader.ini" % i]).decode())
            self.metric.append(reflib.METRIC_OF_NAME[p["DistCalcMethod"]])
            self.vt.append(reflib.VT_OF_NAME[p["ValueType"]])
            raw = np.asarray(g["file:%d:vectors.bin" % i], np.uint8)
            rows, dim = np.frombuffer(raw[:8].tobytes(), np.int32)
            dt = reflib.NP_OF_VT[self.vt[i]]
            self.rows.append(np.frombuffer(raw[8:].tobytes(), dt).reshape(rows, dim))
            self.queries.append(np.ascontiguousarray(g["queries_%d" % i]))
        self.nq = self.queries[0].shape[0]

    def folder(self, i, path):
        """Writes index i's folder (as the reference saved it) to path."""
        os.makedirs(path, exist_ok=True)
        pre = "file:%d:" % i
        for key in self.g.files if hasattr(self.g, "files") else self.g.keys():
            if key.startswith(pre):
                np.asarray(self.g[key], np.uint8).tofile(os.path.join(path, key[len(pre):]))
        return path

    def distance(self, j, q, vid):
        """GetDistance(target_j, vid) = ComputeDistance(target, row vid) (BKT/Index.h:145-147)"""
        a, b = self.queries[j][q], self.rows[j][vid]
        return np.float32(reflib.ora().ora_distance(self.metric[j], self.vt[j], 16, a.ctypes.data, b.ctypes.data,
                                                    a.shape[0]))

    def next1(self, i, q, pos):
        """Index i's pos-th Next(1) for query q: (vid, dist), or None when the iterator returned nothing"""
        if pos < self.slen[i, q]:
            return int(self.sids[i, q, pos]), np.float32(self.sdists[i, q, pos])
        if self.slen[i, q] < self.length:
            return None
        raise IndexError("the recorded stream of index %d, query %d ends before position %d" % (i, q, pos))


def _f32(x):
    return np.float32(x)


def fma32(a, b, c):
    """a * b + c rounded once to float32 (round to nearest even)"""
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    x = np.float32(float(exact))
    best = None
    for cand in (np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))):
        if not np.isfinite(cand):
            continue
        err = abs(Fraction(float(cand)) - exact)
        if best is None or err < best[0] or (err == best[0] and (int(np.array(cand).view(np.int32)) & 1) == 0):
            best = (err, cand)
    return np.float32(best[1])


def weighted_rank(d, w):
    """WeightedRankFunc as compiled: see the module docstring"""
    acc = np.float32(0.0)
    n, i = len(d), 0
    while n - i >= 8:
        for t in range(8):
            acc = _f32(acc + _f32(d[i + t] * w[i + t]))
        i += 8
    if n - i >= 4:
        for t in range(4):
            acc = _f32(acc + _f32(d[i + t] * w[i + t]))
        i += 4
    for t in range(i, n):
        acc = fma32(d[t], w[t], acc)
    return acc


# libstdc++ heap algorithms with pq_item_compare: a < b iff a[0] < b[0]
def _push_hole(h, hole, top, value):
    parent = (hole - 1) // 2
    while hole > top and h[parent][0] < value[0]:
        h[hole] = h[parent]
        hole = parent
        parent = (hole - 1) // 2
    h[hole] = value


def pq_push(h, value):
    h.append(None)
    _push_hole(h, len(h) - 1, 0, value)


def pq_pop(h):
    length = len(h) - 1
    if length > 0:
        value = h[length]
        h[length] = h[0]
        hole = child = 0
        while child < (length - 1) // 2:
            child = 2 * (child + 1)
            if h[child][0] < h[child - 1][0]:
                child -= 1
            h[hole] = h[child]
            hole = child
        if (length & 1) == 0 and child == (length - 2) // 2:
            child = 2 * (child + 1)
            h[hole] = h[child - 1]
            hole = child - 1
        _push_hole(h, hole, 0, value)
    h.pop()


def scan(fx, q, k, term_cond, search_limit, weights=None):
    """Init + Next until false for query q -> dict(ids, scores, rounds, seen, drops, end, used: stream entries read per
    index, scored: (score, id) in scoring order, same_round, tie_evictions)"""
    n = fx.n
    w = [np.float32(1.0)] * n if weights is None else [np.float32(x) for x in weights]
    term = term_cond & 0xFFFFFFFF
    limit = search_limit & 0xFFFFFFFFFFFFFFFF
    pq, seen, scored = [], set(), []
    drops, rounds, end = 0, 0, None
    same_round = tie_evictions = 0  # ids returned twice in one round; evictions with the top's score held twice
    used = [0] * n
    while end is None:
        rounds += 1
        this_round = set()
        for i in range(n):
            r = fx.next1(i, q, used[i])
            if r is None:
                end = END_EXHAUSTED + i
                break
            used[i] += 1
            vid, dist = r
            if vid in seen:
                same_round += vid in this_round
                continue
            this_round.add(vid)
            d = [dist if j == i else fx.distance(j, q, vid) for j in range(n)]
            score = weighted_rank(d, w)
            scored.append((score, vid))
            if len(pq) == k and pq[0][0] <= score:
                drops = (drops + 1) & 0xFFFFFFFF
            else:
                drops = 0
                if len(pq) == k:
                    tie_evictions += sum(e[0] == pq[0][0] for e in pq) > 1
                    pq_pop(pq)
                pq_push(pq, (score, vid))
            seen.add(vid)
        if end is None:
            if drops >= term:
                end = END_DROPS
            elif len(seen) >= limit:
                end = END_LIMIT
    stack = []
    while pq:
        stack.append(pq[0])
        pq_pop(pq)
    out = stack[::-1]
    return dict(ids=np.array([v for _, v in out], np.int32), scores=np.array([s for s, _ in out], np.float32),
                rounds=rounds, seen=len(seen), drops=drops, end=end, used=np.array(used), scored=scored,
                same_round=same_round, tie_evictions=tie_evictions)


def expected(fx, k, term_cond, search_limit, weights=None):
    """Every query of the fixture -> (ids [nq x k], scores [nq x k], counts [nq], stats [nq x 4], per-query results)"""
    ids = np.full((fx.nq, k), -1, np.int32)
    scores = np.full((fx.nq, k), MAXDIST, np.float32)
    counts = np.zeros(fx.nq, np.int32)
    stats = np.zeros((fx.nq, 4), np.int32)
    res = []
    for q in range(fx.nq):
        r = scan(fx, q, k, term_cond, search_limit, weights)
        c = len(r["ids"])
        ids[q, :c], scores[q, :c], counts[q] = r["ids"], r["scores"], c
        stats[q] = (r["rounds"], r["seen"], r["drops"], r["end"])
        res.append(r)
    return ids, scores, counts, stats, res
