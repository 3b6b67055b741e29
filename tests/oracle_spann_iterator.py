"""Plain-Python restatement of SPANN iterators (TEST INFRASTRUCTURE, the debugging aid of the posting step kernel of
sptag_b200_spann_iterator_next): SPANN::Index::GetIterator + SPANNResultIterator::Next for one query, with the head's
SearchIndexIterativeFromNeareast from the pinned C oracle (oracle/sptag_oracle.c) and the posting lists from
oracle_spann.SpannFolder.  Nothing here needs a GPU or the reference."""
import numpy as np

import reflib
from oracle_spann import heapify, parse_ini


def head_oracle(files):
    """The C oracle over the folder's head index, with the [BuildHead] search parameters SPANN::Index::LoadConfig hands
    to the head (SPANNIndex.cpp:59-71)"""
    import os
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        for rel, arr in files.items():
            if rel.startswith("HeadIndex/"):
                os.makedirs(os.path.join(tmp, os.path.dirname(rel)), exist_ok=True)
                with open(os.path.join(tmp, rel), "wb") as fh:
                    fh.write(bytes(arr))
        head = reflib.IndexFiles(os.path.join(tmp, "HeadIndex"))
    o = reflib.OracleIndex(head)
    bh = parse_ini(bytes(files["indexloader.ini"]).decode()).get("BuildHead", {})
    o.max_check = int(bh.get("MaxCheck", o.max_check))
    o.initial_pivots = int(bh.get("NumberOfInitialDynamicPivots", o.initial_pivots))
    o.other_pivots = int(bh.get("NumberOfOtherDynamicPivots", o.other_pivots))
    o.no_better_threshold = int(bh.get("ThresholdOfNumberOfContinuousNoBetterPropagation", o.no_better_threshold))
    return o


class SpannIterator:
    """SPANN::Index::GetIterator + SPANNResultIterator::Next for one query (SPANNResultIterator.h:37-63,
    SPANNIndex.cpp:261-320, :416-446, ExtraFullGraphSearcher.h:131-147, :492-525), one element per SearchNextInPosting
    call.  Head batches come from the C oracle's ora_iter_next_from_nearest at head_batch; folder.internal
    (SearchInternalResultNum) is read at every load.  `cov` counts what a call exercised: the last-element quirk, a refill
    inside a call, a deduper skip of an id seen in an earlier head batch, a truncated list being read."""

    def __init__(self, folder, head, query, head_batch):
        self.folder, self.hb = folder, head_batch
        self.q = np.ascontiguousarray(query)
        self.head = head.iterator(self.q)
        self.first, self.slots = True, None
        self.relaxed, self.loaded, self.load = False, 0, False
        self.seen = {}  # vid -> the head batch (load number) it was inserted in
        self.posts, self.pi, self.offset, self.head_ids = [], 0, 0, None
        self.cov = {"quirk": 0, "refill_mid_call": 0, "dedup_across_batches": 0, "truncated": 0}
        self.maxdist = np.float32(reflib.ora().ora_max_dist())

    def _head_next(self):
        ok, ids, _ = self.head.next_from_nearest(self.hb)
        self.head_ids = ids
        return ok

    def _step(self, res, b):
        """SearchDiskIndexIterative: True when the call found an element and pi did not reach the end"""
        f = self.folder
        if self.load:
            self.posts = []
            for pid in self.head_ids:
                if pid == -1:
                    break
                if f.searched(int(pid)) > 0:  # CheckValidPosting
                    self.posts.append(int(pid))
            if self.loaded >= f.internal:
                self.relaxed = True
            self.loaded += len(self.posts)
            self.pi = self.offset = 0
        found = False
        while not found and self.pi < len(self.posts):
            l = self.posts[self.pi]
            tc = f.searched(l)
            if tc < f.lists[l][0]:
                self.cov["truncated"] += 1
            while self.offset < tc:
                vid, row = f.element(l, self.offset, tc)
                self.offset += 1
                if vid != -1:
                    if vid in self.seen:
                        if self.seen[vid] != self.loaded:
                            self.cov["dedup_across_batches"] += 1
                        continue
                    self.seen[vid] = self.loaded
                rowa = np.frombuffer(row, f.dtype).copy()
                d = np.float32(reflib.ora().ora_distance(f.metric, f.vt, 16, self.q.ctypes.data, rowa.ctypes.data,
                                                         int(f.dim)))
                if d < res[0][1] or (d == res[0][1] and vid < res[0][0]):  # AddPoint
                    res[0] = [vid, d]
                    heapify(res, b)
                found = True
                break
            if self.offset == tc:
                self.pi += 1
                self.offset = 0
        if found and self.pi == len(self.posts):
            self.cov["quirk"] += 1
        return self.pi != len(self.posts)

    def next(self, batch):
        """-> (resultNum, ids [batch], dists [batch], GetRelaxedMono()); slots past resultNum are (-1, MaxDist)"""
        b = batch if self.slots is None else min(batch, self.slots)
        res = [[-1, self.maxdist] for _ in range(b)]
        if self.first:
            self._head_next()
            self.first, self.load = False, True
        cont, count, refilled = True, 0, False
        while cont and count < b:
            found = self._step(res, b)
            self.load = False
            if not found:
                cont = self._head_next()
                self.load = True
                refilled = True
            else:
                count += 1
                if refilled:
                    self.cov["refill_mid_call"] += 1
                    refilled = False
        for i in range(b - 1, -1, -1):  # SortResult
            res[0], res[i] = res[i], res[0]
            heapify(res, i)
        self.slots = count
        ids = np.full(batch, -1, np.int32)
        dists = np.full(batch, self.maxdist, np.float32)
        ids[:count] = [r[0] for r in res[:count]]
        dists[:count] = [r[1] for r in res[:count]]
        return count, ids, dists, self.relaxed

    def close(self):
        self.head.close()
