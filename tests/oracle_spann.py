"""Plain-Python restatement of SPANN search after its head search (TEST INFRASTRUCTURE, the debugging aid of the posting
scan kernel).  Given a SPANN folder's files and the head index's results at W = max(K, SearchInternalResultNum), it runs
SPANN::Index<T>::SearchIndex (SPANNIndex.cpp:193-250) and ExtraFullGraphSearcher<T>::SearchIndex
(ExtraFullGraphSearcher.h:226-375) step by step: translate + choose postings, Reverse, the deduper, AddPoint with
QueryResultSet's exact Heapify, SortResult (QueryResultSet.h:77-112).  Distances come from the pinned C oracle
(oracle/sptag_oracle.c, ora_distance).  Nothing here needs a GPU or the reference."""
import numpy as np

import reflib

VT = {"Float": (reflib.VT_FLOAT, np.float32), "Int8": (reflib.VT_INT8, np.int8), "UInt8": (1, np.uint8),
      "Int16": (2, np.int16)}
INT_MAX = 2**31 - 1


def parse_ini(text):
    """{section: {name: value}} of an indexloader.ini"""
    out, sec = {}, ""
    for ln in text.splitlines():
        ln = ln.rstrip("\r ")
        if not ln or ln[0] in ";#":
            continue
        if ln[0] == "[":
            sec = ln[1:ln.index("]")]
            continue
        if "=" in ln:
            k, v = ln.split("=", 1)
            out.setdefault(sec, {})[k] = v
    return out


class SpannFolder:
    """The parts of a SPANN folder the posting scan reads, from {relative path: bytes}."""

    def __init__(self, files, ini_values=None):
        ini = parse_ini(bytes(files["indexloader.ini"]).decode())
        for k, v in (ini_values or {}).items():
            for sec in ini.values():
                if k in sec:
                    sec[k] = v
        base, ssd = ini["Base"], ini["BuildSSDIndex"]
        self.vt, dtype = VT[base["ValueType"]]
        self.metric = 0 if base["DistCalcMethod"] == "L2" else 1
        self.internal = int(ssd["SearchInternalResultNum"])
        self.max_dist_ratio = np.float32(float(ssd["MaxDistRatio"]))
        self.rearranged = ssd["EnablePostingListRearrange"].lower() == "true"
        tmap = np.frombuffer(bytes(files[base.get("HeadVectorIDs", "SPTAGHeadVectorIDs.bin")]), np.uint64)
        self.translate = (tmap & np.uint64(0xffffffff)).astype(np.uint32).view(np.int32)
        name = ssd.get("SSDIndex", base.get("SSDIndex", "SPTAGFullList.bin"))
        self.lists = []  # per list: (full element count, page count, its file's bytes, its start in them)
        for fi in range(1000):
            blob = files.get(name if fi == 0 else "%s_%d" % (name, fi))
            if blob is None:
                break
            blob = bytes(blob)
            count, _, self.dim, page_off = np.frombuffer(blob[:16], np.int32)
            for i in range(count):
                rec = blob[16 + 12 * i:28 + 12 * i]
                page_num = int(np.frombuffer(rec[:4], np.int32)[0])
                start = ((int(page_off) + page_num) << 12) + int(np.frombuffer(rec[4:6], np.uint16)[0])
                ele = int(np.frombuffer(rec[6:10], np.int32)[0])
                pages = int(np.frombuffer(rec[10:12], np.uint16)[0])
                self.lists.append((ele, pages, blob, start))
        self.dtype = dtype
        self.row_bytes = int(self.dim) * np.dtype(dtype).itemsize
        self.vis = self.row_bytes + 4
        vector_limit = int(ssd.get("PostingVectorLimit", "118"))
        # ExtraFullGraphSearcher::LoadIndex (:167): at least the pages of PostingVectorLimit vectors
        self.page_limit = max(int(ssd["SearchPostingPageLimit"]), (vector_limit * self.vis + 4095) // 4096)

    def searched(self, l):
        """LoadingHeadInfo's truncated element count (ExtraFullGraphSearcher.h:1093-1097)"""
        ele, pages, _, _ = self.lists[l]
        return min(ele, (min(pages, self.page_limit) << 12) // self.vis)

    def element(self, l, i, tc):
        """(id, row bytes) of element i when tc elements are read: ParsePostingList / ParsePostingListRearrange (:1186-1196).
        For a truncated rearranged list (tc < its element count) the id is read at the offset ParsePostingListRearrange
        computes from tc; the reference's results on such lists still differ from this restatement (cause not found), so
        the pin test skips them and the device refuses them."""
        _, _, blob, start = self.lists[l]
        if self.rearranged:
            off_id, off_vec = self.row_bytes * tc + 4 * i, self.row_bytes * i
        else:
            off_id = self.vis * i
            off_vec = off_id + 4
        vid = int(np.frombuffer(blob[start + off_id:start + off_id + 4], np.int32)[0])
        return vid, blob[start + off_vec:start + off_vec + self.row_bytes]


def _less(a, b):  # BasicResult operator< (QueryResultSet.h:17-20)
    return a[1] < b[1] or (a[1] == b[1] and a[0] < b[0])


def heapify(res, count):
    """QueryResultSet::Heapify, including its `next < maxidx` bound"""
    parent, nxt, maxidx = 0, 1, count - 1
    while nxt < maxidx:
        if _less(res[nxt], res[nxt + 1]):
            nxt += 1
        if _less(res[parent], res[nxt]):
            res[nxt], res[parent] = res[parent], res[nxt]
            parent = nxt
            nxt = (parent << 1) + 1
        else:
            break
    if nxt == maxidx and _less(res[parent], res[nxt]):
        res[parent], res[nxt] = res[nxt], res[parent]


def search_one(folder, query, head_ids, head_dists, k):
    """SPANN::Index::SearchIndex for one query from its head results (W entries).  Returns ids [k], dists [k] and
    (postings scanned, list elements read, distances computed)."""
    L = reflib.ora()
    maxdist = np.float32(L.ora_max_dist())
    res = [[int(v), np.float32(d)] for v, d in zip(head_ids, head_dists)]
    w = len(res)
    limit = np.float32(res[0][1] * folder.max_dist_ratio)
    posts = []
    for r in res:
        if r[0] == -1:
            break
        pid = r[0]
        r[0] = int(folder.translate[pid])
        if r[0] == INT_MAX:
            r[0], r[1] = -1, maxdist
        if len(posts) >= folder.internal or (float(limit) > 0.1 and r[1] > limit) or folder.searched(pid) == 0:
            continue
        posts.append(pid)
    res.reverse()
    q = np.ascontiguousarray(query)
    seen, elements, ndist = set(), 0, 0
    for l in posts:
        tc = folder.searched(l)
        elements += tc
        for i in range(tc):
            vid, row = folder.element(l, i, tc)
            if vid != -1:  # the deduper stores vid + 1 with 0 as its empty key: -1 is never found (WorkSpace.h:113-160)
                if vid in seen:
                    continue
                seen.add(vid)
            rowa = np.frombuffer(row, folder.dtype).copy()
            d = np.float32(L.ora_distance(folder.metric, folder.vt, 16, q.ctypes.data, rowa.ctypes.data, int(folder.dim)))
            ndist += 1
            if d < res[0][1] or (d == res[0][1] and vid < res[0][0]):  # AddPoint
                res[0] = [vid, d]
                heapify(res, w)
    for i in range(w - 1, -1, -1):  # SortResult
        res[0], res[i] = res[i], res[0]
        heapify(res, i)
    ids = np.array([r[0] for r in res[:k]], np.int32)
    dists = np.array([r[1] for r in res[:k]], np.float32)
    return ids, dists, (len(posts), elements, ndist)


def search(folder, queries, head_ids, head_dists, k):
    """search_one over a batch: ids [nq, k], dists [nq, k], stats [nq, 3]"""
    out = [search_one(folder, queries[i], head_ids[i], head_dists[i], k) for i in range(len(queries))]
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]),
            np.array([o[2] for o in out], np.int32))


def fixture_files(g):
    """{relative path: bytes} of a tests/golden/spann fixture"""
    return {key[5:]: g[key] for key in g.files if key.startswith("file:")}
