"""Plain-Python restatement of SPANN's posting-list build after its head searches (TEST INFRASTRUCTURE, the debugging aid
of sptag_b200_spann_build).  Given a folder's ini, the rows and every row's head results at InternalResultNum, it runs
the rest of ExtraFullGraphSearcher::BuildIndex (ExtraFullGraphSearcher.h:587-922): ApproximateRNG's selection
(VectorIndex.cpp:940-970) with the pinned C oracle's ora_distance, SortSelections' EdgeCompare order, the posting cut,
the split over SSDIndexFileNum files, SelectPostingOffset (:1206-1290) and OutputSSDIndexFile (:1292-1568).  Returns
{file name: bytes}.  Nothing here needs a GPU or the reference."""
import bisect

import numpy as np

import oracle_spann
import reflib

MAX_SIZE = 2**31 - 1


def _get(ini, section, name, default):
    return ini.get(section, {}).get(name, default)


def normalize(x, base):
    """COMMON::Utils::Normalize per row: the length summed in double in element order, each element divided by it and
    scaled by base, then cast back to the row type (CommonUtils.h:62-76)"""
    out = np.empty_like(x)
    for i, row in enumerate(x):
        v = row.astype(np.float64)
        length = np.sqrt(np.cumsum(v * v)[-1])
        if length < 1e-6:
            vals = np.full(len(v), 1.0 / np.sqrt(float(len(v))) * base)
        else:
            vals = v / length * base
        out[i] = vals if x.dtype == np.float32 else np.trunc(vals)
    return out


def select_posting_offset(nbytes):
    """page number and offset per list, and the placement order: each time the list with the largest bytes % 4096 that
    fits in the current page (the lower id among equals); a page nothing fits in is closed"""
    keys = sorted((-(b % 4096), i) for i, b in enumerate(nbytes) if b)
    page_num, page_off, order = [0] * len(nbytes), [0] * len(nbytes), []
    page = off = 0
    while keys:
        room = 4096 - off
        at = bisect.bisect_left(keys, (-room, -1))
        if at == len(keys) or (room != 4096 and keys[at][0] == 0):
            page, off = page + 1, 0
            continue
        rest, i = keys.pop(at)
        page_num[i], page_off[i] = page, off
        order.append(i)
        off -= rest
        if off == 4096:
            page, off = page + 1, 0
        page += nbytes[i] // 4096
    return page_num, page_off, order


def posting_file(lists, rows, dim, n, rearranged):
    """OutputSSDIndexFile for one file: lists = per list the vector ids written, in order"""
    row_bytes = rows.shape[1] * rows.dtype.itemsize
    vis = row_bytes + 4
    nbytes = [len(l) * vis for l in lists]
    page_num, page_off, order = select_posting_offset(nbytes)
    meta = 16 + 12 * len(lists)
    head = bytearray(-(-meta // 4096) * 4096)
    head[:16] = np.array([len(lists), n, dim, len(head) // 4096], np.int32).tobytes()
    for i, l in enumerate(lists):
        rec = (np.array([page_num[i] if l else 0], np.int32).tobytes() + np.array([page_off[i] if l else 0], np.uint16).tobytes()
               + np.array([len(l)], np.int32).tobytes() + np.array([-(-nbytes[i] // 4096)], np.uint16).tobytes())
        head[16 + 12 * i:28 + 12 * i] = rec
    area = bytearray()
    for i in order:
        start = page_num[i] * 4096 + page_off[i]
        area += bytes(start - len(area))
        ids = np.array(lists[i], np.int32)
        if rearranged:
            area += rows[ids].tobytes() + ids.tobytes()
        else:
            for v in lists[i]:
                area += np.array([v], np.int32).tobytes() + rows[v].tobytes()
    area += bytes(-len(area) % 4096)
    return bytes(head) + bytes(area)


def build(files, vectors, head_ids, head_dists, normalized=False, simd_width=16, read=None):
    """The posting files (and, with ExcludeHead false, the rewritten head-id file) the SSD stage writes.  files: the
    folder's files before the stage {relative path: bytes}; head_ids / head_dists: [n x InternalResultNum] the head
    search of every row.  Returns ({name: bytes}, RNG rejections, edges before the cut, edges after it).  read: an int
    array of n entries or None; it receives how many head results of each row the selection examined."""
    ini = oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())
    vt, dtype = oracle_spann.VT[_get(ini, "Base", "ValueType", "Float")]
    metric = 0 if _get(ini, "Base", "DistCalcMethod", "L2") == "L2" else 1
    replicas = int(_get(ini, "BuildSSDIndex", "ReplicaCount", "8"))
    rng_factor = np.float32(float(_get(ini, "BuildSSDIndex", "RNGFactor", "1.0")))
    page_limit = int(_get(ini, "BuildSSDIndex", "PostingPageLimit", "3"))
    vector_limit = int(_get(ini, "BuildSSDIndex", "PostingVectorLimit", "118"))
    exclude_head = _get(ini, "BuildSSDIndex", "ExcludeHead", "true").lower() == "true"
    rearranged = _get(ini, "BuildSSDIndex", "EnablePostingListRearrange", "false").lower() == "true"
    file_num = int(_get(ini, "Base", "SSDIndexFileNum", "1"))
    ssd = _get(ini, "Base", "SSDIndex", "SPTAGFullList.bin")
    id_name = _get(ini, "Base", "HeadVectorIDs", "SPTAGHeadVectorIDs.bin")
    head_dir = _get(ini, "Base", "HeadIndexFolder", "HeadIndex")
    hv = bytes(files[head_dir + "/vectors.bin"])
    nh, dim = (int(v) for v in np.frombuffer(hv[:8], np.int32))
    heads = np.frombuffer(hv[8:8 + nh * dim * np.dtype(dtype).itemsize], dtype).reshape(nh, dim)
    x = np.ascontiguousarray(vectors, dtype)
    n = len(x)
    if metric == 1 and not normalized:
        x = normalize(x, 1 if dtype == np.float32 else {np.int8: 127, np.uint8: 255, np.int16: 32767}[dtype])
    out = {}
    if not exclude_head:
        out[id_name] = np.full(nh, MAX_SIZE, np.uint64).tobytes()
        id_blob = out[id_name]
    else:
        id_blob = bytes(files[id_name])
    head_set = set((np.frombuffer(id_blob, np.uint64) & np.uint64(0xffffffff)).astype(np.uint32).view(np.int32).tolist())
    L = reflib.ora()
    cache = {}

    def head_distance(a, b):
        key = (a, b)
        if key not in cache:
            ra, rb = np.ascontiguousarray(heads[a]), np.ascontiguousarray(heads[b])
            cache[key] = np.float32(L.ora_distance(metric, vt, simd_width, ra.ctypes.data, rb.ctypes.data, dim))
        return cache[key]

    edges, rejected = [], 0  # (node, distance, tonode)
    for v in range(n):
        if v in head_set:
            continue
        accepted = []
        for col, (vid, d) in enumerate(zip(head_ids[v].tolist(), head_dists[v])):
            if len(accepted) >= replicas or vid == -1:
                break
            if read is not None:
                read[v] = col + 1
            if any(rng_factor * head_distance(vid, a) < d for a in accepted):
                rejected += 1
                continue
            accepted.append(vid)
            edges.append((vid, np.float32(d), v))
    edges.sort(key=lambda e: (e[0], float(e[1]), e[2]))  # EdgeCompare: -0.0 == 0.0
    lists = [[] for _ in range(nh)]
    for node, _, tonode in edges:
        lists[node].append(tonode)
    vis = x.shape[1] * x.dtype.itemsize + 4
    limit = MAX_SIZE
    if page_limit > 0:
        limit = max(page_limit, -(-vector_limit * vis // 4096)) * 4096 // vis
    before = len(edges)
    lists = [l[:limit] for l in lists]
    after = sum(len(l) for l in lists)
    per_file = -(-nh // file_num)
    for i in range(file_num):
        name = ssd if i == 0 else "%s_%d" % (ssd, i)
        out[name] = posting_file(lists[i * per_file:min(nh, (i + 1) * per_file)], x, dim, n, rearranged)
    return out, rejected, before, after
