"""Plain-Python restatement of SPANN search on a PQ/OPQ-quantized index after its head search (TEST INFRASTRUCTURE).
The posting scan is restated as tests/oracle_spann.py restates it (its SpannFolder and heapify are reused); only the
distance differs.  ExtraFullGraphSearcher<std::uint8_t> scores a
code row y with the quantizer's L2Distance to the quantized query (ExtraFullGraphSearcher.h:120-130,
PQQuantizer.h:110-128): sum_i T[i][y_i] in sub-vector order with one float accumulator, where T[i] is
  SDC  the row sdc[i][q_i] of the quantizer's symmetric table (q = the query's codes, QuantizeVector with ADC off)
  ADC  the query's own distances to the codewords of sub-space i (QuantizeVector with ADC on, PQQuantizer.h:141-157;
       OPQ rotates the query first, OPQQuantizer.h:96-121)
Codes, the SDC table and every distance come from the pinned C oracle (oracle/sptag_oracle.c).  Nothing here needs a GPU
or the reference."""
import os
import tempfile

import numpy as np

import oracle_spann
import reflib


def folder_quantizer(files):
    """The quantizer the SPANN folder's [Quantizer] section names (VectorIndex.cpp:642-677)"""
    ini = oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())
    name = ini.get("Quantizer", {}).get("QuantizerFilePath") or os.path.basename(ini["Base"]["QuantizerFilePath"])
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "q.bin")
        with open(path, "wb") as fh:
            fh.write(bytes(files[name]))
        return reflib.Quantizer.read(path)


def query_tables(quant, queries, adc):
    """Per raw query its M x Ks table rows T (see above), float32 [nq, M, Ks]"""
    oq = reflib.OracleQuantizer(quant)
    L = reflib.ora()
    out = np.empty((len(queries), quant.m, quant.ks), np.float32)
    if not adc:
        codes = oq.encode(queries)
        for n in range(len(queries)):
            out[n] = oq.sdc[np.arange(quant.m), codes[n]]
        return out
    d, dsub, ks = quant.dim, quant.dsub, quant.ks
    for n in range(len(queries)):
        vec = np.ascontiguousarray(queries[n], np.float32)
        if quant.qtype == reflib.Q_OPQ:
            # out[i] = 1 - (1 - dot(vec, R^T row i)) with the float cosine tree (OPQQuantizer.h:198-206)
            a = np.ascontiguousarray(np.tile(vec, (d, 1)))
            rt = np.ascontiguousarray(quant.rotation.T)
            cos = np.empty(d, np.float32)
            L.ora_distance_f32_many(1, 16, a.ctypes.data, rt.ctypes.data, d, d, cos.ctypes.data)
            vec = (np.float32(1) - cos).astype(np.float32)
        for i in range(quant.m):
            a = np.ascontiguousarray(np.tile(vec[i * dsub:(i + 1) * dsub], (ks, 1)))
            b = np.ascontiguousarray(quant.codebooks[i])
            L.ora_distance_f32_many(0, 16, a.ctypes.data, b.ctypes.data, dsub, ks, out[n, i].ctypes.data)
    return out


def code_distance(table, row):
    """PQQuantizer::L2Distance: the ordered float sum of table[i][y_i]"""
    acc = np.float32(0)
    for i, y in enumerate(row):
        acc = np.float32(acc + table[i, y])
    return acc


def search_one(folder, table, head_ids, head_dists, k):
    """SPANN::Index<std::uint8_t>::SearchIndex for one query from its head results (W entries), as
    oracle_spann.search_one with code_distance(table, row) in place of the raw-row distance.  Returns ids [k], dists [k]
    and (postings scanned, list elements read, distances computed)."""
    maxdist = np.float32(reflib.ora().ora_max_dist())
    res = [[int(v), np.float32(d)] for v, d in zip(head_ids, head_dists)]
    w = len(res)
    limit = np.float32(res[0][1] * folder.max_dist_ratio)
    posts = []
    for r in res:  # translate and choose the postings (SPANNIndex.cpp:213-234)
        if r[0] == -1:
            break
        pid = r[0]
        r[0] = int(folder.translate[pid])
        if r[0] == oracle_spann.INT_MAX:
            r[0], r[1] = -1, maxdist
        if len(posts) >= folder.internal or (float(limit) > 0.1 and r[1] > limit) or folder.searched(pid) == 0:
            continue
        posts.append(pid)
    res.reverse()
    seen, elements, ndist = set(), 0, 0
    for l in posts:
        tc = folder.searched(l)
        elements += tc
        for i in range(tc):
            vid, row = folder.element(l, i, tc)
            if vid != -1:  # the deduper never finds -1 (WorkSpace.h:113-160)
                if vid in seen:
                    continue
                seen.add(vid)
            d = code_distance(table, row)
            ndist += 1
            if d < res[0][1] or (d == res[0][1] and vid < res[0][0]):  # AddPoint
                res[0] = [vid, d]
                oracle_spann.heapify(res, w)
    for i in range(w - 1, -1, -1):  # SortResult
        res[0], res[i] = res[i], res[0]
        oracle_spann.heapify(res, i)
    ids = np.array([r[0] for r in res[:k]], np.int32)
    dists = np.array([r[1] for r in res[:k]], np.float32)
    return ids, dists, (len(posts), elements, ndist)


def search(folder, quant, queries, head_ids, head_dists, k, adc):
    """search_one over a batch of raw queries: ids [nq, k], dists [nq, k], stats [nq, 3]"""
    tables = query_tables(quant, queries, adc)
    out = [search_one(folder, tables[i], head_ids[i], head_dists[i], k) for i in range(len(queries))]
    return (np.stack([o[0] for o in out]), np.stack([o[1] for o in out]),
            np.array([o[2] for o in out], np.int32))
