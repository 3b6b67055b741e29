"""The multi-index scan on the device (sptag_b200_multi_scan) against the unmodified reference's MultiIndexScan, recorded
in tests/golden/multi_scan: counts, ids, score bits and, against the plain-Python restatement (tests/oracle_multi_scan.py),
the per-query stats of every set and parameter set.  Also: a batch equals its queries run one by one, queries that end
in different rounds share a batch, seen-set tables grow through several doublings, the refusals, and member handles
search and add after a scan exactly as before it."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import oracle_multi_scan as oms
import reflib
from sptag_b200 import capi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SETS = {os.path.basename(p)[:-4]: p for p in sorted(glob.glob(os.path.join(HERE, "golden", "multi_scan", "*.npz")))}
FAIL, LACK_OF_INPUTS = 0x01, 0x13


@pytest.fixture(scope="module", autouse=True)
def _port():
    reflib.build_port()


def load_set(name, tmp_path):
    g = np.load(SETS[name])
    fx = oms.Fixture(g)
    idx = [capi.B200Index.load(fx.folder(i, str(tmp_path / ("%s_%d" % (name, i)))), 0) for i in range(fx.n)]
    return g, fx, idx


def close(idx):
    for ix in idx:
        ix.close()


def params(g, p):
    w = g["weights_" + p]
    return int(g["k_" + p]), int(g["term_" + p]), int(g["limit_" + p]), (None if w.size == 0 else w)


@pytest.mark.parametrize("name", sorted(SETS))
def test_multi_scan_equals_reference(name, tmp_path):
    g, fx, idx = load_set(name, tmp_path)
    try:
        for p in sorted(key[2:] for key in g.files if key.startswith("k_")):
            k, term, limit, w = params(g, p)
            ids, scores, counts, stats = capi.multi_scan(idx, fx.queries, k, weights=w, term_cond=term, search_limit=limit,
                                                         want_stats=True)
            assert np.array_equal(counts, g["counts_" + p]), p
            assert np.array_equal(ids, g["ids_" + p]), p
            assert np.array_equal(scores.view(np.int32), g["scores_" + p].view(np.int32)), p
            _, _, _, st, _ = oms.expected(fx, k, term, limit, w)
            assert np.array_equal(stats, st), p
    finally:
        close(idx)


def test_batch_equals_single_queries_and_mixed_rounds(tmp_path):
    g, fx, idx = load_set("dups", tmp_path)
    try:
        k, term, limit, w = params(g, "limit")
        ids, scores, counts, stats = capi.multi_scan(idx, fx.queries, k, weights=w, term_cond=term, search_limit=limit,
                                                     want_stats=True)
        assert len(set(stats[:, capi.MS_ROUNDS].tolist())) > 1, "every query ended in the same round"
        for q in range(fx.nq):
            one = capi.multi_scan(idx, [x[q:q + 1] for x in fx.queries], k, weights=w, term_cond=term, search_limit=limit,
                                  want_stats=True)
            assert np.array_equal(one[0][0], ids[q]) and np.array_equal(one[1][0].view(np.int32), scores[q].view(np.int32))
            assert one[2][0] == counts[q] and np.array_equal(one[3][0], stats[q])
    finally:
        close(idx)


def test_seen_tables_double_several_times(tmp_path):
    """The scan to exhaustion sees all 500 ids in 501 rounds of 2 indexes: the tables, which start at 128 entries and
    stay below half load for min(n x rounds, N) ids, double three times (to 1024)"""
    g, fx, idx = load_set("dups", tmp_path)
    try:
        k, term, limit, w = params(g, "exhaust")
        ids, scores, counts, stats = capi.multi_scan(idx, fx.queries, k, weights=w, term_cond=term, search_limit=limit,
                                                     want_stats=True)
        assert (stats[:, capi.MS_SEEN] == fx.rows[0].shape[0]).all() and (stats[:, capi.MS_ROUNDS] == 501).all()
        assert np.array_equal(ids, g["ids_exhaust"])
        assert np.array_equal(scores.view(np.int32), g["scores_exhaust"].view(np.int32))
    finally:
        close(idx)


def _raw(handles, n, queries, k, nq=2, out=True):
    ids = np.empty((nq, max(k, 1)), np.int32)
    scores = np.empty((nq, max(k, 1)), np.float32)
    counts = np.empty(nq, np.int32)
    hs = (C.c_void_p * max(n, 1))(*handles[:max(n, 1)])
    qp = (C.c_void_p * max(n, 1))(*queries[:max(n, 1)])
    return capi.lib().sptag_b200_multi_scan(hs, n, qp, None, nq, k, 5, 100, ids.ctypes.data if out else None,
                                            scores.ctypes.data, counts.ctypes.data, None)


def test_refusals(tmp_path):
    g, fx, idx = load_set("bfs", tmp_path)
    _, fx2, idx2 = load_set("dups", tmp_path)
    from tools.gpu_index_builder import save_index_folder
    kg = np.load(os.path.join(HERE, "golden", "kdt_l2_2k_16.npz"))
    kp = dict(zip(kg["param_names"].tolist(), kg["param_values"].tolist()))
    save_index_folder(str(tmp_path / "kdt"), kg["vectors"], kg["graph"], kg["nodes"], kg["tree_starts"], kp["DistCalcMethod"],
                      algo="KDT", value_type=kp["ValueType"])
    kdt = capi.B200Index.load(str(tmp_path / "kdt"), 0)
    shifted = capi.B200Index.load(fx.folder(0, str(tmp_path / "shifted")), 0, id_offset=5)
    qg = np.load(os.path.join(HERE, "golden", "quantized", "pq_f32_1200_16.npz"))
    pq = capi.B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_UINT8, metric=capi.METRIC_L2, vectors=qg["vectors"],
                               graph=qg["graph"], tree_starts=qg["tree_starts"], tree_nodes=qg["nodes"], device=0)
    pq.set_quantizer(qg["quantizer_blob"].tobytes())
    try:
        hs = [ix._h.value for ix in idx]
        qs = [q.ctypes.data for q in fx.queries]
        assert _raw(hs, 2, qs, 10) == 0
        assert _raw(hs, 0, qs, 10) == LACK_OF_INPUTS
        assert _raw(hs * 9, 17, qs * 9, 10) == LACK_OF_INPUTS
        assert _raw(hs, 2, qs, 0) == LACK_OF_INPUTS
        assert _raw(hs, 2, qs, 1025) == LACK_OF_INPUTS
        assert _raw(hs, 2, qs, 10, out=False) == LACK_OF_INPUTS
        assert _raw([hs[0], None], 2, qs, 10) == LACK_OF_INPUTS
        assert _raw(hs, 2, [qs[0], None], 10) == LACK_OF_INPUTS
        assert _raw([hs[0], idx2[0]._h.value], 2, [qs[0], fx2.queries[0].ctypes.data], 10) == LACK_OF_INPUTS  # counts
        kq = np.ascontiguousarray(kg["queries"][:2])
        assert _raw([hs[0], kdt._h.value], 2, [qs[0], kq.ctypes.data], 10) == FAIL
        assert _raw([hs[0], shifted._h.value], 2, [qs[0], qs[0]], 10) == LACK_OF_INPUTS  # id offsets differ
        pq_q = np.ascontiguousarray(qg["queries"][:2])
        assert _raw([hs[0], pq._h.value], 2, [qs[0], pq_q.ctypes.data], 10) == LACK_OF_INPUTS  # quantized
        assert _raw(hs, 2, qs, 10) == 0  # the refused calls left the handles usable
    finally:
        pq.close()
        shifted.close()
        kdt.close()
        close(idx)
        close(idx2)


def test_members_unchanged_by_scan(tmp_path):
    g, fx, idx = load_set("views3", tmp_path)
    try:
        before = [ix.search(fx.queries[i], 10) for i, ix in enumerate(idx)]
        k, term, limit, w = params(g, "drops")
        capi.multi_scan(idx, fx.queries, k, weights=w, term_cond=term, search_limit=limit)
        after = [ix.search(fx.queries[i], 10) for i, ix in enumerate(idx)]
        for b, a in zip(before, after):
            assert np.array_equal(b[0], a[0]) and np.array_equal(b[1].view(np.int32), a[1].view(np.int32))
        # the scan's iterators are closed: the handle takes an add again
        first = idx[0].add(fx.queries[0][:3])
        assert first == fx.rows[0].shape[0]
    finally:
        close(idx)
