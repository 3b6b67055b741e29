"""GPU tests of the row sketches (B200.RowSketch): BKT search tests a graph candidate's 1-byte-per-dimension sketch and
fetches its row only when the sketch cannot prove that m_Results rejects it.  Whatever is skipped, a search must return
what it returns with the sketches off: ids, distance bits and all eight per-query counters."""
import os

import numpy as np
import pytest

import reflib
import test_oracle_pin as pin
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BKT_SETS = ["algo_line_bkt", "bkt_cos_1500_20", "bkt_l2_2k_16", "bkt_l2_dups_1k_12"]


def golden_index(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    pin._files_from_npz(files, g)
    idx = B200Index.create(algo=capi.ALGO_KDT if files.algo == "KDT" else capi.ALGO_BKT, value_type=capi.VT_FLOAT,
                           metric=files.metric, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                           tree_nodes=files.nodes)
    return g, files, idx


def skipped(idx):
    return int(idx.get_param("B200.RowsSkipped"))


def both(idx, run):
    """run() with the sketches off and on -> (results off, results on, candidates skipped by the second)."""
    idx.set_param("B200.RowSketch", 0)
    before = skipped(idx)
    off = run()
    assert skipped(idx) == before
    idx.set_param("B200.RowSketch", 1)
    on = run()
    return off, on, skipped(idx) - before


def same(off, on, what):
    for a, b in zip(off, on):
        assert np.array_equal(np.asarray(a).view(np.int32), np.asarray(b).view(np.int32)), what


@pytest.mark.parametrize("name", BKT_SETS)
def test_results_and_counters_unchanged(name):
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    try:
        total = 0
        for mc in (16, 512, 8192):
            idx.set_param("MaxCheck", mc)
            for k in (1, 10, 100):
                off, on, sk = both(idx, lambda: idx.search(q, k, want_stats=True))
                same(off, on, (name, mc, k))
                total += sk
        # the oracle too, once
        idx.set_param("MaxCheck", 512)
        ids, dists, stats = idx.search(q, 10, want_stats=True)
        o = reflib.OracleIndex(files)
        o.max_check = 512
        ids_o, d_o, st_o = o.search(q, 10)
        assert np.array_equal(ids, ids_o) and np.array_equal(dists.view(np.int32), d_o.view(np.int32))
        assert np.array_equal(stats[:, capi.ST_NDIST], st_o[:, reflib.ST_NDIST])
        if name != "algo_line_bkt":
            assert total > 0, "no candidate was skipped on %s" % name
    finally:
        idx.close()


@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt_cos_1500_20"])
def test_filter_tombstones_hashed_set_and_simd_widths(name):
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    rng = np.random.default_rng(11)
    allowed = (rng.random(files.n) < 0.5).astype(np.uint8)
    try:
        idx.set_param("MaxCheck", 512)
        off, on, _ = both(idx, lambda: idx.search_filtered(q, 10, allowed, want_stats=True))
        same(off, on, "filter")
        for knobs in ({"B200.VisitedSet": 1}, {"B200.VisitedSet": 1, "B200.VisitedHashEntries": 64}):
            for kname, v in knobs.items():
                idx.set_param(kname, v)
            off, on, sk = both(idx, lambda: idx.search(q, 10, want_stats=True))
            same(off, on, knobs)
        idx.set_param("B200.VisitedSet", -1)
        idx.set_param("B200.VisitedHashEntries", 0)
        for width in (8, 4):
            idx.set_param("B200.SimdWidth", width)
            off, on, _ = both(idx, lambda: idx.search(q, 10, want_stats=True))
            same(off, on, width)
        idx.set_param("B200.SimdWidth", 16)
        idx.delete(np.arange(0, files.n, 3, dtype=np.int32))
        off, on, sk = both(idx, lambda: idx.search(q, 10, want_stats=True))
        same(off, on, "tombstones")
        assert sk > 0
    finally:
        idx.close()


def test_rows_added_later_get_sketches():
    g, files, idx = golden_index("bkt_l2_2k_16")
    q = np.ascontiguousarray(g["queries"])
    rng = np.random.default_rng(3)
    try:
        idx.set_param("MaxCheck", 512)
        idx.set_param("B200.RowSketch", 1)
        idx.search(q, 10)                                       # the first 2000 rows are sketched now
        new = (files.vectors[:64] + 0.05 * rng.standard_normal((64, files.dim))).astype(np.float32)
        idx.add(new)
        off, on, sk = both(idx, lambda: idx.search(np.ascontiguousarray(new[:32]), 10, want_stats=True))
        same(off, on, "after add")
        assert sk > 0
        assert (on[0][:, 0] >= files.n).any()                   # the added rows are found
    finally:
        idx.close()


def test_kdt_and_integer_handles_refuse_the_sketch():
    g, files, idx = golden_index("kdt_l2_2k_16")
    try:
        with pytest.raises(capi.SptagB200Error):
            idx.set_param("B200.RowSketch", 1)
        assert int(idx.get_param("B200.RowSketch")) == -1
    finally:
        idx.close()


def _small_bkt(x, metric):
    import torch
    from tools import gpu_index_builder as B
    nodes, starts, graph = B.build_index(torch.from_numpy(x).cuda(), metric, seed=1)
    return B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT, metric=reflib.METRIC_OF_NAME[metric], vectors=x,
                            graph=graph, tree_starts=starts, tree_nodes=nodes)


@pytest.mark.parametrize("metric", ["Cosine", "L2"])
def test_768d_rows_take_the_sketch_by_default(metric):
    x = reflib.gen_lowrank(6000, 768, 32, 5)
    q = reflib.gen_lowrank(64, 768, 32, 6)
    if metric == "Cosine":
        x, q = reflib.normalize_rows(x), reflib.normalize_rows(q)
    idx = _small_bkt(x, metric)
    try:
        idx.set_param("MaxCheck", 2048)
        before = skipped(idx)
        auto = idx.search(q, 10, want_stats=True)
        assert skipped(idx) > before                            # auto is on for 3 KB rows
        idx.set_param("B200.RowSketch", 0)
        same(idx.search(q, 10, want_stats=True), auto, metric)
        # a larger m_Results file (the 32-register kernels)
        idx.set_param("MaxCheck", 16384)
        off, on, sk = both(idx, lambda: idx.search(q, 10, want_stats=True))
        same(off, on, "rpl32")
    finally:
        idx.close()


def test_row_with_nan_is_never_skipped():
    x = reflib.normalize_rows(reflib.gen_lowrank(3000, 64, 16, 8))
    q = reflib.normalize_rows(reflib.gen_lowrank(32, 64, 16, 9))
    import torch
    from tools import gpu_index_builder as B
    nodes, starts, graph = B.build_index(torch.from_numpy(x).cuda(), "Cosine", seed=1)
    x = x.copy()
    x[graph[graph >= 0][:50], 3] = np.nan                       # rows that are somebody's neighbours
    x[graph[graph >= 0][50:60], 1] = np.inf
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT, metric=1, vectors=x, graph=graph,
                           tree_starts=starts, tree_nodes=nodes)
    try:
        idx.set_param("MaxCheck", 1024)
        off, on, _ = both(idx, lambda: idx.search(q, 10, want_stats=True))
        same(off, on, "nan rows")
    finally:
        idx.close()
