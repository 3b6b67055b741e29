"""GPU tests of the row-sketch pass on rows whose sketches do not fit the row ring at once.  The sketch kernels stage a
graph chunk's sketch rows through the shared-memory row ring in TMA batches of ring bytes / sketch stride rows (16 at
768-d with the default ring), so a chunk of up to 32 fresh neighbours takes several batches, and a degree-64 graph row
takes two chunks.  Whatever the batching, a search must return what it returns with the sketches off (ids, distance
bits, all eight per-query counters) and what the C oracle returns."""
import numpy as np
import pytest

import reflib
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

# (dim, metric, graph degree): 768-d takes the 768-d kernels, 700-d (not a multiple of 16) the any-dimension ones
CASES = [(768, "Cosine", 32), (700, "L2", 32), (768, "L2", 64), (700, "Cosine", 64)]
# ring shapes: the default (2 stages x 2 rows: 16 sketch rows per batch at 768-d), one stage (8 per batch), 4-row stages
# (32 per batch: the whole chunk at once)
RINGS = [{}, {"B200.Stages": 1}, {"B200.StageRows": 4}]
RING_DEFAULTS = {"B200.Stages": 2, "B200.StageRows": 0}


def _index(dim, metric, degree, seed):
    import torch
    from tools import gpu_index_builder as B
    x = reflib.gen_lowrank(6000, dim, 32, seed)
    q = reflib.gen_lowrank(48, dim, 32, seed + 1)
    if metric == "Cosine":
        x, q = reflib.normalize_rows(x), reflib.normalize_rows(q)
    nodes, starts, graph = B.build_index(torch.from_numpy(x).cuda(), metric, degree=degree, cand=2 * degree, seed=1)
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    files.folder = None
    files.params = {}
    files.algo = "BKT"
    files.value_type = capi.VT_FLOAT
    files.metric = reflib.METRIC_OF_NAME[metric]
    files.vectors = np.ascontiguousarray(x)
    files.n, files.dim = x.shape
    files.graph = np.ascontiguousarray(graph)
    files.degree = files.graph.shape[1]
    files.tree_starts = np.ascontiguousarray(starts)
    files.tree_num = files.tree_starts.shape[0]
    files.nodes = np.ascontiguousarray(nodes)
    files.node_count = files.nodes.shape[0]
    files.deleted = None
    files.num_deleted = 0
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT, metric=files.metric, vectors=files.vectors,
                           graph=files.graph, tree_starts=files.tree_starts, tree_nodes=files.nodes)
    return files, np.ascontiguousarray(q), idx


def _same(a, b, what):
    for u, v in zip(a, b):
        assert np.array_equal(np.asarray(u).view(np.int32), np.asarray(v).view(np.int32)), what


@pytest.mark.parametrize("dim,metric,degree", CASES)
def test_batched_sketch_pass_matches_rows_and_oracle(dim, metric, degree):
    files, q, idx = _index(dim, metric, degree, seed=dim + degree)
    assert files.degree == degree
    try:
        idx.set_param("MaxCheck", 2048)
        idx.set_param("B200.RowSketch", 0)
        off = idx.search(q, 10, want_stats=True)
        for ring in RINGS:
            for name, v in ring.items():
                idx.set_param(name, v)
            before = int(idx.get_param("B200.RowsSkipped"))
            idx.set_param("B200.RowSketch", 1)
            on = idx.search(q, 10, want_stats=True)
            assert int(idx.get_param("B200.RowsSkipped")) > before, ring
            _same(off, on, (dim, metric, degree, ring))
            idx.set_param("B200.RowSketch", 0)
            _same(off, idx.search(q, 10, want_stats=True), ("sketches off", ring))
            for name in ring:
                idx.set_param(name, RING_DEFAULTS[name])
        o = reflib.OracleIndex(files)
        o.max_check = 2048
        ids_o, d_o, st_o = o.search(q[:16], 10)
        assert np.array_equal(off[0][:16], ids_o)
        assert np.array_equal(off[1][:16].view(np.int32), d_o.view(np.int32))
        assert np.array_equal(off[2][:16, capi.ST_NDIST], st_o[:, reflib.ST_NDIST])
    finally:
        idx.close()
