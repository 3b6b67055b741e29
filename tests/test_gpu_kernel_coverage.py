"""GPU tests: one case per reachable search-family kernel instantiation (search_kernels.cuh, kernel_select_impl.cuh).

Each case builds its index here (tools/gpu_index_builder, or a committed PQ fixture), runs one search or iterator
schedule on the device and checks
  * ids, distance bits and the WorkSpace counters against the C restatement (oracle/sptag_oracle.c, or its EnableBfs
    build tests/oracle_bfs.py), or the iterator results call by call, and
  * that B200.LastSearchKernel names the instantiation the selectors predict for the case's parameters
    (sptag_b200_debug_kernel_for).
tests/test_kernel_coverage.py proves on the CPU that CASES reaches every instantiation the selectors can return.
The fixtures of tests/golden/kernels (the reference's own outputs on KDT-cosine and uint8 indexes) run here too.
"""
import collections
import glob
import os
import sys

import numpy as np
import pytest

import reflib
from make_test_data import _int8_lowrank, _int16_lowrank, _norm_i8, _norm_i16, _uint8_lowrank

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
VT = {"f32": reflib.VT_FLOAT, "i8": reflib.VT_INT8, "u8": reflib.VT_UINT8, "i16": reflib.VT_INT16, "pq": reflib.VT_UINT8}
METRIC = {"L2": 0, "Cosine": 1}
N_ROWS, N_QUERIES = 2000, 32
# integer rows: int8 / uint8 run one 64-, 32- and 16-element step and 12 scalar ones; int16 three 32-element steps, one
# 16- and 8-element step and 4 scalar ones.  Float: 27 = 16 + 8 + 3.
INT_DIM, FLOAT_DIM = 124, 27
PQ_FIXTURES = {"pq_f32": "pq_f32_1200_16", "pq_opq_i8": "opq_i8_1500_24"}

# recipe: (element type, metric, algorithm, dimension); "pq_*" recipes are the committed quantized fixtures.
# family: "search", "iterate" (ResultIterator::Next) or "nearest" (the first SearchIndexIterativeFromNeareast call).
# k: K of the search, the first iterator batch, or the k of SearchIndexIterativeFromNeareast.
# mc: MaxCheck.  qps: B200.QueriesPerSM (0: automatic, 14 slots for these batch sizes on 128-d float rows).
Case = collections.namedtuple("Case", "recipe family k mc simd bfs sketch qps")


def _case(vt, metric, algo, dim, family="search", k=10, mc=1024, simd=16, bfs=0, sketch=0, qps=0):
    return Case((vt, metric, algo, dim), family, k, mc, simd, bfs, sketch, qps)


def _cases():
    c = []
    for m in ("L2", "Cosine"):
        # 512-byte float rows, BKT: the 20-slot and 16-slot fast paths, then the 32- and 64-register m_Results files
        c += [_case("f32", m, "BKT", 128, mc=4096, qps=17), _case("f32", m, "BKT", 128, mc=4096),
              _case("f32", m, "BKT", 128, mc=16384), _case("f32", m, "BKT", 128, k=1100, mc=2048)]
        # KD-trees have no m_Results gate: one kernel per dimension class (and the 20-slot one at 128)
        c += [_case("f32", m, "KDT", 128, mc=2048, qps=17), _case("f32", m, "KDT", 128, mc=8192),
              _case("f32", m, "KDT", 768, mc=2048)]
        c += [_case("f32", m, "BKT", 768, mc=2048), _case("f32", m, "BKT", 768, k=40, mc=16384),
              _case("f32", m, "BKT", 768, mc=32768)]
    # generic-dimension float kernels: tail-heavy rows, and 128 / 768-d rows at SimdWidth 8
    c += [_case("f32", "L2", "BKT", FLOAT_DIM, mc=8192), _case("f32", "L2", "BKT", 128, mc=16384, simd=8),
          _case("f32", "L2", "BKT", 768, mc=32768, simd=8), _case("f32", "L2", "KDT", FLOAT_DIM, mc=4096),
          _case("f32", "Cosine", "BKT", 128, mc=2048, simd=8), _case("f32", "Cosine", "BKT", FLOAT_DIM, k=600, mc=1024),
          _case("f32", "Cosine", "BKT", FLOAT_DIM, k=1500, mc=8192), _case("f32", "Cosine", "KDT", 768, mc=2048, simd=8)]
    # EnableBfs: every float dimension takes the generic-dimension bfs:: kernels
    c += [_case("f32", "L2", "BKT", FLOAT_DIM, mc=4096, bfs=1), _case("f32", "L2", "BKT", 128, mc=16384, bfs=2),
          _case("f32", "L2", "BKT", 768, k=1100, mc=1024, bfs=1), _case("f32", "Cosine", "BKT", 128, mc=2048, bfs=1),
          _case("f32", "Cosine", "BKT", FLOAT_DIM, k=40, mc=16384, bfs=1),
          _case("f32", "Cosine", "BKT", FLOAT_DIM, mc=32768, bfs=1)]
    # row sketches (B200.RowSketch 1): 768-d rows and every other dimension
    for m in ("L2", "Cosine"):
        c += [_case("f32", m, "BKT", 768, mc=4096, sketch=1), _case("f32", m, "BKT", 768, mc=16384, sketch=1),
              _case("f32", m, "BKT", 768, k=1100, mc=4096, sketch=1)]
    c += [_case("f32", "L2", "BKT", FLOAT_DIM, mc=4096, sketch=1), _case("f32", "L2", "BKT", 128, k=600, mc=2048, sketch=1),
          _case("f32", "L2", "BKT", FLOAT_DIM, mc=32768, sketch=1), _case("f32", "Cosine", "BKT", 128, mc=4096, sketch=1),
          _case("f32", "Cosine", "BKT", FLOAT_DIM, mc=16384, sketch=1),
          _case("f32", "Cosine", "BKT", 128, k=1500, mc=1024, simd=8, sketch=1)]
    # integer rows: BKT at the three m_Results files (K > 32 keeps the results unordered in HBM), KDT, EnableBfs
    for vt in ("i8", "u8", "i16"):
        for m in ("L2", "Cosine"):
            big_k = m == "Cosine"
            c += [_case(vt, m, "BKT", INT_DIM, mc=4096),
                  _case(vt, m, "BKT", INT_DIM, k=700 if big_k else 10, mc=1024 if big_k else 16384),
                  _case(vt, m, "BKT", INT_DIM, k=1100 if big_k else 10, mc=8192 if big_k else 32768),
                  _case(vt, m, "KDT", INT_DIM, k=40 if big_k else 10, mc=4096),
                  _case(vt, m, "BKT", INT_DIM, k=40 if big_k else 10, mc=4096, bfs=1),
                  _case(vt, m, "BKT", INT_DIM, mc=16384, bfs=1),
                  _case(vt, m, "BKT", INT_DIM, k=1100 if big_k else 10, mc=32768 if not big_k else 2048, bfs=1)]
    # PQ / OPQ codes (BKT + L2): the 16- and 32-register m_Results files, with and without EnableBfs
    c += [Case(("pq_f32",), "search", 10, 8192, 16, 0, 0, 0), Case(("pq_opq_i8",), "search", 700, 1024, 16, 0, 0, 0),
          Case(("pq_opq_i8",), "search", 40, 4096, 16, 1, 0, 0), Case(("pq_f32",), "search", 10, 16384, 16, 1, 0, 0)]
    # iterators (BKT only): both families, both m_Results files, with and without EnableBfs
    iter_dim = {"f32": 128, "i8": INT_DIM, "u8": INT_DIM, "i16": INT_DIM}
    for vt in ("f32", "i8", "u8", "i16"):
        for m in ("L2", "Cosine"):
            dim = FLOAT_DIM if (vt, m) == ("f32", "Cosine") else iter_dim[vt]
            for fam in ("iterate", "nearest"):
                for bfs in (0, 1):
                    c += [_case(vt, m, "BKT", dim, family=fam, k=10, mc=1024, bfs=bfs),
                          _case(vt, m, "BKT", dim, family=fam, k=600 if bfs else 16, mc=1024 if bfs else 16384, bfs=bfs)]
    return c


CASES = _cases()


def case_id(c):
    r = "-".join(str(v) for v in c.recipe)
    extra = "".join(s for s, on in (("-simd8", c.simd == 8), ("-bfs%d" % c.bfs, c.bfs), ("-sketch", c.sketch),
                                    ("-qps%d" % c.qps, c.qps)) if on)
    return "%s-%s-k%d-mc%d%s" % (r, c.family, c.k, c.mc, extra)


def case_launch(c):
    """The selector inputs of the case's launch (the keyword arguments of capi.debug_kernel_for)."""
    from sptag_b200 import capi
    if c.recipe[0].startswith("pq"):
        vt, metric, algo, dim, quantized = reflib.VT_UINT8, 0, capi.ALGO_BKT, 0, True
    else:
        vt, metric, algo, dim = VT[c.recipe[0]], METRIC[c.recipe[1]], reflib.ALGO_OF_NAME[c.recipe[2]], c.recipe[3]
        quantized = False
    family = {"search": capi.FAMILY_SEARCH, "iterate": capi.FAMILY_ITERATE, "nearest": capi.FAMILY_NEAREST_FIRST}[c.family]
    fast128 = (family == capi.FAMILY_SEARCH and vt == reflib.VT_FLOAT and not quantized and dim == 128 and c.simd == 16
               and not c.sketch and not (c.bfs and algo == capi.ALGO_BKT))
    slots = (c.qps or 14) if fast128 else 0
    return dict(value_type=vt, metric=metric, algo=algo, dim=dim, simd_width=c.simd, enable_bfs=c.bfs,
                row_sketch=c.sketch, quantized=quantized, mres_cap=max(c.mc // 16, c.k), slots=slots, family=family)


def predicted_kernel(c):
    from sptag_b200 import capi
    return capi.debug_kernel_for(**case_launch(c))


# ---------------------------------------------------------------------------------------------------------------------
# index recipes
# ---------------------------------------------------------------------------------------------------------------------
def _norm_u8(x):
    # Utils::Normalize for uint8 (CommonUtils.h:62-76): base = 255, truncation toward zero
    v = x.astype(np.float64)
    n = np.sqrt((v * v).sum(1, keepdims=True))
    return np.trunc(v / n * 255).astype(np.uint8)


def recipe_rows(vt, metric, dim, n, seed):
    """Rows of a recipe's element type; cosine rows are normalised to the type's base, as the reference expects."""
    cos = metric == "Cosine"
    if vt == "f32":
        x = reflib.gen_lowrank(n, dim, 12, seed)
        return reflib.normalize_rows(x) if cos else x
    if vt == "i8":
        x = _int8_lowrank(n, dim, 12, seed)
        return _norm_i8(x) if cos else x
    if vt == "u8":
        x = _uint8_lowrank(n, dim, 12, seed)
        return _norm_u8(x) if cos else x
    x = _int16_lowrank(n, dim, 12, seed)
    return _norm_i16(x) if cos else x


def files_of(algo, vectors, metric, graph, nodes, tree_starts, quantizer=None):
    """A reflib.IndexFiles over in-memory arrays (what OracleIndex reads)."""
    f = reflib.IndexFiles.__new__(reflib.IndexFiles)
    f.folder, f.params, f.algo = None, {}, algo
    f.vectors = np.ascontiguousarray(vectors)
    f.value_type = {np.dtype(np.float32): reflib.VT_FLOAT, np.dtype(np.int8): reflib.VT_INT8,
                    np.dtype(np.uint8): reflib.VT_UINT8, np.dtype(np.int16): reflib.VT_INT16}[f.vectors.dtype]
    f.metric = metric
    f.n, f.dim = f.vectors.shape
    f.graph = np.ascontiguousarray(graph, np.int32)
    f.degree = f.graph.shape[1]
    f.tree_starts = np.ascontiguousarray(tree_starts, np.int32)
    f.tree_num = f.tree_starts.shape[0]
    f.nodes = np.ascontiguousarray(nodes, np.int32)
    f.node_count = f.nodes.shape[0]
    f.deleted, f.num_deleted = None, 0
    f.quantizer = quantizer
    return f


class Recipe:
    def __init__(self, files, queries, blob=None):
        self.files, self.queries, self.blob = files, queries, blob


def _build(recipe, tmpdir):
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import gpu_index_builder as gib
    if recipe[0].startswith("pq"):
        import test_oracle_pin as pin
        g = np.load(os.path.join(GOLDEN, "quantized", PQ_FIXTURES[recipe[0]] + ".npz"))
        files = reflib.IndexFiles.__new__(reflib.IndexFiles)
        pin._files_from_npz(files, g)
        qpath = os.path.join(tmpdir, recipe[0] + ".quantizer.bin")
        g["quantizer_blob"].tofile(qpath)
        files.quantizer = reflib.Quantizer.read(qpath)
        return Recipe(files, np.ascontiguousarray(g["queries"][:N_QUERIES]), g["quantizer_blob"])
    vt, metric, algo, dim = recipe
    seed = 1000 + 97 * sorted(VT).index(vt) + 13 * dim + (5 if metric == "Cosine" else 0) + (3 if algo == "KDT" else 0)
    n = 1500 if dim == 768 else N_ROWS
    x = recipe_rows(vt, metric, dim, n, seed)
    q = recipe_rows(vt, metric, dim, N_QUERIES, seed + 1)
    xt = torch.from_numpy(x.astype(np.float32)).cuda()
    nodes, starts, graph = gib.build_index(xt, metric=metric, degree=32, cand=64, algo=algo, seed=seed)
    del xt
    return Recipe(files_of(algo, x, METRIC[metric], graph, nodes, starts), q)


@pytest.fixture(scope="module")
def recipes(tmp_path_factory):
    tmpdir = str(tmp_path_factory.mktemp("kernel_coverage"))
    cache = {}

    def get(recipe):
        if recipe not in cache:
            cache[recipe] = _build(recipe, tmpdir)
        return cache[recipe]
    return get


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
def _device_index(r, c):
    from sptag_b200 import B200Index, capi
    f = r.files
    idx = B200Index.create(algo=capi.ALGO_KDT if f.algo == "KDT" else capi.ALGO_BKT, value_type=f.value_type,
                           metric=f.metric, vectors=f.vectors, graph=f.graph, tree_starts=f.tree_starts,
                           tree_nodes=f.nodes, device=0)
    if r.blob is not None:
        idx.set_quantizer(r.blob.tobytes())
    idx.set_param("MaxCheck", c.mc)
    idx.set_param("B200.SimdWidth", c.simd)
    if c.bfs:
        idx.set_param("EnableBfs", c.bfs)
    if f.value_type == reflib.VT_FLOAT and f.quantizer is None and f.algo == "BKT":
        idx.set_param("B200.RowSketch", c.sketch)  # 768-d rows take the sketches by default
    if c.qps:
        idx.set_param("B200.QueriesPerSM", c.qps)
    return idx


def _oracle(r, c):
    if c.bfs:
        import oracle_bfs
        o = oracle_bfs.OracleBfsIndex(r.files, c.bfs, simd_width=c.simd)
    else:
        o = reflib.OracleIndex(r.files, simd_width=c.simd)
    o.max_check = c.mc
    return o


def _check_search(idx, o, q, c):
    from sptag_b200 import capi
    ids, dists, stats = idx.search(q, c.k, want_stats=True)
    ids_o, d_o, st_o = o.search(q, c.k)
    bad = np.nonzero((ids != ids_o).any(axis=1))[0]
    assert bad.size == 0, "%d/%d queries differ, first %d: gpu %s oracle %s" % (bad.size, q.shape[0], bad[0], ids[bad[0]],
                                                                                ids_o[bad[0]])
    assert np.array_equal(dists.view(np.int32), d_o.view(np.int32))
    pairs = [(capi.ST_CHECKED, reflib.ST_CHECKED), (capi.ST_NG_LEFT, reflib.ST_NG_LEFT),
             (capi.ST_SPT_LEFT, reflib.ST_SPT_LEFT), (capi.ST_NDIST, reflib.ST_NDIST),
             (capi.ST_NEXPAND, reflib.ST_NEXPAND), (capi.ST_NTREE, reflib.ST_NTREE)]
    if not c.bfs:  # the breadth-first seeding counts its tree leaves differently (as tests/test_gpu_bfs.py)
        pairs.append((capi.ST_TREE_CHECKED, reflib.ST_TREE_CHECKED))
    for a, b in pairs:
        assert np.array_equal(stats[:, a], st_o[:, b]), ("stat", a)
    assert not stats[:, capi.ST_FLAGS].any()


def _check_iterate(idx, o, q, c):
    its = idx.iterators(q)
    oits = [o.iterator(qq) for qq in q]
    try:
        for step, b in enumerate([c.k, c.k, max(1, c.k // 2), c.k]):  # a batch never grows past the previous count
            counts, ids, dists, relaxed = its.next(b)
            for i, oi in enumerate(oits):
                cnt, io, do, ro = oi.next(b)
                assert counts[i] == cnt, (step, i)
                assert np.array_equal(ids[i, :cnt], io[:cnt]), (step, i)
                assert np.array_equal(dists[i, :cnt].view(np.int32), do[:cnt].view(np.int32)), (step, i)
                assert bool(relaxed[i]) == ro, (step, i)
    finally:
        its.close()
        for oi in oits:
            oi.close()


def _check_nearest(idx, o, q, c):
    its = idx.iterators(q)
    oits = [o.iterator(qq) for qq in q]
    try:
        found, ids, dists = its.next_from_nearest(c.k)
        name = idx.get_param("B200.LastSearchKernel")
        for i, oi in enumerate(oits):
            ok, io, do = oi.next_from_nearest(c.k)
            assert bool(found[i]) == ok, i
            assert np.array_equal(ids[i], io), i
            assert np.array_equal(dists[i].view(np.int32), do.view(np.int32)), i
    finally:
        its.close()
        for oi in oits:
            oi.close()
    return name


@pytest.mark.parametrize("c", CASES, ids=[case_id(c) for c in CASES])
def test_kernel_instantiation_bit_exact(recipes, c):
    r = recipes(c.recipe)
    q = r.queries
    idx = _device_index(r, c)
    try:
        o = _oracle(r, c)
        if c.family == "search":
            _check_search(idx, o, q, c)
            name = idx.get_param("B200.LastSearchKernel")
        elif c.family == "iterate":
            _check_iterate(idx, o, q, c)
            name = idx.get_param("B200.LastSearchKernel")
        else:
            name = _check_nearest(idx, o, q, c)
        assert name == predicted_kernel(c)
    finally:
        idx.close()


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own outputs on the combinations the oracle was never pinned on (tests/golden/make_golden_kernels.py)
# ---------------------------------------------------------------------------------------------------------------------
def kernel_golden_cases():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "kernels", "*.npz")))


@pytest.mark.parametrize("name", kernel_golden_cases())
def test_gpu_matches_reference_kernel_golden(name):
    from sptag_b200 import B200Index, capi
    import test_oracle_pin as pin
    g = np.load(os.path.join(GOLDEN, "kernels", name + ".npz"))
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    pin._files_from_npz(files, g)
    idx = B200Index.create(algo=capi.ALGO_KDT if files.algo == "KDT" else capi.ALGO_BKT, value_type=files.value_type,
                           metric=files.metric, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                           tree_nodes=files.nodes, device=0)
    try:
        q = np.ascontiguousarray(g["queries"])
        for i, (k, mc) in enumerate(g["runs"].tolist()):
            idx.set_param("MaxCheck", mc)
            ids, dists, stats = idx.search(q, k, want_stats=True)
            assert np.array_equal(ids, g["ref_ids_%d" % i]), (name, k, mc)
            assert np.array_equal(dists.view(np.int32), g["ref_dists_%d" % i].view(np.int32)), (name, k, mc)
            st = g["ref_stats_%d" % i]
            assert np.array_equal(stats[:, capi.ST_CHECKED], st[:, 0]), (name, k, mc)
            assert np.array_equal(stats[:, capi.ST_TREE_CHECKED], st[:, 1]), (name, k, mc)
            assert np.array_equal(stats[:, capi.ST_NG_LEFT], st[:, 2]), (name, k, mc)
            assert np.array_equal(stats[:, capi.ST_SPT_LEFT], st[:, 3]), (name, k, mc)
    finally:
        idx.close()
