"""CPU tests: pin the C restatement's breadth-first tree seeding (EnableBfs != 0, BKTree.h:703-758: tests/oracle_bfs.c on
top of oracle/sptag_oracle.c, built by tests/oracle_bfs.py) to

1. committed golden outputs of the UNMODIFIED reference (tests/golden/bfs/*.npz, generator tests/golden/make_golden_bfs.py):
   search ids, distance bits and WorkSpace counters, RefineSearchIndex lists, ResultIterator::Next batches and
   SearchIndexIterativeFromNeareast calls;
2. the reference itself (oracle/_ref/libsptag_ref.so) on the same indexes and on random queries, where it is built.
"""
import glob
import os
import tempfile

import numpy as np
import pytest

import oracle_bfs
import reflib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_ref = pytest.mark.skipif(not reflib.have_ref(), reason="oracle/_ref not built on this box")


def bfs_sets():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "bfs", "*.npz")))


def load_set(name):
    """(fixture, IndexFiles-like view of its index, quantizer or None, queries)"""
    g = np.load(os.path.join(GOLDEN, "bfs", name + ".npz"))
    base = str(g["base"])
    src = np.load(os.path.join(GOLDEN, base)) if base else g
    prefix = "base_" if base.startswith("mutation/") else ""
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    names = src[prefix + "param_names"].tolist()
    values = src[prefix + "param_values"].tolist()
    files.folder = None
    files.params = {str(k): str(v) for k, v in zip(names, values)}
    files.algo = files.params["IndexAlgoType"]
    files.value_type = reflib.VT_OF_NAME[files.params["ValueType"]]
    files.metric = reflib.METRIC_OF_NAME[files.params.get("DistCalcMethod", "Cosine")]
    files.vectors = np.ascontiguousarray(src[prefix + "vectors"])
    files.n, files.dim = files.vectors.shape
    files.graph = np.ascontiguousarray(src[prefix + "graph"])
    files.degree = files.graph.shape[1]
    files.tree_starts = np.ascontiguousarray(src[prefix + "tree_starts"])
    files.tree_num = files.tree_starts.shape[0]
    files.nodes = np.ascontiguousarray(src[prefix + "nodes"])
    files.node_count = files.nodes.shape[0]
    files.deleted, files.num_deleted = None, 0
    files.quantizer = None
    blob = src["quantizer_blob"] if "quantizer_blob" in src.files else None
    if blob is not None:
        with tempfile.NamedTemporaryFile(suffix=".bin") as f:
            f.write(blob.tobytes())
            f.flush()
            files.quantizer = reflib.Quantizer.read(f.name)
    return g, files, blob, np.ascontiguousarray(g["queries"])


def golden_module():
    """tests/golden/make_golden_bfs.py (its write_folder lays an index out as the reference's SaveIndex does)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_bfs", os.path.join(GOLDEN, "make_golden_bfs.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def oracle_for(files, bfs, max_check=8192, adc=False):
    o = oracle_bfs.OracleBfsIndex(files, bfs)
    o.max_check = int(max_check)
    o.enable_adc = adc
    return o


@pytest.mark.parametrize("name", bfs_sets())
def test_oracle_bfs_search_matches_golden(oracle_lib, name):
    g, files, blob, q = load_set(name)
    k = int(g["k"])
    modes = ("sdc", "adc") if blob is not None else ("",)
    for mode in modes:
        tag = "_" + mode if mode else ""
        for a, bfs in enumerate(g["bfs_values"].tolist()):
            for b, mc in enumerate(g["max_checks"].tolist()):
                ids, dists, stats = oracle_for(files, bfs, mc, mode == "adc").search(q, k)
                assert np.array_equal(ids, g["ref_ids" + tag][a, b]), (name, mode, bfs, mc)
                assert np.array_equal(dists.view(np.int32), g["ref_dists" + tag][a, b].view(np.int32)), (name, mode, bfs, mc)
                if blob is None:  # the reference's WorkSpace counters
                    st = g["ref_stats"][a, b]
                    assert np.array_equal(stats[:, reflib.ST_CHECKED], st[:, 0]), (name, bfs, mc)
                    assert np.array_equal(stats[:, reflib.ST_NG_LEFT], st[:, 2]), (name, bfs, mc)
                    assert np.array_equal(stats[:, reflib.ST_SPT_LEFT], st[:, 3]), (name, bfs, mc)


@pytest.mark.parametrize("name", bfs_sets())
def test_oracle_bfs_refine_matches_golden(oracle_lib, name):
    g, files, _, _ = load_set(name)
    for a, bfs in enumerate(g["bfs_values"].tolist()):
        o = oracle_for(files, bfs)
        o.max_check_refine = int(g["refine_max_check"])
        _, ids, dists = o.refine_nodes(0, int(g["refine_nodes"]), int(g["refine_cef"]), 16, 1.0)
        assert np.array_equal(ids, g["refine_ids"][a]), (name, bfs)
        assert np.array_equal(dists.view(np.int32), g["refine_dists"][a].view(np.int32)), (name, bfs)


@pytest.mark.parametrize("name", [n for n in bfs_sets() if n not in ("pq_f32_1200_16", "opq_i8_1500_24")])
def test_oracle_bfs_iterators_match_golden(oracle_lib, name):
    g, files, _, q = load_set(name)
    nq, calls, batch = g["iter_ids"].shape[1:]
    k = g["nearest_ids"].shape[3]
    for a, bfs in enumerate(g["bfs_values"].tolist()):
        o = oracle_for(files, bfs, int(g["iter_max_check"]))
        for i in range(nq):
            it = o.iterator(q[i])
            for c in range(calls):
                n, ids, dists, _ = it.next(int(batch))
                assert n == g["iter_counts"][a, i, c], (name, bfs, i, c)
                assert np.array_equal(ids[:n], g["iter_ids"][a, i, c, :n]), (name, bfs, i, c)
                assert np.array_equal(dists[:n].view(np.int32), g["iter_dists"][a, i, c, :n].view(np.int32)), (name, bfs, i, c)
            it.close()
            it = o.iterator(q[i])
            for c in range(g["nearest_ids"].shape[2]):
                _, ids, dists = it.next_from_nearest(int(k))
                assert np.array_equal(ids, g["nearest_ids"][a, i, c]), (name, bfs, i, c)
                assert np.array_equal(dists.view(np.int32), g["nearest_dists"][a, i, c].view(np.int32)), (name, bfs, i, c)
            it.close()


def test_default_seeding_is_the_pinned_restatement(oracle_lib):
    """At EnableBfs = 0 the library is oracle/sptag_oracle.c's own search: ids, distance bits and every counter agree."""
    for name in ("bkt_l2_2k_16", "bkt2_cos_1600_24", "pq_f32_1200_16"):
        g, files, _, q = load_set(name)
        for mc in (64, 8192):
            o = reflib.OracleIndex(files)
            o.max_check = mc
            want = o.search(q, 10)
            got = oracle_for(files, 0, mc).search(q, 10)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.int32), want[1].view(np.int32))
            assert np.array_equal(got[2], want[2]), (name, mc)


def test_golden_bfs_sets_cover_the_seeding_edges(oracle_lib):
    """The fixtures exercise what the seeding's tests must cover: a second tree, root children beyond the 1.1e9
    sentinel, and results that differ from the default seeding."""
    _, files, _, _ = load_set("bkt2_cos_1600_24")
    assert files.tree_num == 2
    g, files, _, q = load_set("bkt_l2_big_1500_16")
    root = files.nodes[files.tree_starts[0]]
    child_rows = files.vectors[files.nodes[root[1]:root[2], 0]].astype(np.float64)
    d = ((q[:, None, :].astype(np.float64) - child_rows[None]) ** 2).sum(-1)
    assert (d > 1.1e9).all()
    differs = 0
    for name in bfs_sets():
        g, files, blob, q = load_set(name)
        if blob is not None:
            continue
        ids0, _, _ = oracle_for(files, 0, 64).search(q, int(g["k"]))
        differs += int((ids0 != g["ref_ids"][list(g["bfs_values"]).index(2), list(g["max_checks"]).index(64)]).any())
    assert differs >= 3


@needs_ref
@pytest.mark.parametrize("name", bfs_sets())
def test_oracle_bfs_matches_reference_on_random_queries(oracle_lib, name):
    """The reference itself at every EnableBfs of the fixtures, on the set's queries and on random ones."""
    mk = golden_module()
    g, files, blob, q = load_set(name)
    if blob is not None:
        pytest.skip("quantized sets: covered by the golden outputs (the per-query overload takes raw queries)")
    rng = np.random.default_rng(5)
    if files.value_type == reflib.VT_FLOAT:
        extra = (q[rng.integers(0, q.shape[0], 32)] + rng.standard_normal((32, files.dim)).astype(np.float32)
                 * np.float32(np.abs(q).mean())).astype(np.float32)
    else:
        extra = rng.integers(-60, 60, (32, files.dim)).astype(reflib.NP_OF_VT[files.value_type])
    qq = np.ascontiguousarray(np.concatenate([q, extra]).astype(q.dtype))
    k = int(g["k"])
    with tempfile.TemporaryDirectory() as tmp:
        ix = dict(params=files.params, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                  nodes=files.nodes, quantizer_blob=None)
        mk.write_folder(ix, tmp)
        r = reflib.RefIndex.load(tmp)
        assert r.enable_stats() == 0
        for bfs in (1, 3, -2, 1000):
            r.set_param("EnableBfs", bfs)
            for mc in (16, 256):
                r.set_param("MaxCheck", mc)
                ids, dists, stats = oracle_for(files, bfs, mc).search(qq, k)
                for i in range(qq.shape[0]):
                    ri, rd, rs = r.search_one_stats(qq[i], k)
                    assert np.array_equal(ids[i], ri), (name, bfs, mc, i)
                    assert np.array_equal(dists[i].view(np.int32), rd.view(np.int32)), (name, bfs, mc, i)
                    assert (stats[i, reflib.ST_CHECKED], stats[i, reflib.ST_NG_LEFT], stats[i, reflib.ST_SPT_LEFT]) == (
                        rs[0], rs[2], rs[3]), (name, bfs, mc, i)


# The reference's work spaces are thread-local and only ever grow (Heap::clear, WorkSpace::Reset), so their queue lengths
# depend on what the process searched before; a fresh process has exactly the lengths the case sets up.
_FRESH_REFERENCE = """
import sys
import numpy as np
import reflib
folder, qpath, k, out = sys.argv[1], sys.argv[2], int(sys.argv[3]), sys.argv[4]
q = np.load(qpath)
r = reflib.RefIndex.load(folder)
assert r.enable_stats() == 0
res = [r.search_one_stats(q[i], k) for i in range(q.shape[0])]
np.savez(out, ids=np.stack([x[0] for x in res]), dists=np.stack([x[1] for x in res]), stats=np.stack([x[2] for x in res]))
"""


@needs_ref
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt2_cos_1600_24"])
@pytest.mark.parametrize("bfs", [2, 8, -1])
def test_oracle_bfs_full_queues_match_reference(oracle_lib, name, bfs):
    """MaxCheck = MaxCheckForRefineGraph = 16: SPTQueue holds 160 and NGQueue 480 entries, so the seeding itself fills
    them and Heap::insert's full-heap branch runs during it.  The reference runs in a fresh process (see above)."""
    import subprocess
    import sys
    mk = golden_module()
    g, files, _, q = load_set(name)
    k = int(g["k"])
    o = oracle_for(files, bfs, 16)
    o.max_check_refine = 16
    ids, dists, stats = o.search(q, k)
    assert (stats[:, reflib.ST_NTREE] > 160).any()  # more tree cells than SPTQueue holds were read
    with tempfile.TemporaryDirectory() as tmp:
        params = dict(files.params, MaxCheck="16", MaxCheckForRefineGraph="16", EnableBfs=str(bfs))
        mk.write_folder(dict(params=params, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                             nodes=files.nodes, quantizer_blob=None), os.path.join(tmp, "idx"))
        np.save(os.path.join(tmp, "q.npy"), q)
        subprocess.run([sys.executable, "-c", _FRESH_REFERENCE, os.path.join(tmp, "idx"), os.path.join(tmp, "q.npy"),
                        str(k), os.path.join(tmp, "out.npz")], check=True, cwd=os.path.dirname(os.path.abspath(__file__)),
                       capture_output=True, timeout=300)
        r = np.load(os.path.join(tmp, "out.npz"))
    assert np.array_equal(ids, r["ids"]), (name, bfs)
    assert np.array_equal(dists.view(np.int32), r["dists"].view(np.int32)), (name, bfs)
    assert np.array_equal(stats[:, reflib.ST_CHECKED], r["stats"][:, 0]), (name, bfs)
    assert np.array_equal(stats[:, reflib.ST_NG_LEFT], r["stats"][:, 2]), (name, bfs)
    assert np.array_equal(stats[:, reflib.ST_SPT_LEFT], r["stats"][:, 3]), (name, bfs)
    if name == "bkt_l2_2k_16":
        assert (r["stats"][:, 3] >= 150).any()  # SPTQueue is (nearly) full at exit
