"""Golden fixtures for breadth-first tree seeding (EnableBfs != 0, BKTree.h:703-758) -- TEST INFRASTRUCTURE.

tests/golden/bfs/<name>.npz holds the UNMODIFIED REFERENCE's outputs (oracle/_ref/libsptag_ref.so) with EnableBfs set
through SetParameter, for EnableBfs in BFS_VALUES and MaxCheck in MAX_CHECKS:
  * per-query SearchIndex ids, distances and WorkSpace counters (m_iNumberOfCheckedLeaves, NGQueue / SPTQueue sizes),
  * RefineSearchIndex result lists of the first nodes (MaxCheckForRefineGraph = REFINE_MAX_CHECK),
  * on the non-quantized sets, ResultIterator::Next batches and SearchIndexIterativeFromNeareast calls of the first
    queries;
  * on ADD_SETS, the graph after one AddIndex batch (the mutation fixture's batch A, AddCEF 64, MaxCheckForRefineGraph
    512, EnableBfs 2, run by tests/cpp/mutation_ref.cpp): the refine search inside the add seeds breadth-first.
The index of a set is the committed golden index named by `base` (tests/golden/<base>.npz or quantized/<base>.npz, or the
mutation fixture's base index); the two sets made here (two trees, and float rows whose root-child distances exceed the
1.1e9 seeding sentinel) carry their own index arrays.
/root/reference is not needed to USE the fixtures.  Run (where oracle/_ref exists): python tests/golden/make_golden_bfs.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import reflib  # noqa: E402

BFS_VALUES = [1, 2, 8, -1]
MAX_CHECKS = [16, 64, 8192]
REFINE_NODES, REFINE_CEF, REFINE_MAX_CHECK = 64, 40, 512
ITER_QUERIES, ITER_BATCHES, ITER_BATCH = 8, 3, 8
NEAREST_K, NEAREST_CALLS = 10, 2
ADD_SETS, ADD_BFS, ADD_PARAMS = ("bkt_l2_2k_16",), 2, {"AddCEF": 64, "MaxCheckForRefineGraph": 512}


def index_from_npz(g, prefix=""):
    """The arrays of a committed golden index: params, vectors, graph, tree starts, nodes, optional quantizer blob."""
    if prefix:  # the mutation fixtures store their base index under base_*
        params = {str(k): str(v) for k, v in zip(g["base_param_names"].tolist(), g["base_param_values"].tolist())}
    else:
        params = {str(k): str(v) for k, v in zip(g["param_names"].tolist(), g["param_values"].tolist())}
    return dict(params=params, vectors=np.ascontiguousarray(g[prefix + "vectors"]), graph=np.ascontiguousarray(g[prefix + "graph"]),
                tree_starts=np.ascontiguousarray(g[prefix + "tree_starts"]), nodes=np.ascontiguousarray(g[prefix + "nodes"]),
                quantizer_blob=g["quantizer_blob"] if "quantizer_blob" in g.files else None)


def write_folder(ix, folder):
    """The index as the reference's SaveIndex lays it out (VectorIndex.cpp:197-222 for the ini)."""
    os.makedirs(folder, exist_ok=True)
    v, gr, ts, nd = ix["vectors"], ix["graph"], ix["tree_starts"], ix["nodes"]
    with open(os.path.join(folder, "vectors.bin"), "wb") as f:
        np.array(v.shape, np.int32).tofile(f)
        v.tofile(f)
    with open(os.path.join(folder, "graph.bin"), "wb") as f:
        np.array(gr.shape, np.int32).tofile(f)
        gr.astype(np.int32).tofile(f)
    with open(os.path.join(folder, "tree.bin"), "wb") as f:
        np.array([ts.shape[0]], np.int32).tofile(f)
        ts.astype(np.int32).tofile(f)
        np.array([nd.shape[0]], np.int32).tofile(f)
        nd.astype(np.int32).tofile(f)
    params = dict(ix["params"])
    params.update(VectorFilePath="vectors.bin", GraphFilePath="graph.bin", TreeFilePath="tree.bin")
    params.pop("DeleteVectorFilePath", None)
    qpath = params.pop("QuantizerFilePath", None)
    with open(os.path.join(folder, "indexloader.ini"), "w") as f:
        if ix["quantizer_blob"] is not None:
            qpath = qpath or "quantizer.bin"
            ix["quantizer_blob"].tofile(os.path.join(folder, qpath))
            f.write("[Quantizer]\nQuantizerFilePath=%s\n\n" % qpath)
        f.write("[Index]\n")
        for k in ("IndexAlgoType", "ValueType"):
            f.write("%s=%s\n" % (k, params.pop(k)))
        for k in sorted(params):
            f.write("%s=%s\n" % (k, params[k]))


def two_tree_data():
    return reflib.gen_lowrank(1600, 24, 6, 61)


def big_l2_data():
    # float rows scaled so that squared L2 distances to the root's children are far above 1.1e9: every root child goes
    # straight to SPTQueue
    return (reflib.gen_iid(1500, 16, 63) * np.float32(3.0e4)).astype(np.float32)


# name -> (source, queries); source: ("golden", file relative to tests/golden, npz prefix) or ("build", data, metric,
# build parameters)
SETS = {
    "algo_line_bkt": (("golden", "algo_line_bkt.npz", ""), None),
    "bkt_l2_2k_16": (("golden", "bkt_l2_2k_16.npz", ""), None),
    "bkt_cos_1500_20": (("golden", "bkt_cos_1500_20.npz", ""), None),
    "bkt_l2_dups_1k_12": (("golden", "bkt_l2_dups_1k_12.npz", ""), None),
    "pq_f32_1200_16": (("golden", "quantized/pq_f32_1200_16.npz", ""), None),
    "opq_i8_1500_24": (("golden", "quantized/opq_i8_1500_24.npz", ""), None),
    "bkt_cos_i8_1200_24": (("golden", "mutation/bkt_cos_i8_1200_24.npz", "base_"), None),
    "bkt2_cos_1600_24": (("build", two_tree_data, "Cosine", "BKTNumber=2"),
                         lambda: reflib.normalize_rows(reflib.gen_lowrank(48, 24, 6, 62))),
    "bkt_l2_big_1500_16": (("build", big_l2_data, "L2", ""),
                           lambda: (reflib.gen_iid(48, 16, 64) * np.float32(3.0e4)).astype(np.float32)),
}


def base_index(name, tmp):
    src, gen_q = SETS[name]
    if src[0] == "golden":
        g = np.load(os.path.join(HERE, src[1]))
        ix = index_from_npz(g, src[2])
        q = np.ascontiguousarray(g["base_queries"] if src[2] else g["queries"])
        return ix, q, None
    _, gen, metric, params = src
    data = np.ascontiguousarray(gen())
    folder = os.path.join(tmp, "built")
    reflib.RefIndex.build("BKT", data, metric, threads=1, params=params).save(folder)
    files = reflib.IndexFiles(folder)
    ix = dict(params=dict(files.params), vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
              nodes=files.nodes, quantizer_blob=None)
    return ix, np.ascontiguousarray(gen_q()), ix


def add_after(name, folder, tmp):
    """The reference's graph after AddIndex(batch A of tests/golden/mutation/<name>.npz) with EnableBfs = ADD_BFS."""
    import subprocess
    sys.path.insert(0, HERE)
    import make_golden_mutation as mut
    m = np.load(os.path.join(HERE, "mutation", name + ".npz"))
    driver, batch, after = os.path.join(tmp, "mutation_ref"), os.path.join(tmp, "a.bin"), os.path.join(tmp, "after")
    mut.build_driver(driver)
    np.ascontiguousarray(m["batch_a"]).tofile(batch)
    sets = []
    for k, v in dict(ADD_PARAMS, EnableBfs=ADD_BFS).items():
        sets += ["set", k, str(v)]
    subprocess.check_call([driver, folder] + sets + ["add", batch, str(m["batch_a"].shape[0]), "0", "save", after])
    return dict(add_bfs=np.int32(ADD_BFS), add_cef=np.int32(ADD_PARAMS["AddCEF"]),
                add_max_check_refine=np.int32(ADD_PARAMS["MaxCheckForRefineGraph"]),
                add_graph=reflib.IndexFiles(after).graph)


def make(name):
    with tempfile.TemporaryDirectory() as tmp:
        ix, q, own = base_index(name, tmp)
        folder = os.path.join(tmp, "idx")
        write_folder(ix, folder)
        quantized = ix["quantizer_blob"] is not None
        r = reflib.RefIndex.load(folder)
        assert r.enable_stats() == 0
        k = 3 if name == "algo_line_bkt" else 10
        out = dict(base=np.array(SETS[name][0][1] if own is None else ""), queries=q, k=np.int32(k),
                   bfs_values=np.array(BFS_VALUES, np.int32), max_checks=np.array(MAX_CHECKS, np.int32))
        if own is not None:
            names = sorted(own["params"])
            out.update(param_names=np.array(names), param_values=np.array([own["params"][n] for n in names]),
                       vectors=own["vectors"], graph=own["graph"], tree_starts=own["tree_starts"], nodes=own["nodes"])
        shape = (len(BFS_VALUES), len(MAX_CHECKS), q.shape[0], k)
        modes = ("sdc", "adc") if quantized else ("",)
        for mode in modes:
            ids_a, d_a, st_a = np.empty(shape, np.int32), np.empty(shape, np.float32), np.empty(shape[:3] + (4,), np.int32)
            if quantized:
                r.set_adc(mode == "adc")
            for a, bfs in enumerate(BFS_VALUES):
                assert r.set_param("EnableBfs", bfs) == 0
                for b, mc in enumerate(MAX_CHECKS):
                    r.set_param("MaxCheck", mc)
                    if quantized:  # raw queries: the per-query overload quantizes them (no counters there)
                        ids, dists, _ = r.search_each(q, k, threads=1)
                        ids_a[a, b], d_a[a, b] = ids, dists
                        st_a[a, b] = -1
                    else:
                        for i in range(q.shape[0]):
                            ids_a[a, b, i], d_a[a, b, i], st_a[a, b, i] = r.search_one_stats(q[i], k)
            tag = "_" + mode if mode else ""
            out["ref_ids" + tag], out["ref_dists" + tag] = ids_a, d_a
            if not quantized:
                out["ref_stats"] = st_a
        if quantized:
            r.set_adc(False)
        # RefineSearchIndex lists of the first nodes (the refine flavour: searchDuplicated = false)
        r.set_param("MaxCheckForRefineGraph", REFINE_MAX_CHECK)
        rshape = (len(BFS_VALUES), REFINE_NODES, REFINE_CEF + 1)
        rids, rd = np.empty(rshape, np.int32), np.empty(rshape, np.float32)
        for a, bfs in enumerate(BFS_VALUES):
            r.set_param("EnableBfs", bfs)
            _, i_, d_ = r.refine_nodes(0, REFINE_NODES, REFINE_CEF, 16, 1.0, threads=1)
            rids[a], rd[a] = i_, d_
        out.update(refine_nodes=np.int32(REFINE_NODES), refine_cef=np.int32(REFINE_CEF),
                   refine_max_check=np.int32(REFINE_MAX_CHECK), refine_ids=rids, refine_dists=rd)
        if not quantized:
            # ResultIterator::Next and SearchIndexIterativeFromNeareast at MaxCheck 64 on the first queries
            r.set_param("MaxCheck", 64)
            nq = min(ITER_QUERIES, q.shape[0])
            it_ids = np.full((len(BFS_VALUES), nq, ITER_BATCHES, ITER_BATCH), -2, np.int32)
            it_d = np.zeros(it_ids.shape, np.float32)
            it_n = np.zeros((len(BFS_VALUES), nq, ITER_BATCHES), np.int32)
            ne_ids = np.full((len(BFS_VALUES), nq, NEAREST_CALLS, NEAREST_K), -2, np.int32)
            ne_d = np.zeros(ne_ids.shape, np.float32)
            for a, bfs in enumerate(BFS_VALUES):
                r.set_param("EnableBfs", bfs)
                for i in range(nq):
                    it = r.iterator(q[i])
                    for c in range(ITER_BATCHES):
                        n, ids, dists, _ = it.next(ITER_BATCH)
                        it_n[a, i, c] = n
                        it_ids[a, i, c], it_d[a, i, c] = ids, dists
                    it.close()
                    s = reflib.RefNearestScan(r, q[i], NEAREST_K)
                    for c in range(NEAREST_CALLS):
                        _, ids, dists = s.next()
                        ne_ids[a, i, c], ne_d[a, i, c] = ids, dists
                    s.close()
            out.update(iter_max_check=np.int32(64), iter_counts=it_n, iter_ids=it_ids, iter_dists=it_d,
                       nearest_ids=ne_ids, nearest_dists=ne_d)
        if name in ADD_SETS:
            out.update(add_after(name, folder, tmp))
        out["ref_isa"] = np.int32(reflib.ref().ref_isa())
    os.makedirs(os.path.join(HERE, "bfs"), exist_ok=True)
    path = os.path.join(HERE, "bfs", name + ".npz")
    np.savez_compressed(path, **out)
    print("golden bfs", name, os.path.getsize(path))


if __name__ == "__main__":
    for nm in (sys.argv[1:] or SETS):
        make(nm)
