"""Golden fixtures for index mutation (AddIndex / DeleteIndex / DeleteIndex(vectors)) -- TEST INFRASTRUCTURE.

For each committed search fixture below (an index built by the unmodified reference) this runs the UNMODIFIED REFERENCE
(tests/cpp/mutation_ref.cpp, linked with oracle/_ref/libsptag_ref.so) through one fixed sequence of calls:

  AddIndex(batch A)            200 rows: fresh, exact copies of indexed rows, near-copies            -> state 1
  DeleteIndex(id) x ids        live ids, a repeat, an out-of-range id                               (codes recorded)
  DeleteIndex(vectors)         copies of indexed rows (duplicate groups included), one OpenMP thread
  AddIndex(batch B)            50 rows                                                               -> state 2

with AddCEF 64 and MaxCheckForRefineGraph 512 (fewer adds than AddCountForRebuild, so the tree is never rebuilt), and
writes tests/golden/mutation/<case>.npz: the inputs, the graph / vectors after each state, the tombstones, and the
reference's searches on both states (MaxCheck 512 and 2048, searchDeleted 0 and 1).  /root/reference is not needed to
USE the fixtures.
Run (where oracle/_ref exists):  python tests/golden/make_golden_mutation.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import reflib  # noqa: E402

# case -> (fixture, AddIndex's p_normalized); fixture None: an int8 Cosine index the reference builds here (stored in the
# npz), so the integer branches of Normalize (base 127) and of the distance trees are covered
CASES = {
    "bkt_cos_i8_1200_24": (None, 0),
    "bkt_l2_2k_16": ("bkt_l2_2k_16", 0),
    "bkt_cos_1500_20": ("bkt_cos_1500_20", 0),
    "bkt_cos_1500_20_normalized": ("bkt_cos_1500_20", 1),
    "kdt_l2_2k_16": ("kdt_l2_2k_16", 0),
    "bkt_l2_dups_1k_12": ("bkt_l2_dups_1k_12", 0),
}
PARAMS = {"AddCEF": 64, "MaxCheckForRefineGraph": 512}
MAX_CHECKS = (512, 2048)
K = 10


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "mutation_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def inputs(vectors, normalized, seed):
    """Batch A: 120 fresh rows, 40 exact copies of indexed rows, 40 near-copies; batch B: 50 fresh rows; the ids and
    vectors to delete."""
    rng = np.random.default_rng(seed)
    n, dim = vectors.shape
    if vectors.dtype == np.int8:
        x = vectors
        fresh = rng.integers(-127, 128, (120, dim)).astype(np.int8)
        copies = x[rng.choice(n, 40, replace=False)]
        near = np.clip(x[rng.choice(n, 40, replace=False)].astype(np.int32) + rng.integers(-1, 2, (40, dim)), -127,
                       127).astype(np.int8)
        batch_a = np.concatenate([fresh, copies, near])[rng.permutation(200)]
        batch_b = rng.integers(-127, 128, (50, dim)).astype(np.int8)
        live = rng.choice(n + 200, 30, replace=False).astype(np.int32)
        del_ids = np.concatenate([live, live[:3], np.array([n + 200 + 5], np.int32)]).astype(np.int32)
        del_vecs = np.concatenate([x[rng.choice(n, 12, replace=False)], batch_a[:4]])
        return batch_a, batch_b, del_ids, del_vecs
    x = vectors.astype(np.float32)
    scale = float(np.abs(x).mean()) * 2 + 1e-3
    fresh = (rng.standard_normal((120, dim)) * scale).astype(np.float32)
    copies = x[rng.choice(n, 40, replace=False)]
    near = x[rng.choice(n, 40, replace=False)] + (rng.standard_normal((40, dim)) * scale * 1e-3).astype(np.float32)
    batch_a = np.concatenate([fresh, copies, near])[rng.permutation(200)]
    batch_b = (rng.standard_normal((50, dim)) * scale).astype(np.float32)
    if normalized:  # the caller promises unit rows
        batch_a /= np.linalg.norm(batch_a, axis=1, keepdims=True)
        batch_b /= np.linalg.norm(batch_b, axis=1, keepdims=True)
    live = rng.choice(n + 200, 30, replace=False).astype(np.int32)
    del_ids = np.concatenate([live, live[:3], np.array([n + 200 + 5], np.int32)]).astype(np.int32)
    del_vecs = np.concatenate([x[rng.choice(n, 12, replace=False)], batch_a[:4]]).astype(np.float32)
    return batch_a, batch_b, del_ids, del_vecs


def searches(folder, queries):
    r = reflib.RefIndex.load(folder)
    ids, dists = [], []
    for mc in MAX_CHECKS:
        r.set_param("MaxCheck", mc)
        for sd in (0, 1):
            i, d = r.search_flag(queries, K, sd, threads=1)
            ids.append(i)
            dists.append(d)
    return np.stack(ids).reshape(len(MAX_CHECKS), 2, -1, K), np.stack(dists).reshape(len(MAX_CHECKS), 2, -1, K)


def build_int8_cosine():
    """An int8 Cosine BKT index built by the reference from seeded rows (BuildIndex normalises them, base 127)."""
    rng = np.random.default_rng(20261016)
    data = rng.integers(-127, 128, (1200, 24)).astype(np.int8)
    with tempfile.TemporaryDirectory() as tmp:
        reflib.RefIndex.build("BKT", data, "Cosine", threads=1).save(tmp)
        f = reflib.IndexFiles(tmp)
        nodes = f.nodes[:f.node_count]  # as tree.bin holds them (IndexFiles appends LoadTrees' sentinel)
        return {"vectors": f.vectors.copy(), "graph": f.graph.copy(), "nodes": nodes.copy(),
                "tree_starts": f.tree_starts.copy(), "queries": rng.integers(-127, 128, (64, 24)).astype(np.int8),
                "param_names": np.array(["IndexAlgoType", "DistCalcMethod", "ValueType"]),
                "param_values": np.array(["BKT", "Cosine", "Int8"])}


def iterator_scans(folder, queries, rounds=3, batch=8):
    """GetIterator(query, searchDeleted = false) + `rounds` x Next(batch) per query, MaxCheck 512."""
    r = reflib.RefIndex.load(folder)
    r.set_param("MaxCheck", 512)
    counts = np.zeros((len(queries), rounds), np.int32)
    ids = np.full((len(queries), rounds, batch), -1, np.int32)
    dists = np.zeros((len(queries), rounds, batch), np.float32)
    for i, q in enumerate(queries):
        it = r.iterator(q, False)
        for j in range(rounds):
            c, ids[i, j], dists[i, j], _ = it.next(batch)
            counts[i, j] = c
        it.close()
    return counts, ids, dists


def make(case, driver):
    from tools.gpu_index_builder import save_index_folder
    fixture, normalized = CASES[case]
    g = np.load(os.path.join(HERE, fixture + ".npz")) if fixture else build_int8_cosine()
    params = dict(zip(g["param_names"].tolist(), g["param_values"].tolist()))
    a, b, del_ids, del_vecs = inputs(g["vectors"], normalized, 20261015)
    q = np.ascontiguousarray(g["queries"])
    with tempfile.TemporaryDirectory() as tmp:
        src, s1, s2 = (os.path.join(tmp, d) for d in ("src", "s1", "s2"))
        save_index_folder(src, g["vectors"], g["graph"], g["nodes"], g["tree_starts"], params["DistCalcMethod"],
                          algo=params["IndexAlgoType"], value_type=params["ValueType"])
        for name, arr in (("a", a), ("b", b), ("ids", del_ids), ("dv", del_vecs)):
            arr.tofile(os.path.join(tmp, name + ".bin"))
        sets = []
        for k, v in PARAMS.items():
            sets += ["set", k, str(v)]
        t = lambda nm: os.path.join(tmp, nm)  # noqa: E731
        subprocess.check_call([driver, src] + sets + ["add", t("a.bin"), "200", str(normalized), "save", s1,
                                                      "del", t("ids.bin"), str(len(del_ids)), t("codes.bin"),
                                                      "delvec", t("dv.bin"), str(len(del_vecs)),
                                                      "add", t("b.bin"), "50", str(normalized), "save", s2])
        f1, f2 = reflib.IndexFiles(s1), reflib.IndexFiles(s2)
        codes = np.fromfile(t("codes.bin"), np.int32)
        ids1, d1 = searches(s1, q)
        ids2, d2 = searches(s2, q)
        extra = {}
        if params["IndexAlgoType"] == "BKT":  # iterators opened after the deletes (KDT has none)
            extra["it_counts"], extra["it_ids"], extra["it_dists"] = iterator_scans(s2, q[:8])
        if fixture is None:
            extra.update({"base_" + k: g[k] for k in g})
    os.makedirs(os.path.join(HERE, "mutation"), exist_ok=True)
    out = os.path.join(HERE, "mutation", case + ".npz")
    np.savez_compressed(out, fixture=np.array(fixture or ""), normalized=np.int32(normalized),
                        param_names=np.array(list(PARAMS)), param_values=np.array(list(PARAMS.values()), np.int32),
                        batch_a=a, batch_b=b, del_ids=del_ids, del_vecs=del_vecs, queries=q, max_checks=np.array(MAX_CHECKS, np.int32),
                        k=np.int32(K), graph1=f1.graph, added1=f1.vectors[len(g["vectors"]):], graph2=f2.graph,
                        added2=f2.vectors[len(g["vectors"]) + 200:],
                        deleted2=f2.deleted, num_deleted2=np.int32(f2.num_deleted), del_codes=codes,
                        ids1=ids1, dists1=d1, ids2=ids2, dists2=d2, **extra)
    print("golden mutation", case, "rows changed by A:", int((f1.graph[:len(g["graph"])] != g["graph"]).any(1).sum()),
          "tombstones:", f2.num_deleted, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as d:
        drv = os.path.join(d, "mutation_ref")
        build_driver(drv)
        for c in (sys.argv[1:] or sorted(CASES)):
            make(c, drv)
