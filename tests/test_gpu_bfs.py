"""GPU tests of EnableBfs: BKT breadth-first tree seeding (BKTree.h:703-758), run by the bfs:: kernels.  Every result is
compared bit for bit with the unmodified reference's golden outputs (tests/golden/bfs, make_golden_bfs.py) and with the
C restatement (tests/oracle_bfs.py: oracle/sptag_oracle.c with the seeding of tests/oracle_bfs.c), counters included: search, filtered and tombstoned search, both visited sets,
RefineSearchIndex, iterators, PQ / OPQ, the ini round trip, parameter changes between calls and the drop-in
SPTAG::B200::Index."""
import os
import subprocess

import numpy as np
import pytest

import reflib
import test_oracle_pin_bfs as pin

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SETS = pin.bfs_sets()
QUANTIZED = ("opq_i8_1500_24", "pq_f32_1200_16")
PLAIN = [n for n in SETS if n not in QUANTIZED]
PARAM_NOT_FOUND = 0x0010  # include/sptag_b200.h


def stat_pairs():
    from sptag_b200 import capi
    return [(capi.ST_CHECKED, reflib.ST_CHECKED), (capi.ST_NG_LEFT, reflib.ST_NG_LEFT),
            (capi.ST_SPT_LEFT, reflib.ST_SPT_LEFT), (capi.ST_NDIST, reflib.ST_NDIST),
            (capi.ST_NEXPAND, reflib.ST_NEXPAND), (capi.ST_NTREE, reflib.ST_NTREE)]


def gpu_index(files, blob, **params):
    from sptag_b200 import B200Index, capi
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=files.value_type, metric=files.metric, vectors=files.vectors,
                           graph=files.graph, tree_starts=files.tree_starts, tree_nodes=files.nodes, device=0)
    if blob is not None:
        idx.set_quantizer(blob.tobytes())
    for k, v in params.items():
        idx.set_param(k, v)
    return idx


def same(ids, dists, ids_ref, dists_ref, tag):
    bad = np.nonzero((ids != ids_ref).any(axis=1))[0]
    assert bad.size == 0, "%s: %d queries differ, first %d: gpu %s ref %s" % (tag, bad.size, bad[0], ids[bad[0]],
                                                                             ids_ref[bad[0]])
    assert np.array_equal(dists.view(np.int32), np.asarray(dists_ref, np.float32).view(np.int32)), tag


def check_against_oracle(idx, files, q, k, bfs, mc, adc=False, tag=""):
    ids, dists, stats = idx.search(q, k, want_stats=True)
    ids_o, d_o, st_o = pin.oracle_for(files, bfs, mc, adc).search(q, k)
    same(ids, dists, ids_o, d_o, "%s oracle bfs=%d mc=%d k=%d" % (tag, bfs, mc, k))
    for a, b in stat_pairs():
        assert np.array_equal(stats[:, a], st_o[:, b]), (tag, bfs, mc, k, "stat", a)
    return ids, dists, stats


def check_golden_search(idx, g, files, blob, q, tag=""):
    k = int(g["k"])
    for mode in (("sdc", "adc") if blob is not None else ("",)):
        if blob is not None:
            idx.set_param("EnableADC", 1 if mode == "adc" else 0)
        sfx = "_" + mode if mode else ""
        for a, bfs in enumerate(g["bfs_values"].tolist()):
            idx.set_param("EnableBfs", bfs)
            for b, mc in enumerate(g["max_checks"].tolist()):
                idx.set_param("MaxCheck", mc)
                ids, dists, stats = check_against_oracle(idx, files, q, k, bfs, mc, mode == "adc", tag)
                same(ids, dists, g["ref_ids" + sfx][a, b], g["ref_dists" + sfx][a, b],
                     "%s golden %s bfs=%d mc=%d" % (tag, mode, bfs, mc))
                if blob is None:
                    from sptag_b200 import capi
                    st = g["ref_stats"][a, b]
                    assert np.array_equal(stats[:, capi.ST_CHECKED], st[:, 0]), (tag, bfs, mc)
                    assert np.array_equal(stats[:, capi.ST_NG_LEFT], st[:, 2]), (tag, bfs, mc)
                    assert np.array_equal(stats[:, capi.ST_SPT_LEFT], st[:, 3]), (tag, bfs, mc)


# 1 + 6: every set (PQ / OPQ with SDC and ADC) x EnableBfs x MaxCheck, against the reference and the oracle
@pytest.mark.parametrize("name", SETS)
def test_search_matches_reference(name):
    g, files, blob, q = pin.load_set(name)
    idx = gpu_index(files, blob)
    try:
        check_golden_search(idx, g, files, blob, q, name)
    finally:
        idx.close()


@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("k", [1, 100, 2048])
def test_result_counts_match_oracle(name, k):
    g, files, blob, q = pin.load_set(name)
    if blob is not None and k > 1024:
        pytest.skip("quantized indexes: K up to 1024")
    idx = gpu_index(files, blob)
    try:
        for bfs in (2, -1, 8):
            idx.set_param("EnableBfs", bfs)
            for mc in (64, 8192):
                idx.set_param("MaxCheck", mc)
                check_against_oracle(idx, files, q, k, bfs, mc, tag=name)
    finally:
        idx.close()


# 128- and 768-d float rows normally run their own kernels; with EnableBfs they run the generic-dimension ones
@pytest.mark.parametrize("name", ["bkt_l2_10k_128", "bkt_cos_3k_768"])
def test_specialised_dimensions_route_to_the_bfs_kernels(name):
    from sptag_b200 import B200Index
    from conftest import data_folder
    folder = data_folder(name)
    files = reflib.IndexFiles(folder)
    q = np.ascontiguousarray(np.load(os.path.join(folder, "queries.npy"))[:128])
    idx = B200Index.load(folder, device=0)
    try:
        for bfs in (0, 2, -1):
            idx.set_param("EnableBfs", bfs)
            for mc in (64, 2048):
                idx.set_param("MaxCheck", mc)
                check_against_oracle(idx, files, q, 10, bfs, mc, tag=name)
    finally:
        idx.close()


# 2: filtered search, tombstones and p_searchDeleted
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt2_cos_1600_24", "bkt_cos_i8_1200_24", "bkt_l2_dups_1k_12"])
def test_filtered_and_tombstoned(name):
    from sptag_b200 import capi
    g, files, blob, q = pin.load_set(name)
    idx = gpu_index(files, blob)
    rng = np.random.default_rng(11)
    allowed = (rng.random(files.n) < 0.5).astype(np.uint8)
    try:
        for bfs in (2, -1):
            idx.set_param("EnableBfs", bfs)
            for mc in (0, 64):
                ids, dists, stats = idx.search_filtered(q, 10, allowed, max_check=mc, want_stats=True)
                o = pin.oracle_for(files, bfs, mc or 8192)
                o.filter = allowed
                ids_o, d_o, st_o = o.search(q, 10)
                same(ids, dists, ids_o, d_o, "%s filtered bfs=%d mc=%d" % (name, bfs, mc))
                assert np.array_equal(stats[:, capi.ST_CHECKED], st_o[:, reflib.ST_CHECKED])
        dead = np.nonzero(rng.random(files.n) < 0.3)[0].astype(np.int32)
        idx.delete(dead)
        files.deleted = np.zeros(files.n, np.int8)
        files.deleted[dead] = 1
        files.num_deleted = int(dead.size)
        for bfs in (2, 8):
            idx.set_param("EnableBfs", bfs)
            for sd in (False, True):
                ids, dists = idx.search(q, 10, search_deleted=sd, max_check=512)
                o = pin.oracle_for(files, bfs, 512)
                o.search_deleted = sd
                ids_o, d_o, _ = o.search(q, 10)
                same(ids, dists, ids_o, d_o, "%s tombstones bfs=%d searchDeleted=%d" % (name, bfs, sd))
    finally:
        idx.close()


# 3: the hashed visited set, at its default size and at 64 entries (a limit the seeding's inserts alone can reach)
@pytest.mark.parametrize("entries", [0, 64])
@pytest.mark.parametrize("name", PLAIN + ["pq_f32_1200_16"])
def test_hashed_visited_set(name, entries):
    g, files, blob, q = pin.load_set(name)
    idx = gpu_index(files, blob, **{"B200.VisitedSet": 1, "B200.VisitedHashEntries": entries})
    try:
        check_golden_search(idx, g, files, blob, q, "%s hashed %d" % (name, entries))
        idx.set_param("EnableBfs", 8)
        idx.set_param("MaxCheck", 8192)
        idx.search(q, 10)
        overflows = int(idx.get_param("B200.LastVisitedOverflows"))
        if entries == 64:
            assert overflows > 0
        else:
            assert overflows == 0
    finally:
        idx.close()


# 4: RefineSearchIndex lists (the refine pass and the host-query call) and AddIndex
@pytest.mark.parametrize("name", SETS)
def test_refine_matches_reference(name):
    g, files, blob, q = pin.load_set(name)
    idx = gpu_index(files, blob, MaxCheckForRefineGraph=int(g["refine_max_check"]))
    num, cef = int(g["refine_nodes"]), int(g["refine_cef"])
    try:
        for a, bfs in enumerate(g["bfs_values"].tolist()):
            idx.set_param("EnableBfs", bfs)
            _, ids, dists = idx.refine_graph(cef, first=0, num=num, neighborhood=16, want_results=True)
            same(ids, dists, g["refine_ids"][a], g["refine_dists"][a], "%s refine_graph bfs=%d" % (name, bfs))
            if blob is None:
                ids, dists = idx.refine_search(files.vectors[:num], cef + 1)
                same(ids, dists, g["refine_ids"][a], g["refine_dists"][a], "%s refine_search bfs=%d" % (name, bfs))
    finally:
        idx.close()


# the graph after AddIndex: the refine search of every added row seeds breadth-first
def test_add_equals_reference():
    g, files, blob, q = pin.load_set("bkt_l2_2k_16")
    m = np.load(os.path.join(pin.GOLDEN, "mutation", "bkt_l2_2k_16.npz"))
    assert not np.array_equal(g["add_graph"], m["graph1"])  # the reference's graph differs from the EnableBfs = 0 add
    idx = gpu_index(files, blob, AddCEF=int(g["add_cef"]), MaxCheckForRefineGraph=int(g["add_max_check_refine"]),
                    EnableBfs=int(g["add_bfs"]))
    try:
        assert idx.add(m["batch_a"]) == files.n
        assert np.array_equal(idx.get_graph(), g["add_graph"]), "graph after AddIndex differs from the reference's"
    finally:
        idx.close()


# 5: ResultIterator::Next and SearchIndexIterativeFromNeareast, on bitmaps and on 64-entry hash tables
ITER_MODES = {"bitmap": {"B200.IteratorVisitedSet": 0},
              "hash64": {"B200.IteratorVisitedSet": 1, "B200.IteratorVisitedHashEntries": 64}}


@pytest.mark.parametrize("mode", sorted(ITER_MODES))
@pytest.mark.parametrize("name", PLAIN)
def test_iterators_match_reference(name, mode):
    g, files, blob, q = pin.load_set(name)
    idx = gpu_index(files, blob, MaxCheck=int(g["iter_max_check"]), **ITER_MODES[mode])
    nq, calls, batch = g["iter_ids"].shape[1:]
    ncalls, k = g["nearest_ids"].shape[2:]
    qq = np.ascontiguousarray(q[:nq])
    try:
        for a, bfs in enumerate(g["bfs_values"].tolist()):
            idx.set_param("EnableBfs", bfs)
            its = idx.iterators(qq)
            for c in range(calls):
                counts, ids, dists, _ = its.next(int(batch))
                assert np.array_equal(counts, g["iter_counts"][a, :, c]), (name, mode, bfs, c)
                for i in range(nq):
                    n = counts[i]
                    assert np.array_equal(ids[i, :n], g["iter_ids"][a, i, c, :n]), (name, mode, bfs, i, c)
                    assert np.array_equal(dists[i, :n].view(np.int32), g["iter_dists"][a, i, c, :n].view(np.int32))
            its.close()
            its = idx.iterators(qq)
            for c in range(ncalls):
                _, ids, dists = its.next_from_nearest(int(k))
                same(ids, dists, g["nearest_ids"][a, :, c], g["nearest_dists"][a, :, c],
                     "%s %s nearest bfs=%d call %d" % (name, mode, bfs, c))
            its.close()
    finally:
        idx.close()


@pytest.mark.parametrize("mode", sorted(ITER_MODES))
def test_iterator_takes_the_value_of_its_first_call(mode):
    """InitSearchTrees runs at an iterator's first Next: the EnableBfs in force then decides the seeding, whatever it
    was at open or is set to later."""
    g, files, blob, q = pin.load_set("bkt_l2_2k_16")
    idx = gpu_index(files, blob, MaxCheck=int(g["iter_max_check"]), EnableBfs=0, **ITER_MODES[mode])
    nq, calls, batch = g["iter_ids"].shape[1:]
    a = g["bfs_values"].tolist().index(2)
    try:
        its = idx.iterators(np.ascontiguousarray(q[:nq]))
        idx.set_param("EnableBfs", 2)
        for c in range(calls):
            counts, ids, _, _ = its.next(int(batch))
            assert np.array_equal(counts, g["iter_counts"][a, :, c])
            for i in range(nq):
                assert np.array_equal(ids[i, :counts[i]], g["iter_ids"][a, i, c, :counts[i]]), (mode, i, c)
            idx.set_param("EnableBfs", 0 if c % 2 == 0 else -1)
        its.close()
    finally:
        idx.close()


# 7: the ini: a folder with EnableBfs loads (it used to be refused), save keeps the value, KDT ignores the key
def test_load_and_save_keep_enable_bfs(tmp_path):
    from sptag_b200 import B200Index
    mk = pin.golden_module()
    g, files, blob, q = pin.load_set("bkt_l2_2k_16")
    a, b = g["bfs_values"].tolist().index(2), g["max_checks"].tolist().index(64)
    mk.write_folder(dict(params=dict(files.params, EnableBfs="2", MaxCheck="64"), vectors=files.vectors,
                         graph=files.graph, tree_starts=files.tree_starts, nodes=files.nodes, quantizer_blob=None),
                    str(tmp_path / "in"))
    idx = B200Index.load(str(tmp_path / "in"), device=0)
    try:
        assert idx.get_param("EnableBfs") == "2"
        ids, dists = idx.search(q, 10)
        same(ids, dists, g["ref_ids"][a, b], g["ref_dists"][a, b], "loaded EnableBfs=2")
        idx.save(str(tmp_path / "out"))
    finally:
        idx.close()
    with open(tmp_path / "out" / "indexloader.ini") as f:
        assert "EnableBfs=2\n" in f.read()
    idx = B200Index.load(str(tmp_path / "out"), device=0)
    try:
        assert idx.get_param("EnableBfs") == "2"
        ids, dists = idx.search(q, 10)
        same(ids, dists, g["ref_ids"][a, b], g["ref_dists"][a, b], "saved and loaded EnableBfs=2")
        idx.set_param("EnableBfs", 0)
        idx.save(str(tmp_path / "zero"))
    finally:
        idx.close()
    with open(tmp_path / "zero" / "indexloader.ini") as f:
        assert "EnableBfs" not in f.read()


def test_kdt_folder_with_enable_bfs_loads_and_searches_as_before(tmp_path):
    from sptag_b200 import B200Index, capi
    mk = pin.golden_module()
    g = np.load(os.path.join(pin.GOLDEN, "kdt_l2_2k_16.npz"))
    ix = mk.index_from_npz(g)
    ix["params"]["EnableBfs"] = "2"
    mk.write_folder(ix, str(tmp_path))
    idx = B200Index.load(str(tmp_path), device=0)
    try:
        with pytest.raises(capi.SptagB200Error) as e:
            idx.get_param("EnableBfs")
        assert e.value.code == PARAM_NOT_FOUND
        with pytest.raises(capi.SptagB200Error) as e:
            idx.set_param("EnableBfs", 2)
        assert e.value.code == PARAM_NOT_FOUND
        q, k = np.ascontiguousarray(g["queries"]), int(g["k"])
        for i, mc in enumerate(g["max_checks"].tolist()):
            idx.set_param("MaxCheck", int(mc))
            ids, dists = idx.search(q, k)
            same(ids, dists, g["ref_ids"][i], g["ref_dists"][i], "kdt mc=%d" % mc)
    finally:
        idx.close()


# 8: set_param between batches takes effect at the next call; get_param reports it
def test_set_param_between_batches():
    g, files, blob, q = pin.load_set("bkt_cos_1500_20")
    idx = gpu_index(files, blob, MaxCheck=64)
    b = g["max_checks"].tolist().index(64)
    try:
        assert idx.get_param("EnableBfs") == "0"
        ids0, d0 = idx.search(q, 10)
        ids_o, d_o, _ = pin.oracle_for(files, 0, 64).search(q, 10)
        same(ids0, d0, ids_o, d_o, "EnableBfs=0")
        for a, bfs in list(enumerate(g["bfs_values"].tolist())) * 2:
            idx.set_param("EnableBfs", bfs)
            assert idx.get_param("EnableBfs") == str(bfs)
            ids, dists = idx.search(q, 10)
            same(ids, dists, g["ref_ids"][a, b], g["ref_dists"][a, b], "EnableBfs=%d" % bfs)
        idx.set_param("EnableBfs", 0)
        ids, dists = idx.search(q, 10)
        same(ids, dists, ids0, d0, "back to EnableBfs=0")
    finally:
        idx.close()


# 9: the drop-in SPTAG::B200::Index (tests/cpp/bfs_dropin.cpp)
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt2_cos_1600_24"])
def test_dropin_attach_and_set_parameter(name, tmp_path):
    exe = os.path.join(ROOT, "tests", "cpp", "bfs_dropin")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/bfs_dropin was not built (needs the reference's headers at build time)")
    mk = pin.golden_module()
    g, files, blob, q = pin.load_set(name)
    mk.write_folder(dict(params=files.params, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                         nodes=files.nodes, quantizer_blob=None), str(tmp_path / "idx"))
    qf = str(tmp_path / "q.bin")
    np.ascontiguousarray(q).tofile(qf)
    r = subprocess.run([exe, str(tmp_path / "idx"), qf, str(q.shape[0]), "10", "64"], capture_output=True, text=True,
                       timeout=600)
    lines = [l for l in r.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert r.returncode == 0, r.stdout + r.stderr
    assert len(lines) == 7 and all(l.startswith("PASS") for l in lines), r.stdout
