"""GPU tests: AddIndex / DeleteIndex / DeleteIndex(vectors) / SaveIndex on the device against the reference.

The reference's results come from tests/golden/mutation/*.npz (made by tests/golden/make_golden_mutation.py with the
unmodified reference: AddCEF 64, MaxCheckForRefineGraph 512, fewer adds than AddCountForRebuild).  Where oracle/_ref is
built, the folder the device saves is also loaded by the reference itself and searched.
"""
import os

import numpy as np
import pytest

import reflib
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
CASES = sorted(f[:-4] for f in os.listdir(os.path.join(GOLDEN, "mutation")) if f.endswith(".npz"))


def load_case(case):
    m = np.load(os.path.join(GOLDEN, "mutation", case + ".npz"))
    if "base_vectors" in m:  # an index the generator had the reference build (int8 Cosine)
        g = {k[5:]: m[k] for k in m.files if k.startswith("base_")}
    else:
        g = np.load(os.path.join(GOLDEN, str(m["fixture"]) + ".npz"))
    return m, g


def make_index(g, m, id_offset=0, deleted=None, num_deleted=0):
    params = dict(zip(g["param_names"].tolist(), g["param_values"].tolist()))
    idx = B200Index.create(algo=reflib.ALGO_OF_NAME[params["IndexAlgoType"]],
                           value_type=reflib.VT_OF_NAME[params.get("ValueType", "Float")],
                           metric=reflib.METRIC_OF_NAME[params["DistCalcMethod"]], vectors=g["vectors"], graph=g["graph"],
                           tree_starts=g["tree_starts"], tree_nodes=g["nodes"], device=0, id_offset=id_offset,
                           deleted=deleted, num_deleted=num_deleted)
    for name, value in zip(m["param_names"].tolist(), m["param_values"].tolist()):
        idx.set_param(name, value)
    return idx


def check_searches(idx, m, ids_ref, dists_ref, id_offset=0):
    q = m["queries"]
    k = int(m["k"])
    for a, mc in enumerate(m["max_checks"].tolist()):
        for sd in (0, 1):
            ids, dists = idx.search(q, k, search_deleted=bool(sd), max_check=mc)
            want = np.where(ids_ref[a, sd] >= 0, ids_ref[a, sd] + id_offset, -1)
            assert np.array_equal(ids, want), "ids differ at MaxCheck %d, searchDeleted %d" % (mc, sd)
            assert np.array_equal(dists.view(np.int32), dists_ref[a, sd].view(np.int32)), \
                "distances differ at MaxCheck %d, searchDeleted %d" % (mc, sd)


@pytest.mark.parametrize("case", CASES)
def test_add_equals_reference(case, tmp_path):
    m, g = load_case(case)
    idx = make_index(g, m)
    n = g["vectors"].shape[0]
    first = idx.add(m["batch_a"], normalized=bool(m["normalized"]))
    assert first == n and idx.num_vectors == n + 200
    assert np.array_equal(idx.get_graph(), m["graph1"]), "graph after AddIndex differs from the reference's"
    check_searches(idx, m, m["ids1"], m["dists1"])
    idx.save(str(tmp_path))
    saved = reflib.IndexFiles(str(tmp_path))
    assert np.array_equal(saved.vectors[n:].view(np.int32), m["added1"].view(np.int32)), "added (normalised) rows differ"
    idx.close()


@pytest.mark.parametrize("case", CASES)
def test_add_delete_interleaved_equals_reference(case, tmp_path):
    m, g = load_case(case)
    idx = make_index(g, m)
    n = g["vectors"].shape[0]
    normalized = bool(m["normalized"])
    idx.add(m["batch_a"], normalized=normalized)
    codes = idx.delete(m["del_ids"])
    # live ids and repeats: the reference's codes; the last id is out of range, which the device refuses with
    # VectorNotFound (the reference's Labelset answers Success for ids >= R without tombstoning anything)
    assert np.array_equal(codes[:-1], m["del_codes"][:-1]), "DeleteIndex(id) codes differ"
    assert set(codes[:-1].tolist()) == {0, 0x14} and codes[-1] == 0x14
    idx.delete_vectors(m["del_vecs"])
    first = idx.add(m["batch_b"], normalized=normalized)
    assert first == n + 200
    assert np.array_equal(idx.get_graph(), m["graph2"]), "graph after the mutation sequence differs"
    assert idx.num_deleted == int(m["num_deleted2"])
    check_searches(idx, m, m["ids2"], m["dists2"])
    if "it_ids" in m:  # iterators opened after the deletes: GetIterator(q, false) + 3 x Next(8), MaxCheck 512
        idx.set_param("MaxCheck", 512)
        it = idx.iterators(m["queries"][:8], search_deleted=False)
        for j in range(m["it_ids"].shape[1]):
            counts, ids, dists, _ = it.next(8)
            assert np.array_equal(counts, m["it_counts"][:, j]), "iterator counts differ in round %d" % j
            assert np.array_equal(ids, m["it_ids"][:, j]), "iterator ids differ in round %d" % j
            assert np.array_equal(dists.view(np.int32), m["it_dists"][:, j].view(np.int32))
        it.close()
        idx.set_param("MaxCheck", 8192)

    # SaveIndex -> both loaders read the folder and agree with the mutated handle
    folder = str(tmp_path / "saved")
    idx.save(folder)
    saved = reflib.IndexFiles(folder)
    assert saved.num_deleted == int(m["num_deleted2"])
    # the tombstone set; the reference's bytes for added rows are 0xff where the device writes 0 (Dataset::AddBatch
    # fills new blocks with -1; both read as live: Labelset::Contains tests == 1)
    assert np.array_equal(saved.deleted == 1, m["deleted2"] == 1)
    assert np.array_equal(saved.graph, m["graph2"])
    assert np.array_equal(saved.vectors[n + 200:].view(np.int32), m["added2"].view(np.int32))
    again = B200Index.load(folder, device=0)
    assert np.array_equal(again.get_graph(), m["graph2"])
    assert again.get_param("AddCEF") == str(int(m["param_values"][0]))
    check_searches(again, m, m["ids2"], m["dists2"])
    again.close()
    if reflib.have_ref():
        r = reflib.RefIndex.load(folder)
        k = int(m["k"])
        for a, mc in enumerate(m["max_checks"].tolist()):
            r.set_param("MaxCheck", mc)
            ids, dists = r.search_flag(m["queries"], k, 0, threads=1)
            assert np.array_equal(ids, m["ids2"][a, 0])
            assert np.array_equal(dists.view(np.int32), m["dists2"][a, 0].view(np.int32))
    idx.close()


def test_many_small_adds_equal_one_large_add():
    m, g = load_case("bkt_l2_2k_16")
    idx = make_index(g, m)
    n = g["vectors"].shape[0]
    for i in range(50):  # crosses several geometric reallocations of vectors and graph
        assert idx.add(m["batch_a"][4 * i:4 * i + 4]) == n + 4 * i
    assert np.array_equal(idx.get_graph(), m["graph1"])
    check_searches(idx, m, m["ids1"], m["dists1"])
    idx.close()


def test_refusals_and_delete_codes():
    m, g = load_case("bkt_l2_2k_16")
    idx = make_index(g, m)
    n, dim = g["vectors"].shape
    with pytest.raises(capi.SptagB200Error) as e:
        idx.add(np.zeros((0, dim), np.float32))
    assert e.value.code == 0x16  # EmptyData
    with pytest.raises(capi.SptagB200Error) as e:
        idx.add(np.zeros((3, dim + 1), np.float32))
    assert e.value.code == 0x17  # DimensionSizeMismatch
    it = idx.iterators(m["queries"][:2])
    for call in (lambda: idx.add(m["batch_a"][:2]), lambda: idx.delete([1]), lambda: idx.delete_vectors(m["batch_a"][:1])):
        with pytest.raises(capi.SptagB200Error) as e:
            call()
        assert e.value.code == 0x01 and "iterator" in str(e.value)
    it.close()
    assert idx.num_vectors == n and idx.num_deleted == 0
    assert idx.delete([5, 5, n, -3, 7]).tolist() == [0, 0x14, 0x14, 0x14, 0]
    assert idx.delete([5]).tolist() == [0x14]
    assert idx.num_deleted == 2
    ids, _ = idx.search(g["vectors"][[5, 7]], 5)
    assert 5 not in ids[0] and 7 not in ids[1]
    ids, _ = idx.search(g["vectors"][[5, 7]], 5, search_deleted=True)
    assert ids[0, 0] == 5 and ids[1, 0] == 7
    idx.close()


def test_shard_handle_mutates_by_global_id_and_group_keeps_working():
    m, g = load_case("bkt_l2_2k_16")
    off = 100000
    a = make_index(g, m)
    b = make_index(g, m, id_offset=off)
    n = g["vectors"].shape[0]
    assert b.delete([off + 9, 9]).tolist() == [0, 0x14]  # global ids; 9 is outside this shard
    group = capi.B200ShardGroup([a, b])
    first = b.add(m["batch_a"][:8])
    assert first == off + n
    ids, dists = group.search(m["batch_a"][:8], 2)  # the group re-reads the shard's size: the new rows are found
    fresh = np.where(ids[:, 0] >= off)[0]
    assert len(fresh) > 0 and np.all(ids[fresh, 0] >= off)
    ids_b, _ = b.search(g["vectors"][[9]], 3)
    assert off + 9 not in ids_b[0]
    group.close()
    a.close()
    b.close()


def test_rows_with_0xff_tombstone_bytes_are_live():
    """The reference saves the tombstone bytes of rows it added as 0xff (Dataset::AddBatch fills new blocks with -1);
    Labelset treats every byte but 1 as live.  Such a map must delete by id and by vector like a zeroed one."""
    m, g = load_case("bkt_l2_2k_16")
    n = g["vectors"].shape[0]
    deleted = np.zeros(n, np.int8)
    deleted[n - 100:] = -1
    deleted[[3, n - 1]] = 1
    idx = make_index(g, m, deleted=deleted, num_deleted=2)
    assert idx.delete([n - 50, n - 50, n - 1, 3]).tolist() == [0, 0x14, 0x14, 0x14]
    assert idx.num_deleted == 3
    ids, _ = idx.search(g["vectors"][[n - 50]], 5)
    assert n - 50 not in ids[0]
    # DeleteIndex(vectors) of a 0xff row: its exact copy is found (distance 0) and tombstoned
    ids, dists = idx.search(g["vectors"][[n - 20]], 1)
    assert ids[0, 0] == n - 20 and dists[0, 0] == 0.0
    idx.delete_vectors(g["vectors"][[n - 20]])
    assert idx.num_deleted == 4
    ids, _ = idx.search(g["vectors"][[n - 20]], 5)
    assert n - 20 not in ids[0]
    assert idx.delete([n - 20]).tolist() == [0x14]
    idx.close()


def test_quantized_index_refuses_add_save_and_delete_by_vector():
    g = np.load(os.path.join(GOLDEN, "quantized", "pq_f32_1200_16.npz"))
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_UINT8, metric=capi.METRIC_L2, vectors=g["vectors"],
                           graph=g["graph"], tree_starts=g["tree_starts"], tree_nodes=g["nodes"], device=0)
    idx.set_quantizer(g["quantizer_blob"].tobytes())
    raw = np.ascontiguousarray(g["queries"][:2])
    for call in (lambda: idx.add(g["vectors"][:2]), lambda: idx.delete_vectors(raw), lambda: idx.save("/nonexistent/x")):
        with pytest.raises(capi.SptagB200Error) as e:
            call()
        assert e.value.code == 0x13  # LackOfInputs
    assert idx.delete([3]).tolist() == [0]  # tombstones only: allowed
    assert idx.num_deleted == 1
    idx.close()
