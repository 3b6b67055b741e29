"""GPU tests of the hashed visited set (B200.VisitedSet = 1): a per-slot open-addressed table instead of a bitmap over the
whole index, and the bitmap re-run of the queries that fill it.  Every result must be bit-identical to the bitmap path's,
i.e. to the reference's: ids, distance bits and the WorkSpace counters.

Two modes run every check: the default table capacity ("hash": no query overflows on these fixtures) and a 64-entry
table ("overflow": nearly every query is abandoned at 32 distinct ids and re-run on the bitmap).  The committed golden
fixtures need nothing but the repository; the tests/_data sets are used where they exist.
"""
import os
import threading

import numpy as np
import pytest

import reflib
import test_gpu_mutation as tgm
import test_gpu_parity as tgp
import test_oracle_pin as pin
from conftest import data_folder
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_SETS = ["algo_line_bkt", "bkt_cos_1500_20", "bkt_l2_2k_16", "bkt_l2_dups_1k_12", "kdt_l2_2k_16"]
MODES = {"hash": {"B200.VisitedSet": 1}, "overflow": {"B200.VisitedSet": 1, "B200.VisitedHashEntries": 64}}


@pytest.fixture(params=sorted(MODES))
def mode(request, monkeypatch):
    """Every index created or loaded while the test runs gets the mode's parameters, so the existing parity checks run
    unchanged on the hashed set."""
    knobs = MODES[request.param]
    for name in ("create", "load"):
        orig = getattr(B200Index, name)

        def made(*args, _orig=orig, **kwargs):
            idx = _orig(*args, **kwargs)
            for k, v in knobs.items():
                idx.set_param(k, v)
            return idx

        monkeypatch.setattr(B200Index, name, made)
    return request.param


def overflows(idx):
    return int(idx.get_param("B200.LastVisitedOverflows"))


def golden_index(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    pin._files_from_npz(files, g)
    idx = B200Index.create(algo=capi.ALGO_KDT if files.algo == "KDT" else capi.ALGO_BKT, value_type=capi.VT_FLOAT,
                           metric=files.metric, vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts,
                           tree_nodes=files.nodes)
    return g, files, idx


def check_overflow_count(mode, idx):
    if mode == "overflow":
        assert overflows(idx) > 0
    else:
        assert overflows(idx) == 0


# ---- 1. searches against the reference's outputs and the oracle -----------------------------------------------------
@pytest.mark.parametrize("name", GOLDEN_SETS)
def test_golden_reference_outputs(mode, name):
    tgp.test_gpu_matches_reference_golden_outputs(name)


@pytest.mark.parametrize("name", GOLDEN_SETS)
def test_golden_budgets_and_result_counts(mode, name):
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    try:
        for mc in (64, 8192):
            for k in (1, 10, 100, 2048):
                tgp._compare(idx, files, q, k, mc, "%s %s k=%d" % (name, mode, k))
                if mc == 8192 and name != "algo_line_bkt":
                    check_overflow_count(mode, idx)
    finally:
        idx.close()


@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "kdt_l2_2k_16"])
def test_tiny_budget_keeps_room_for_a_row(mode, name):
    """MaxCheck = MaxCheckForRefineGraph = 4 would make the default table 32 entries; it is at least 64, so that one row
    of 32 neighbours past the fill limit still finds empty positions."""
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    try:
        assert files.degree == 32
        idx.set_param("MaxCheck", 4)
        idx.set_param("MaxCheckForRefineGraph", 4)
        ids, dists, stats = idx.search(q, 10, want_stats=True)
        o = reflib.OracleIndex(files)
        o.max_check = 4
        o.max_check_refine = 4
        ids_o, d_o, st_o = o.search(q, 10)
        assert np.array_equal(ids, ids_o)
        assert np.array_equal(dists.view(np.int32), d_o.view(np.int32))
        assert np.array_equal(stats[:, capi.ST_CHECKED], st_o[:, reflib.ST_CHECKED])
    finally:
        idx.close()


@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt_l2_dups_1k_12", "bkt_cos_1500_20"])
def test_golden_filtered_and_tombstoned(mode, name):
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    rng = np.random.default_rng(7)
    allowed = (rng.random(files.n) < 0.5).astype(np.uint8)
    try:
        for mc in (0, 512):
            ids, dists, stats = idx.search_filtered(q, 10, allowed, max_check=mc, want_stats=True)
            o = reflib.OracleIndex(files)
            o.filter = allowed
            if mc:
                o.max_check = mc
            ids_o, d_o, st_o = o.search(q, 10)
            assert np.array_equal(ids, ids_o), (name, mc)
            assert np.array_equal(dists.view(np.int32), d_o.view(np.int32)), (name, mc)
            assert np.array_equal(stats[:, capi.ST_CHECKED], st_o[:, reflib.ST_CHECKED])
        # tombstones: a third of the ids deleted, searched with p_searchDeleted 0 and 1
        dead = np.nonzero(rng.random(files.n) < 0.3)[0].astype(np.int32)
        idx.delete(dead)
        files.deleted = np.zeros(files.n, np.int8)
        files.deleted[dead] = 1
        files.num_deleted = int(dead.size)
        for sd in (False, True):
            ids, dists = idx.search(q, 10, search_deleted=sd, max_check=2048)
            o = reflib.OracleIndex(files)
            o.max_check = 2048
            o.search_deleted = sd
            ids_o, d_o, _ = o.search(q, 10)
            assert np.array_equal(ids, ids_o), (name, sd)
            assert np.array_equal(dists.view(np.int32), d_o.view(np.int32)), (name, sd)
            if not sd:
                assert not files.deleted[ids[ids >= 0]].any()
    finally:
        idx.close()


@pytest.mark.parametrize("name", ["opq_i8_1500_24", "pq_f32_1200_16"])
def test_golden_quantized_sdc_and_adc(mode, name):
    g = np.load(os.path.join(GOLDEN, "quantized", name + ".npz"))
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_UINT8, metric=capi.METRIC_L2, vectors=g["vectors"],
                           graph=g["graph"], tree_starts=g["tree_starts"], tree_nodes=g["nodes"], device=0)
    try:
        idx.set_quantizer(g["quantizer_blob"].tobytes())
        q, k = np.ascontiguousarray(g["queries"]), int(g["k"])
        for adc, tag in ((0, "sdc"), (1, "adc")):
            idx.set_param("EnableADC", adc)
            for i, mc in enumerate(g["max_checks"].tolist()):
                ids, dists = idx.search(q, k, max_check=int(mc))
                assert np.array_equal(ids, g["ref_ids_" + tag][i]), (name, tag, mc)
                assert np.array_equal(dists.view(np.int32), g["ref_dists_" + tag][i].view(np.int32)), (name, tag, mc)
    finally:
        idx.close()


# the reference-built sets of tests/_data (skipped where they are not built): every BKT set, the KDT sets, the integer
# element types and the quantized sets, through the parity tests themselves
@pytest.mark.parametrize("name", tgp.BKT_SETS)
def test_bkt_sets(mode, name):
    tgp.test_bkt_search_bit_exact(name)


@pytest.mark.parametrize("name", ["kdt_l2_10k_64", "kdt2_l2_6k_32"])
def test_kdt_sets(mode, name):
    tgp.test_kdt_search_bit_exact(name)


@pytest.mark.parametrize("name", ["bkt_i8_cos_6k_64", "bkt_u8_l2_6k_128", "kdt_i8_l2_6k_32", "bkt_i16_l2_5k_64",
                                  "kdt_i16_l2_5k_32"])
def test_integer_sets(mode, name):
    tgp.test_integer_index_search_bit_exact(name)


@pytest.mark.parametrize("name", tgp.QUANT_SETS)
def test_quantized_sets(mode, name):
    tgp.test_quantized_bkt_search_bit_exact(name)
    tgp.test_quantized_adc_search_bit_exact(name)


@pytest.mark.parametrize("name", ["bkt_l2_10k_128", "kdt_l2_10k_64"])
def test_large_k_sets(mode, name):
    tgp.test_large_k_result_set(name)


# ---- 2. the re-run is stream-ordered --------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "kdt_l2_2k_16"])
def test_search_device_equals_blocking_search(mode, name):
    import torch
    g, files, idx = golden_index(name)
    q = np.ascontiguousarray(g["queries"])
    try:
        idx.set_param("MaxCheck", 8192)
        ids, dists = idx.search(q, 40)
        check_overflow_count(mode, idx)
        d_q = torch.from_numpy(q).cuda()
        d_ids = torch.full((q.shape[0], 40), -7, dtype=torch.int32, device="cuda")
        d_dists = torch.zeros((q.shape[0], 40), dtype=torch.float32, device="cuda")
        stream = torch.cuda.current_stream()
        idx.search_device(d_q.data_ptr(), q.shape[0], 40, d_ids.data_ptr(), d_dists.data_ptr(), stream=stream.cuda_stream)
        stream.synchronize()
        assert np.array_equal(d_ids.cpu().numpy(), ids)
        assert np.array_equal(d_dists.cpu().numpy().view(np.int32), dists.view(np.int32))
        if mode == "hash":  # the table layout is bound: 256 KB per slot against a 256-byte bitmap on this index
            bitmap = golden_index(name)[2]
            try:
                bitmap.set_param("B200.VisitedSet", 0)
                bitmap.search(q, 40, max_check=8192)
                assert int(idx.get_param("B200.ScratchBytes")) > 2 * int(bitmap.get_param("B200.ScratchBytes"))
            finally:
                bitmap.close()
    finally:
        idx.close()


# ---- 3. mutation and refine ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", tgm.CASES)
def test_mutation_sequence(mode, case, tmp_path):
    tgm.test_add_delete_interleaved_equals_reference(case, tmp_path)


@pytest.mark.parametrize("name", ["algo_line_bkt", "bkt_cos_1500_20", "bkt_l2_2k_16", "bkt_l2_dups_1k_12", "kdt_l2_2k_16"])
def test_refine_pass(mode, name):
    r = np.load(os.path.join(GOLDEN, "refine", name + ".npz"))
    g, files, idx = golden_index(name)
    try:
        idx.set_param("MaxCheckForRefineGraph", int(r["max_check_refine"]))
        num = r["rows"].shape[0]
        rows, ids, dists = idx.refine_graph(int(r["cef"]), first=0, num=num, neighborhood=int(r["neighborhood"]),
                                            rng_factor=float(r["rng_factor"]), want_results=True)
        assert np.array_equal(ids, r["res_ids"]), name
        assert np.array_equal(dists.view(np.int32), r["res_dists"].view(np.int32)), name
        assert np.array_equal(rows, r["rows"]), name
    finally:
        idx.close()


# ---- 4.-6. selection, scratch size, concurrent callers ---------------------------------------------------------------
def test_auto_selects_the_bitmap_when_it_fits():
    g, files, auto = golden_index("bkt_l2_2k_16")
    _, _, bitmap = golden_index("bkt_l2_2k_16")
    q = np.ascontiguousarray(g["queries"])
    try:
        assert auto.get_param("B200.VisitedSet") == "-1"
        bitmap.set_param("B200.VisitedSet", 0)
        for k, mc in ((10, 8192), (100, 512)):
            a = auto.search(q, k, max_check=mc)
            b = bitmap.search(q, k, max_check=mc)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.int32), b[1].view(np.int32))
        assert overflows(auto) == 0
        assert int(auto.get_param("B200.ScratchBytes")) == int(bitmap.get_param("B200.ScratchBytes")) > 0
    finally:
        auto.close()
        bitmap.close()


def _flat_index(n, seed):
    """An index whose scratch depends only on its sizes: a one-leaf tree, an empty graph of degree 16."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 32), dtype=np.float32)
    graph = np.full((n, 16), -1, np.int32)
    nodes = np.array([[n, 1, 2], [0, -1, -1], [-1, -1, -1]], np.int32)
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT, metric=0, vectors=x, graph=graph,
                           tree_starts=np.array([0], np.int32), tree_nodes=nodes)
    idx.set_param("MaxCheck", 32)
    idx.set_param("MaxCheckForRefineGraph", 32)
    return idx, x


def test_hashed_scratch_does_not_grow_with_the_index():
    """Per resident slot, the hashed set's scratch is independent of N; only the bitmaps of the re-run grid (one slot per
    SM, at most one per query) grow with it.  The bitmap layout grows by one bitmap per resident slot."""
    import torch
    nq = 8
    grow = {}
    for visited_set in (0, 1):
        sizes = []
        for n in (5000, 80000):
            idx, x = _flat_index(n, n)
            idx.set_param("B200.VisitedSet", visited_set)
            idx.search(x[:nq], 10)
            sizes.append(int(idx.get_param("B200.ScratchBytes")))
            idx.close()
        grow[visited_set] = sizes[1] - sizes[0]
    words = [((n + 1 + 31) // 32 + 3) // 4 * 4 for n in (5000, 80000)]
    rerun_slots = min(nq, torch.cuda.get_device_properties(0).multi_processor_count)
    assert grow[1] == rerun_slots * (words[1] - words[0]) * 4
    assert grow[0] > 10 * grow[1]


def test_concurrent_callers_use_both_scratch_sets(mode):
    g, files, idx = golden_index("bkt_l2_2k_16")
    q = np.ascontiguousarray(np.concatenate([g["queries"]] * 8))
    idx.set_param("MaxCheck", 8192)
    jobs = [(q[0:300], 10), (q[300:512], 40), (q[100:400], 5), (q[200:260], 1)]
    expect = [idx.search(b, k) for b, k in jobs]
    one_set = int(idx.get_param("B200.ScratchBytes"))  # serial calls use scratch set 0 only
    out = [None] * len(jobs)
    errs = []

    def run(i):
        try:
            for _ in range(5):
                out[i] = idx.search(jobs[i][0], jobs[i][1])
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    try:
        assert not errs, errs
        for (ids, dists), (ids_e, d_e) in zip(out, expect):
            assert np.array_equal(ids, ids_e)
            assert np.array_equal(dists.view(np.int32), d_e.view(np.int32))
        # two device-pointer launches on two streams while the first stream is still busy: the second takes scratch set 1
        import torch
        b, k = jobs[0]
        d_q = torch.from_numpy(b).cuda()
        outs = [(torch.empty((b.shape[0], k), dtype=torch.int32, device="cuda"),
                 torch.empty((b.shape[0], k), dtype=torch.float32, device="cuda")) for _ in range(2)]
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        torch.cuda.synchronize()
        with torch.cuda.stream(streams[0]):
            torch.cuda._sleep(200000000)  # keeps set 0 busy while the second launch is set up
        for s_, (o_ids, o_d) in zip(streams, outs):
            idx.search_device(d_q.data_ptr(), b.shape[0], k, o_ids.data_ptr(), o_d.data_ptr(), stream=s_.cuda_stream)
        torch.cuda.synchronize()
        assert int(idx.get_param("B200.ScratchBytes")) > one_set  # set 1 was allocated
        for o_ids, o_d in outs:
            assert np.array_equal(o_ids.cpu().numpy(), expect[0][0])
            assert np.array_equal(o_d.cpu().numpy().view(np.int32), expect[0][1].view(np.int32))
    finally:
        idx.close()


def _random_graph_index(n, degree, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 4), dtype=np.float32)
    graph = rng.integers(0, n, (n, degree), dtype=np.int32)
    nodes = np.array([[n, 1, 2], [0, -1, -1], [-1, -1, -1]], np.int32)
    idx = B200Index.create(algo=capi.ALGO_BKT, value_type=capi.VT_FLOAT, metric=0, vectors=x, graph=graph,
                           tree_starts=np.array([0], np.int32), tree_nodes=nodes)
    idx.set_param("MaxCheck", 64)
    idx.set_param("MaxCheckForRefineGraph", 64)
    return idx, x


def test_auto_falls_back_to_the_hashed_set_when_the_bitmaps_do_not_fit():
    """Auto mode on an index whose per-slot bitmaps (1 MB each at 8M vectors) do not fit in what is left of device memory
    while the hashed scratch does: the search runs on the hashed set and returns the bitmap's results, call after call."""
    import torch
    n = 8000000
    ref, x = _random_graph_index(n, 8, 3)
    q = np.ascontiguousarray(x[:: n // 256][:256] + np.float32(0.01))
    try:
        ref.set_param("B200.VisitedSet", 0)
        want = ref.search(q, 10)
        bitmap_bytes = int(ref.get_param("B200.ScratchBytes"))
    finally:
        ref.close()
    idx, _ = _random_graph_index(n, 8, 3)
    hold = None
    try:
        idx.set_param("B200.VisitedSet", 1)
        idx.search(q, 10)
        hashed_bytes = int(idx.get_param("B200.ScratchBytes"))
        idx.close()
        idx, _ = _random_graph_index(n, 8, 3)
        assert idx.get_param("B200.VisitedSet") == "-1"
        margin = hashed_bytes + (256 << 20)
        assert bitmap_bytes > margin + (512 << 20), (bitmap_bytes, hashed_bytes)
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        hold = torch.empty(free - margin, dtype=torch.uint8, device="cuda")  # leaves room for the table, not the bitmaps
        for _ in range(3):
            got = idx.search(q, 10)
            assert np.array_equal(got[0], want[0])
            assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32))
            assert int(idx.get_param("B200.ScratchBytes")) < bitmap_bytes // 2
    finally:
        del hold
        torch.cuda.empty_cache()
        idx.close()


def test_parameter_checks():
    g, files, idx = golden_index("algo_line_bkt")
    try:
        for name, bad in (("B200.VisitedSet", 2), ("B200.VisitedHashEntries", 100), ("B200.VisitedHashEntries", 32)):
            with pytest.raises(capi.SptagB200Error):
                idx.set_param(name, bad)
        idx.set_param("B200.VisitedHashEntries", 4096)
        assert idx.get_param("B200.VisitedHashEntries") == "4096"
        with pytest.raises(capi.SptagB200Error):
            idx.set_param("B200.ScratchBytes", 1)  # read-only
    finally:
        idx.close()
