"""SPANN with the posting lists in pinned host memory (sptag_b200_spann_load_ex, posting_placement="host"): each search
or iterator step gathers the lists its queries read into an HBM stage and scans them there.  Against the reference's
results recorded in tests/golden/spann, spann_pq and spann_iter: ids and distance bits of every case, parameter set, K
and distance; the gathered bytes and rounds against a restatement of the union and of the halving rule; a stage small
enough to force rounds; parameters changed between batches; two threads; and what each placement reports."""
import os
import threading

import numpy as np
import pytest

import oracle_spann
import oracle_spann_pq
import reflib
from golden.make_golden_spann import KS, PARAMS, write_folder
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from golden.make_golden_spann_pq import MODES
from sptag_b200 import capi
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann")
GOLDEN_PQ = os.path.join(HERE, "golden", "spann_pq")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_iter")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
PQ_CASES = sorted(f[:-4] for f in os.listdir(GOLDEN_PQ) if f.endswith(".npz"))
ITER_CASES = sorted(f[:-4] for f in os.listdir(GOLDEN_ITER) if f.endswith(".npz"))
LACK_OF_INPUTS = 0x13
INT_MAX = 2**31 - 1
DEFAULT_STAGE = 256 << 20


@pytest.fixture
def host_index(tmp_path):
    """load(folder, 0, "host") of a fixture's files written with ini values; closed after the test"""
    opened = []

    def load(files, values=None, sub="index", placement="host"):
        folder = str(tmp_path / sub)
        write_folder(files, folder, values or {})
        s = capi.B200SpannIndex.load(folder, 0, posting_placement=placement)
        opened.append(s)
        return s

    yield load
    for s in opened:
        s.close()


def _fixture(golden, case):
    g = np.load(os.path.join(golden, case + ".npz"))
    return g, oracle_spann.fixture_files(g)


def _refused_truncation(folder):
    return folder.rearranged and any(folder.searched(l) < folder.lists[l][0] for l in range(len(folder.lists)))


def chosen_lists(folder, head_ids, head_dists):
    """The lists one query's scan reads: oracle_spann.search_one's choice rule (SPANNIndex.cpp:213-234)"""
    maxdist = np.float32(reflib.ora().ora_max_dist())
    limit = np.float32(np.float32(head_dists[0]) * folder.max_dist_ratio)
    posts = []
    for pid, d in zip(head_ids, head_dists):
        pid = int(pid)
        if pid == -1:
            break
        d = maxdist if int(folder.translate[pid]) == INT_MAX else np.float32(d)
        if len(posts) >= folder.internal or (float(limit) > 0.1 and d > limit) or folder.searched(pid) == 0:
            continue
        posts.append(pid)
    return posts


def elem_bytes(folder):
    """Bytes one staged element takes: its row at the head's row stride (16-byte aligned) and its int32 id"""
    return (folder.row_bytes + 15) // 16 * 16 + 4


def gather_rounds(folder, per_query, stage_bytes=DEFAULT_STAGE):
    """The halving rule over a batch's per-query list sets -> bytes gathered per round"""
    eb = elem_bytes(folder)
    longest = max(folder.searched(l) for l in range(len(folder.lists)))
    cap_elems = max(stage_bytes, folder.internal * longest * eb) // eb
    n, b, m, out = len(per_query), 0, len(per_query), []
    while b < n:
        m = min(m, n - b)
        while True:
            elems = sum(folder.searched(l) for l in set().union(*per_query[b:b + m]))
            if elems <= cap_elems or m == 1:
                break
            m = (m + 1) // 2
        out.append(elems * eb)
        b += m
    return out


def _assert_gathered(s, folder, head_ids, head_dists, stage_bytes=DEFAULT_STAGE):
    per_query = [set(chosen_lists(folder, i, d)) for i, d in zip(head_ids, head_dists)]
    want = gather_rounds(folder, per_query, stage_bytes)
    assert int(s.get_param("B200.LastGatherBytes")) == sum(want)
    assert int(s.get_param("B200.LastGatherRounds")) == len(want)
    return want


def _assert_search(s, g, folder, pname, q, stage_bytes=DEFAULT_STAGE):
    rounds = []
    for k in KS:
        ids, dists, stats = s.search(q, k, want_stats=True)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (pname, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (pname, k)
        hid, hd = g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)]
        _, _, st = oracle_spann.search(folder, q, hid, hd, k)
        assert np.array_equal(stats, st), (pname, k)
        rounds.append(_assert_gathered(s, folder, hid, hd, stage_bytes))
    return rounds


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_host_search_equals_reference(case, pname, host_index):
    """Results, stats and the gathered union (not every list) of every K on host-placed lists"""
    g, files = _fixture(GOLDEN, case)
    s = host_index(files, PARAMS[pname])
    assert s.get_param("B200.PostingPlacement") == "host"
    q = g["queries"]
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        with pytest.raises(capi.SptagB200Error) as e:
            s.search(q, 10)
        assert e.value.code == LACK_OF_INPUTS
        return
    every_list = sum(folder.searched(l) for l in range(len(folder.lists))) * elem_bytes(folder)
    for per_k in _assert_search(s, g, folder, pname, q):
        assert len(per_k) == 1 and per_k[0] <= every_list


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_smallest_stage_splits_the_batch(case, pname, host_index):
    """B200.PostingStageBytes 0 leaves one query's worst case: the batch runs in several rounds, results unchanged"""
    g, files = _fixture(GOLDEN, case)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        pytest.skip("truncated lists of the rearranged layout: refused on either placement")
    s = host_index(files, PARAMS[pname])
    s.set_param("B200.PostingStageBytes", 0)
    assert s.get_param("B200.PostingStageBytes") == "0"
    rounds = _assert_search(s, g, folder, pname, g["queries"], stage_bytes=0)
    # with MaxDistRatio 1.5 some fixtures choose so few lists that the batch's union fits one query's worst case
    assert max(len(r) for r in rounds) > 1 or pname == "ratio", "no K split the batch"


@pytest.mark.parametrize("case", PQ_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
def test_host_pq_search_equals_reference(case, pname, mode, host_index):
    g, files = _fixture(GOLDEN_PQ, case)
    s = host_index(files, dict(PARAMS[pname], EnableADC="true" if mode == "adc" else "false"))
    q = g["queries"]
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    quant = oracle_spann_pq.folder_quantizer(files)
    for stage in (DEFAULT_STAGE, 0):
        s.set_param("B200.PostingStageBytes", stage)
        for k in KS:
            ids, dists, stats = s.search(q, k, want_stats=True)
            key = "%s_%s_%d" % (mode, pname, k)
            assert np.array_equal(ids, g["ids_" + key]), (key, stage)
            assert np.array_equal(dists.view(np.int32), g["dists_" + key].view(np.int32)), (key, stage)
            w = max(k, folder.internal)
            hid, hd = g["head_ids_%s_%d" % (mode, w)], g["head_dists_%s_%d" % (mode, w)]
            _, _, st = oracle_spann_pq.search(folder, quant, q, hid, hd, k, mode == "adc")
            assert np.array_equal(stats, st), (key, stage)
            _assert_gathered(s, folder, hid, hd, stage)


@pytest.mark.parametrize("case", ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_host_iterators_equal_reference(case, pname, sname, stage, host_index):
    g = np.load(os.path.join(GOLDEN_ITER, case + ".npz"))
    src = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    s = host_index(files, ITER_PARAMS[pname])
    s.set_param("B200.PostingStageBytes", stage)
    q = schedule_queries(src["queries"], sname)
    it = s.iterators(q)
    try:
        if not applies(case, pname):
            with pytest.raises(capi.SptagB200Error) as e:
                it.next(10)
            assert e.value.code == LACK_OF_INPUTS
            return
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
        assert_calls_equal(got, want, (case, pname, sname, stage))
        assert int(s.get_param("B200.LastGatherRounds")) >= 1
    finally:
        it.close()


def test_host_iterator_rounds_split_at_the_smallest_stage(host_index):
    """The first Next of 32 iterators loads 32 head batches of 32 lists: more than one query's worst case"""
    src = np.load(os.path.join(GOLDEN, "spann_l2_3k_16.npz"))
    files = oracle_spann.fixture_files(src)
    s = host_index(files)
    big = host_index(files, sub="big")
    s.set_param("B200.PostingStageBytes", 0)
    q = src["queries"]
    a, b = s.iterators(q), big.iterators(q)
    try:
        more = []
        for batch in (64, 64, 16):
            assert_calls_equal([a.next(batch)], [b.next(batch)], batch)
            small_rounds, big_rounds = int(s.get_param("B200.LastGatherRounds")), int(big.get_param("B200.LastGatherRounds"))
            assert small_rounds >= big_rounds >= 1
            more.append(small_rounds > big_rounds)
        assert any(more)
    finally:
        a.close()
        b.close()


def test_set_param_between_batches(host_index, tmp_path):
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    values = {"PostingVectorLimit": "1"}  # SearchPostingPageLimit alone decides the truncation, as in PARAMS["pages"]
    s = host_index(files, values)
    dev = host_index(files, values, sub="device", placement="device")
    q = g["queries"]
    for pname, changes in (("ratio", {"MaxDistRatio": "1.5"}), ("default", {"MaxDistRatio": "10000"}),
                           ("pages", {"SearchPostingPageLimit": "1"}), ("default", {"SearchPostingPageLimit": "12"}),
                           (None, {"SearchInternalResultNum": "8"}), (None, {"SearchInternalResultNum": "200"}),
                           ("default", {"SearchInternalResultNum": "64"})):
        for name, v in changes.items():
            s.set_param(name, v)
            dev.set_param(name, v)
        for k in (10, 100):
            ids, dists = s.search(q, k)
            if pname is None:  # no recorded results at this SearchInternalResultNum: the HBM placement's
                want_ids, want_d = dev.search(q, k)
            else:
                want_ids, want_d = g["ids_%s_%d" % (pname, k)], g["dists_%s_%d" % (pname, k)]
            assert np.array_equal(ids, want_ids), (changes, k)
            assert np.array_equal(dists.view(np.int32), want_d.view(np.int32)), (changes, k)


@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_two_threads_on_one_handle(stage, host_index):
    g, files = _fixture(GOLDEN, "spann_i8_l2_2k_16")
    s = host_index(files)
    s.set_param("B200.PostingStageBytes", stage)
    q = g["queries"]
    want = {k: (g["ids_default_%d" % k], g["dists_default_%d" % k].view(np.int32)) for k in (10, 100)}
    errors = []

    def run(k):
        try:
            for _ in range(20):
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, want[k][0])
                assert np.array_equal(dists.view(np.int32), want[k][1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(k,)) for k in (10, 100)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


@pytest.mark.parametrize("case", CASES)
def test_placement_reporting(case, host_index):
    _, files = _fixture(GOLDEN, case)
    folder = oracle_spann.SpannFolder(files)
    total = sum(l[0] for l in folder.lists)
    rows_and_ids = (total + 1) * elem_bytes(folder)
    host = host_index(files, sub="host")
    dev = host_index(files, sub="device", placement="device")
    old = host_index(files, sub="old", placement=None)
    auto = host_index(files, sub="auto", placement="auto")
    assert dev.get_param("B200.PostingPlacement") == "device"
    assert old.get_param("B200.PostingPlacement") == "device"
    assert auto.get_param("B200.PostingPlacement") == "device"  # a fixture's lists fit in HBM
    assert int(dev.get_param("B200.PostingHostBytes")) == 0
    assert int(dev.get_param("PostingBytes")) == int(old.get_param("PostingBytes"))
    assert int(dev.get_param("PostingBytes")) - int(host.get_param("PostingBytes")) >= rows_and_ids
    assert int(host.get_param("B200.PostingHostBytes")) >= rows_and_ids
    with pytest.raises(capi.SptagB200Error):
        host.set_param("B200.PostingHostBytes", 1)
    with pytest.raises(capi.SptagB200Error):
        host.set_param("B200.PostingStageBytes", -1)


def test_unknown_placement_is_refused(tmp_path):
    _, files = _fixture(GOLDEN, "spann_l2_3k_16")
    write_folder(files, str(tmp_path))
    with pytest.raises(ValueError):
        capi.B200SpannIndex.load(str(tmp_path), 0, posting_placement="ssd")
    L = capi.lib()
    h = capi.C.c_void_p()
    o = capi.SpannLoadOptions(capi.C.sizeof(capi.SpannLoadOptions), 7)
    assert L.sptag_b200_spann_load_ex(os.fsencode(str(tmp_path)), 0, capi.C.byref(o), capi.C.byref(h)) == LACK_OF_INPUTS
