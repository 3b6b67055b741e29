"""SPANN with the posting lists left in their files (sptag_b200_spann_load_ex, posting_placement="file"): each search,
iterator step or cache install reads its union of lists from the posting files into the HBM stage.  Against the
reference's results recorded in tests/golden/spann, spann_elem, spann_pq, spann_iter and spann_elem_iter: ids and
distance bits of every case, parameter set and K, at the default stage and at B200.PostingStageBytes 0; the staged bytes
and rounds against the restatement of the union and the halving rule, and the file bytes read against the same rounds;
the cache against a host-placed handle's; files moved, truncated and restored under a loaded handle; the load's
refusals; and two threads on one handle."""
import os
import threading

import numpy as np
import pytest

import oracle_spann
import oracle_spann_pq
from golden.make_golden_spann import KS, PARAMS, write_folder
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from golden.make_golden_spann_pq import MODES
from sptag_b200 import capi
from test_gpu_spann_host import DEFAULT_STAGE, _refused_truncation, chosen_lists, elem_bytes, gather_rounds
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann")
GOLDEN_ELEM = os.path.join(HERE, "golden", "spann_elem")
GOLDEN_PQ = os.path.join(HERE, "golden", "spann_pq")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_iter")
GOLDEN_ELEM_ITER = os.path.join(HERE, "golden", "spann_elem_iter")
FAIL = 0x01
LACK_OF_INPUTS = 0x13


def _cases(golden):
    return sorted(f[:-4] for f in os.listdir(golden) if f.endswith(".npz"))


CASES = [(GOLDEN, c) for c in _cases(GOLDEN)] + [(GOLDEN_ELEM, c) for c in _cases(GOLDEN_ELEM)]
PQ_CASES = _cases(GOLDEN_PQ)
ITER_CASES = [(GOLDEN, GOLDEN_ITER, c) for c in _cases(GOLDEN_ITER)] + \
             [(GOLDEN_ELEM, GOLDEN_ELEM_ITER, c) for c in _cases(GOLDEN_ELEM_ITER)]


def _id(case):
    return case[-1]


@pytest.fixture
def spann(tmp_path):
    """load(files, values, sub, placement) -> (handle, folder); every handle is closed after the test"""
    opened = []

    def load(files, values=None, sub="index", placement="file"):
        folder = str(tmp_path / sub)
        write_folder(files, folder, values or {})
        s = capi.B200SpannIndex.load(folder, 0, posting_placement=placement)
        opened.append(s)
        return s, folder

    yield load
    for s in opened:
        s.close()


def _fixture(golden, case):
    g = np.load(os.path.join(golden, case + ".npz"))
    return g, oracle_spann.fixture_files(g)


def posting_files(folder):
    """The posting files a folder's lists are read from: SSDIndex, SSDIndex_1, ..."""
    ini = oracle_spann.parse_ini(open(os.path.join(folder, "indexloader.ini")).read())
    name = ini["BuildSSDIndex"].get("SSDIndex", ini["Base"].get("SSDIndex", "SPTAGFullList.bin"))
    out = []
    while os.path.exists(os.path.join(folder, name if not out else "%s_%d" % (name, len(out)))):
        out.append(os.path.join(folder, name if not out else "%s_%d" % (name, len(out))))
    return out


def read_bytes(folder, per_query, stage, cached=()):
    """The file bytes the rounds of gather_rounds read: each round's union of uncached lists, element count x vis (the
    searched prefix, or the whole list of the rearranged layout, which is never truncated here)"""
    eb = elem_bytes(folder)
    per_query = [q - set(cached) for q in per_query]
    rounds = gather_rounds(folder, per_query, stage)
    return sum(r // eb for r in rounds) * folder.vis, rounds


def assert_staged(s, folder, head_ids, head_dists, stage, cached=()):
    per_query = [set(chosen_lists(folder, i, d)) for i, d in zip(head_ids, head_dists)]
    want_read, rounds = read_bytes(folder, per_query, stage, cached)
    assert int(s.get_param("B200.LastGatherBytes")) == sum(rounds)
    assert int(s.get_param("B200.LastGatherRounds")) == len(rounds)
    assert int(s.get_param("B200.LastReadBytes")) == want_read
    return rounds


def assert_search(s, g, folder, pname, q, stage, ks=KS):
    for k in ks:
        ids, dists, stats = s.search(q, k, want_stats=True)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (pname, k, stage)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (pname, k, stage)
        hid, hd = g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)]
        _, _, st = oracle_spann.search(folder, q, hid, hd, k)
        assert np.array_equal(stats, st), (pname, k, stage)
        assert_staged(s, folder, hid, hd, stage)


@pytest.mark.parametrize("case", CASES, ids=_id)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_file_search_equals_reference(case, pname, spann):
    """Every K at the default stage and at the smallest one: results, stats, staged bytes, rounds and file bytes"""
    g, files = _fixture(*case)
    s, _ = spann(files, PARAMS[pname])
    assert s.get_param("B200.PostingPlacement") == "file"
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        with pytest.raises(capi.SptagB200Error) as e:
            s.search(g["queries"], 10)
        assert e.value.code == LACK_OF_INPUTS
        return
    for stage in (DEFAULT_STAGE, 0):
        s.set_param("B200.PostingStageBytes", stage)
        assert_search(s, g, folder, pname, g["queries"], stage)


@pytest.mark.parametrize("case", PQ_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
def test_file_pq_search_equals_reference(case, pname, mode, spann):
    """Code rows (vis = M + 4) read from the files, scanned with SDC and ADC"""
    g, files = _fixture(GOLDEN_PQ, case)
    s, _ = spann(files, dict(PARAMS[pname], EnableADC="true" if mode == "adc" else "false"))
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
            assert_staged(s, folder, hid, hd, stage)


@pytest.mark.parametrize("case", ITER_CASES, ids=_id)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_file_iterators_equal_reference(case, pname, sname, stage, spann):
    golden, golden_iter, name = case
    g = np.load(os.path.join(golden_iter, name + ".npz"))
    src = np.load(os.path.join(golden, name + ".npz"))
    files = oracle_spann.fixture_files(src)
    refused = _refused_truncation(oracle_spann.SpannFolder(files, ITER_PARAMS[pname]))
    if not applies(name, pname) and not refused:
        pytest.skip("no recorded calls (the pages set is not run on the rearranged layout), and no list is truncated")
    s, _ = spann(files, ITER_PARAMS[pname])
    s.set_param("B200.PostingStageBytes", stage)
    q = schedule_queries(src["queries"], sname)
    it = s.iterators(q)
    try:
        if refused:
            with pytest.raises(capi.SptagB200Error) as e:
                it.next(10)
            assert e.value.code == LACK_OF_INPUTS
            return
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
        assert int(s.get_param("B200.LastGatherRounds")) >= 1
    finally:
        it.close()
    assert_calls_equal(got, want, (name, pname, sname, stage))


@pytest.mark.parametrize("case", ["spann_l2_3k_16", "spann_cos_rearr_2k_24", "spann_i8_l2_2k_16"])
def test_cache_on_a_file_handle(case, spann):
    """cache_warm takes the lists a host-placed handle takes; cached lists are never read; cache_lists([]) releases"""
    g, files = _fixture(GOLDEN, case)
    folder = oracle_spann.SpannFolder(files)
    s, _ = spann(files)
    host, _ = spann(files, sub="host", placement="host")
    q = g["queries"]
    every = sum(l[0] for l in folder.lists) * elem_bytes(folder)
    hid, hd = g["head_ids_default_10"], g["head_dists_default_10"]
    for budget in (every // 2, every):
        got = s.cache_warm(q, budget)
        assert got.tolist() == host.cache_warm(q, budget).tolist()
        assert int(s.get_param("B200.LastReadBytes")) == sum(folder.lists[l][0] for l in got) * folder.vis
        assert int(s.get_param("B200.PostingCacheBytes")) == int(host.get_param("B200.PostingCacheBytes"))
        for stage in (DEFAULT_STAGE, 0):
            s.set_param("B200.PostingStageBytes", stage)
            for k in (10, 100):
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, g["ids_default_%d" % k]), (budget, stage, k)
                assert np.array_equal(dists.view(np.int32), g["dists_default_%d" % k].view(np.int32)), (budget, stage, k)
                assert_staged(s, folder, g["head_ids_default_%d" % k], g["head_dists_default_%d" % k], stage,
                              cached=got.tolist())
    # every list cached: nothing is staged or read
    s.cache_lists(list(range(len(folder.lists))))
    for k in (10, 100):
        ids, dists = s.search(q, k)
        assert np.array_equal(ids, g["ids_default_%d" % k]), k
        assert np.array_equal(dists.view(np.int32), g["dists_default_%d" % k].view(np.int32)), k
        assert int(s.get_param("B200.LastReadBytes")) == 0
        assert int(s.get_param("B200.LastGatherBytes")) == 0
    s.cache_lists([])
    assert int(s.get_param("B200.PostingCacheLists")) == 0
    s.set_param("B200.PostingStageBytes", DEFAULT_STAGE)
    ids, dists = s.search(q, 10)
    assert np.array_equal(ids, g["ids_default_10"])
    assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32))
    assert_staged(s, folder, hid, hd, DEFAULT_STAGE)


def _assert_default_10(s, g):
    ids, dists = s.search(g["queries"], 10)
    assert np.array_equal(ids, g["ids_default_10"])
    assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32))


@pytest.mark.parametrize("case", ["spann_l2_3k_16", "spann_i8_l2_2k_16"])
def test_files_are_read_at_search_time(case, spann):
    """A posting file moved away, then back; truncated, then restored: Fail naming the file, then the golden results on
    the same handle"""
    g, files = _fixture(GOLDEN, case)
    s, folder = spann(files)
    _assert_default_10(s, g)
    for path in posting_files(folder):
        os.rename(path, path + ".away")
        with pytest.raises(capi.SptagB200Error) as e:
            s.search(g["queries"], 10)
        assert e.value.code == FAIL and path in str(e.value), str(e.value)
        os.rename(path + ".away", path)
        _assert_default_10(s, g)
        blob = open(path, "rb").read()
        os.truncate(path, 4096)
        with pytest.raises(capi.SptagB200Error) as e:
            s.search(g["queries"], 10)
        assert e.value.code == FAIL and path in str(e.value), str(e.value)
        with open(path, "r+b") as fh:
            fh.write(blob)
        _assert_default_10(s, g)


def test_load_refusals_and_reporting(spann, tmp_path):
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    s, folder = spann(files)
    assert s.get_param("B200.PostingPlacement") == "file"
    assert int(s.get_param("B200.PostingHostBytes")) == 0
    host, _ = spann(files, sub="host", placement="host")
    assert int(s.get_param("PostingBytes")) == int(host.get_param("PostingBytes"))
    assert int(s.get_param("B200.LastReadBytes")) == 0
    with pytest.raises(capi.SptagB200Error):
        s.set_param("B200.LastReadBytes", 1)
    # a posting file cut one byte short of its last list's end (the page padding after it gone too)
    cut = str(tmp_path / "cut")
    write_folder(files, cut)
    path = posting_files(cut)[-1]
    blob = open(path, "rb").read()
    parsed = oracle_spann.SpannFolder(files)
    end = max(start + ele * parsed.vis for ele, _, data, start in parsed.lists if data == blob and ele > 0)
    os.truncate(path, end - 1)
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.load(cut, 0, posting_placement="file")
    assert e.value.code == FAIL
    for key in ("EnableDataCompression", "EnableDeltaEncoding"):
        refused = str(tmp_path / key)
        write_folder(files, refused, {key: "true"})
        with pytest.raises(capi.SptagB200Error) as e:
            capi.B200SpannIndex.load(refused, 0, posting_placement="file")
        assert e.value.code == LACK_OF_INPUTS


@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_two_threads_on_one_handle(stage, spann):
    g, files = _fixture(GOLDEN, "spann_i8_l2_2k_16")
    s, _ = spann(files)
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
