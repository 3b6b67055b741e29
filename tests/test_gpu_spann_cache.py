"""SPANN with the posting lists in pinned host memory and an HBM cache of some of them (sptag_b200_spann_cache_warm,
sptag_b200_spann_cache_lists): cached lists are read in place from the cache, only the others are gathered over the host
link.  Against the reference's results recorded in tests/golden/spann, spann_pq, spann_iter, spann_elem and
spann_elem_iter: ids and distance bits with a warmed cache, every list cached and every other list cached; the gathered
bytes and rounds against the union and halving rule over the uncached lists only, at the default stage and the smallest
one; the ranking cache_warm returns against a numpy restatement at several budgets; page-limit changes after install;
installs while two threads search; an iterator opened before an install; and the refusals."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import oracle_spann
from golden.make_golden_spann import KS, PARAMS
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from golden.make_golden_spann_pq import MODES
from sptag_b200 import capi
from test_gpu_spann_host import (DEFAULT_STAGE, LACK_OF_INPUTS, _fixture, _refused_truncation, chosen_lists,
                                 elem_bytes, gather_rounds, host_index)  # noqa: F401 (host_index is a fixture)
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann")
GOLDEN_PQ = os.path.join(HERE, "golden", "spann_pq")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_iter")
GOLDEN_ELEM = os.path.join(HERE, "golden", "spann_elem")
GOLDEN_ELEM_ITER = os.path.join(HERE, "golden", "spann_elem_iter")


def _cases(golden):
    return sorted(f[:-4] for f in os.listdir(golden) if f.endswith(".npz"))


CASES, PQ_CASES, ITER_CASES = _cases(GOLDEN), _cases(GOLDEN_PQ), _cases(GOLDEN_ITER)
ELEM_CASES, ELEM_ITER_CASES = _cases(GOLDEN_ELEM), _cases(GOLDEN_ELEM_ITER)


def list_bytes(folder, l):
    """What caching list l takes: every element, whatever the page limit"""
    return folder.lists[l][0] * elem_bytes(folder)


def all_list_bytes(folder):
    return sum(list_bytes(folder, l) for l in range(len(folder.lists)))


def every_other(folder):
    return list(range(0, len(folder.lists), 2))


def ranking(folder, head_ids, head_dists, budget):
    """cache_warm's choice restated: the lists the queries choose, counted, ordered by (-count, id) and taken greedily by
    full-list bytes while they fit the budget (None: no limit)"""
    counts = np.zeros(len(folder.lists), np.int64)
    for i, d in zip(head_ids, head_dists):
        for l in chosen_lists(folder, i, d):
            counts[l] += 1
    order = sorted((l for l in range(len(counts)) if counts[l] > 0), key=lambda l: (-counts[l], l))
    taken, left = [], budget
    for l in order:
        if left is None or list_bytes(folder, l) <= left:
            taken.append(l)
            if left is not None:
                left -= list_bytes(folder, l)
    return taken


def assert_cache_params(s, folder, lists):
    assert int(s.get_param("B200.PostingCacheLists")) == len(lists)
    assert int(s.get_param("B200.PostingCacheBytes")) == sum(list_bytes(folder, l) for l in lists)
    assert s.get_param("B200.PostingPlacement") == "host"


def assert_gathered(s, folder, head_ids, head_dists, cached, stage=DEFAULT_STAGE):
    cached = set(cached)
    per_query = [set(chosen_lists(folder, i, d)) - cached for i, d in zip(head_ids, head_dists)]
    want = gather_rounds(folder, per_query, stage)
    assert int(s.get_param("B200.LastGatherBytes")) == sum(want)
    assert int(s.get_param("B200.LastGatherRounds")) == len(want)
    return want


def assert_search(s, g, folder, pname, cached, stage=DEFAULT_STAGE, ks=KS):
    for k in ks:
        ids, dists = s.search(g["queries"], k)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (pname, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (pname, k)
        assert_gathered(s, folder, g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)], cached, stage)


def warm_half(s, g, folder, pname):
    """cache_warm with the fixture's own queries at half of all list bytes, checked against the restatement"""
    budget = all_list_bytes(folder) // 2
    got = s.cache_warm(g["queries"], budget)
    want = ranking(folder, g["head_ids_%s_10" % pname], g["head_dists_%s_10" % pname], budget)
    assert got.dtype == np.int32 and got.tolist() == want
    assert_cache_params(s, folder, want)
    return want


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_cached_search_equals_reference(case, pname, host_index):
    """A warmed cache at half the list bytes, every list, every other list: results and gathered bytes and rounds"""
    g, files = _fixture(GOLDEN, case)
    s = host_index(files, PARAMS[pname])
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        with pytest.raises(capi.SptagB200Error) as e:
            s.cache_warm(g["queries"])
        assert e.value.code == LACK_OF_INPUTS
        return
    assert_search(s, g, folder, pname, warm_half(s, g, folder, pname))
    every = list(range(len(folder.lists)))
    s.cache_lists(every)
    assert_cache_params(s, folder, every)
    assert_search(s, g, folder, pname, every)
    assert int(s.get_param("B200.LastGatherBytes")) == 0
    s.cache_lists(every_other(folder))
    assert_cache_params(s, folder, every_other(folder))
    assert_search(s, g, folder, pname, every_other(folder))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_cached_smallest_stage(case, pname, host_index):
    """B200.PostingStageBytes 0 with every other list cached: the halving rule counts the uncached elements only"""
    g, files = _fixture(GOLDEN, case)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        pytest.skip("truncated lists of the rearranged layout: refused on either placement")
    s = host_index(files, PARAMS[pname])
    s.set_param("B200.PostingStageBytes", 0)
    s.cache_lists(every_other(folder))
    assert_search(s, g, folder, pname, every_other(folder), stage=0)
    s.set_param("B200.PostingStageBytes", DEFAULT_STAGE)  # a larger stage than the cache was installed with
    assert_search(s, g, folder, pname, every_other(folder))


@pytest.mark.parametrize("case", PQ_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
def test_cached_pq_search_equals_reference(case, pname, mode, host_index):
    g, files = _fixture(GOLDEN_PQ, case)
    s = host_index(files, dict(PARAMS[pname], EnableADC="true" if mode == "adc" else "false"))
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    q = g["queries"]
    w = folder.internal
    warm = s.cache_warm(q, all_list_bytes(folder) // 2).tolist()
    assert warm == ranking(folder, g["head_ids_%s_%d" % (mode, w)], g["head_dists_%s_%d" % (mode, w)],
                           all_list_bytes(folder) // 2)
    for cached in (warm, every_other(folder)):
        s.cache_lists(cached)
        for k in KS:
            ids, dists = s.search(q, k)
            key = "%s_%s_%d" % (mode, pname, k)
            assert np.array_equal(ids, g["ids_" + key]), key
            assert np.array_equal(dists.view(np.int32), g["dists_" + key].view(np.int32)), key
            hw = max(k, w)
            assert_gathered(s, folder, g["head_ids_%s_%d" % (mode, hw)], g["head_dists_%s_%d" % (mode, hw)], cached)


@pytest.mark.parametrize("case", ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_cached_iterators_equal_reference(case, pname, sname, stage, host_index):
    g = np.load(os.path.join(GOLDEN_ITER, case + ".npz"))
    src = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    if not applies(case, pname):
        pytest.skip("no recorded calls: the pages set truncates lists of the rearranged layout")
    s = host_index(files, ITER_PARAMS[pname])
    s.set_param("B200.PostingStageBytes", stage)
    s.cache_warm(src["queries"], all_list_bytes(oracle_spann.SpannFolder(files)) // 2)
    assert int(s.get_param("B200.PostingCacheLists")) > 0
    q = schedule_queries(src["queries"], sname)
    it = s.iterators(q)
    try:
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
    finally:
        it.close()
    assert_calls_equal(got, want, (case, pname, sname, stage))


@pytest.mark.parametrize("case", ITER_CASES)
def test_iterator_opened_before_an_install(case, host_index):
    """An iterator holds list ids and positions, not addresses: installs between its calls leave its results unchanged"""
    g = np.load(os.path.join(GOLDEN_ITER, case + ".npz"))
    src = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    folder = oracle_spann.SpannFolder(files)
    s = host_index(files)
    q = schedule_queries(src["queries"], "short")
    sched, want = expected(g, "default_short", len(q))
    installs = [every_other(folder), list(range(len(folder.lists))), [], list(range(1, len(folder.lists), 2)), []]
    it = s.iterators(q)
    try:
        got = []
        for i, b in enumerate(sched):
            got.append(it.next(int(b)))
            s.cache_lists(installs[i % len(installs)])
    finally:
        it.close()
    assert_calls_equal(got, want, case)


@pytest.mark.parametrize("case", ELEM_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("stage", [DEFAULT_STAGE, 0])
def test_cached_elem_search_equals_reference(case, pname, stage, host_index):
    """uint8, int16 and integer-cosine rows with padded row strides, every other list cached"""
    g, files = _fixture(GOLDEN_ELEM, case)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        pytest.skip("truncated lists of the rearranged layout: refused on either placement")
    s = host_index(files, PARAMS[pname])
    s.set_param("B200.PostingStageBytes", stage)
    s.cache_lists(every_other(folder))
    assert_cache_params(s, folder, every_other(folder))
    assert_search(s, g, folder, pname, every_other(folder), stage)


@pytest.mark.parametrize("case", ELEM_ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
def test_cached_elem_iterators_equal_reference(case, pname, sname, host_index):
    g = np.load(os.path.join(GOLDEN_ELEM_ITER, case + ".npz"))
    src = np.load(os.path.join(GOLDEN_ELEM, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    folder = oracle_spann.SpannFolder(files, ITER_PARAMS[pname])
    if _refused_truncation(folder) or not applies(case, pname):
        pytest.skip("truncated lists of the rearranged layout: refused on either placement")
    s = host_index(files, ITER_PARAMS[pname])
    s.cache_lists(every_other(folder))
    q = schedule_queries(src["queries"], sname)
    it = s.iterators(q)
    try:
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
    finally:
        it.close()
    assert_calls_equal(got, want, (case, pname, sname))


@pytest.mark.parametrize("case", CASES)
def test_warm_ranking(case, host_index):
    """The lists cache_warm takes, in rank order, at budgets 0, one byte below the first-ranked list, a third and half
    of all list bytes, and -1 (free HBM less 1 GB: every chosen list of a fixture)"""
    g, files = _fixture(GOLDEN, case)
    folder = oracle_spann.SpannFolder(files)
    s = host_index(files)
    q, hid, hd = g["queries"], g["head_ids_default_10"], g["head_dists_default_10"]
    everything = ranking(folder, hid, hd, None)
    first = list_bytes(folder, everything[0])
    total = all_list_bytes(folder)
    for budget in (0, first - 1, first, total // 3, total // 2, -1):
        got = s.cache_warm(q, budget).tolist()
        want = everything if budget == -1 else ranking(folder, hid, hd, budget)
        assert got == want, budget
        assert_cache_params(s, folder, want)
        if budget == 0:
            assert want == []
        if budget == first - 1:
            assert everything[0] not in got
        ids, dists = s.search(q, 10)
        assert np.array_equal(ids, g["ids_default_10"]), budget
        assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32)), budget
        assert_gathered(s, folder, hid, hd, want)
    # the full count when the caller's array is shorter: only the first `capacity` ids are written
    out = np.full(2, -7, np.int32)
    n = C.c_int32(-1)
    L = capi.lib()
    assert L.sptag_b200_spann_cache_warm(s._h, q.ctypes.data, len(q), -1, out.ctypes.data, 2, C.byref(n)) == 0
    assert n.value == len(everything) and out.tolist() == everything[:2]
    assert L.sptag_b200_spann_cache_warm(s._h, q.ctypes.data, len(q), 0, None, 0, C.byref(n)) == 0
    assert n.value == 0


def test_page_limit_change_after_install(host_index):
    """Cached lists hold every element: a page limit set after the install reads its prefix of them"""
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    values = {"PostingVectorLimit": "1"}  # SearchPostingPageLimit alone decides the truncation, as in PARAMS["pages"]
    s = host_index(files, values)
    folder = oracle_spann.SpannFolder(files, values)
    s.cache_lists(every_other(folder))
    for pname, limit in (("pages", "1"), ("default", "12"), ("pages", "1")):
        s.set_param("SearchPostingPageLimit", limit)
        f = oracle_spann.SpannFolder(files, dict(values, SearchPostingPageLimit=limit))
        assert_search(s, g, f, pname, every_other(folder), ks=(10, 100))
    cached = s.cache_warm(g["queries"]).tolist()  # ranked at page limit 1, read at 12
    s.set_param("SearchPostingPageLimit", "12")
    f = oracle_spann.SpannFolder(files, dict(values, SearchPostingPageLimit="12"))
    assert_search(s, g, f, "default", cached, ks=(10, 100))


def test_installs_while_two_threads_search(host_index):
    g, files = _fixture(GOLDEN, "spann_i8_l2_2k_16")
    folder = oracle_spann.SpannFolder(files)
    s = host_index(files)
    q = g["queries"]
    want = {k: (g["ids_default_%d" % k], g["dists_default_%d" % k].view(np.int32)) for k in (10, 100)}
    sets = [[], every_other(folder), list(range(len(folder.lists)))]
    errors = []
    done = threading.Event()

    def run(k):
        try:
            for _ in range(30):
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, want[k][0])
                assert np.array_equal(dists.view(np.int32), want[k][1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    def install():
        try:
            i = 0
            while not done.is_set() or i < len(sets):
                s.cache_lists(sets[i % len(sets)])
                i += 1
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    searchers = [threading.Thread(target=run, args=(k,)) for k in (10, 100)]
    installer = threading.Thread(target=install)
    installer.start()
    for t in searchers:
        t.start()
    for t in searchers:
        t.join()
    done.set()
    installer.join()
    assert not errors, errors


def test_refusals_and_release(host_index):
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    folder = oracle_spann.SpannFolder(files)
    nl = len(folder.lists)
    q = g["queries"]
    L = capi.lib()
    dev = host_index(files, sub="device", placement="device")
    s = host_index(files, sub="host")
    n = C.c_int32()

    def lists(ids):
        a = np.asarray(ids, np.int32)
        return L.sptag_b200_spann_cache_lists(s._h, a.ctypes.data, len(a))

    one = np.zeros(1, np.int32)
    assert L.sptag_b200_spann_cache_lists(dev._h, one.ctypes.data, 1) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(dev._h, q.ctypes.data, len(q), -1, None, 0, C.byref(n)) == LACK_OF_INPUTS
    s.cache_lists(every_other(folder))
    for bad in ([nl], [-1], [3, 5, 3]):
        assert lists(bad) == LACK_OF_INPUTS, bad
    assert L.sptag_b200_spann_cache_lists(s._h, None, 2) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(s._h, None, 4, -1, None, 0, C.byref(n)) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(s._h, q.ctypes.data, len(q), -1, None, 0, None) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(s._h, q.ctypes.data, len(q), -1, None, 3, C.byref(n)) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(s._h, q.ctypes.data, len(q), -2, None, 0, C.byref(n)) == LACK_OF_INPUTS
    assert_cache_params(s, folder, every_other(folder))  # a refused call leaves the cache as it was
    with pytest.raises(capi.SptagB200Error):
        s.set_param("B200.PostingCacheLists", 1)
    assert L.sptag_b200_spann_cache_lists(s._h, None, 0) == 0
    assert s.get_param("B200.PostingCacheLists") == "0" and s.get_param("B200.PostingCacheBytes") == "0"
    assert dev.get_param("B200.PostingCacheLists") == "0" and dev.get_param("B200.PostingCacheBytes") == "0"
    ids, dists = s.search(q, 10)
    assert np.array_equal(ids, g["ids_default_10"])
    assert int(s.get_param("B200.LastGatherBytes")) > 0


def test_stage_changes_while_installing(host_index):
    """B200.PostingStageBytes raised and lowered while installs and searches run: a search never meets a cache whose
    stage is smaller than its own (it refits and takes its set again), so no call fails"""
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    folder = oracle_spann.SpannFolder(files)
    s = host_index(files)
    q = g["queries"]
    want = (g["ids_default_10"], g["dists_default_10"].view(np.int32))
    sets = [every_other(folder), list(range(len(folder.lists))), list(range(1, len(folder.lists), 2))]
    errors = []
    done = threading.Event()

    def search():
        try:
            for _ in range(30):
                ids, dists = s.search(q, 10)
                assert np.array_equal(ids, want[0])
                assert np.array_equal(dists.view(np.int32), want[1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    def churn(step):
        try:
            i = 0
            while not done.is_set():
                step(i)
                i += 1
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=search) for _ in range(2)]
    churners = [threading.Thread(target=churn, args=(lambda i: s.cache_lists(sets[i % len(sets)]),)),
                threading.Thread(target=churn, args=(lambda i: s.set_param("B200.PostingStageBytes",
                                                                           (0, 1 << 20, 8 << 20)[i % 3]),))]
    for t in churners + threads:
        t.start()
    for t in threads:
        t.join()
    done.set()
    for t in churners:
        t.join()
    assert not errors, errors


def test_warm_refuses_a_width_the_head_search_cannot_run(host_index):
    """SearchInternalResultNum above 2048 from the folder: cache_warm refuses it as a search does"""
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    s = host_index(files, {"SearchInternalResultNum": "3000"})
    for call in (lambda: s.search(g["queries"], 10), lambda: s.cache_warm(g["queries"])):
        with pytest.raises(capi.SptagB200Error) as e:
            call()
        assert e.value.code == LACK_OF_INPUTS
    assert s.get_param("B200.PostingCacheLists") == "0"
