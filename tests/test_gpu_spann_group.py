"""A SPANN group (sptag_b200_spann_group_*): one pinned copy of the posting lists shared by members on several devices,
an HBM cache spread over the members with each list held at most once, and a gather that reads a list another member
caches from that member's HBM.  Members sit on devices i % device_count, so two members may share one GPU.  Against the
reference's results recorded in tests/golden/spann, spann_elem, spann_pq, spann_iter and spann_elem_iter: ids and
distance bits of groups of 2 and 3 with no cache, a warmed cache, every list on member 1 and lists dealt alternately;
each member's gathered bytes and rounds against the union and halving rule over the lists it does not cache; the warm
assignment against a numpy restatement; member iterators on peer-cached lists; installs while two threads search; a
stage that grows after an install; peers on different devices; and the refusals."""
import ctypes as C
import os
import threading

import numpy as np
import pytest
import torch

import oracle_spann
import oracle_spann_pq
from golden.make_golden_spann import KS, PARAMS, write_folder
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from golden.make_golden_spann_pq import MODES
from sptag_b200 import capi
from test_gpu_spann_cache import all_list_bytes, list_bytes, ranking
from test_gpu_spann_host import (DEFAULT_STAGE, LACK_OF_INPUTS, _fixture, _refused_truncation, chosen_lists,
                                 elem_bytes, gather_rounds)
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann")
GOLDEN_ELEM = os.path.join(HERE, "golden", "spann_elem")
GOLDEN_PQ = os.path.join(HERE, "golden", "spann_pq")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_iter")
GOLDEN_ELEM_ITER = os.path.join(HERE, "golden", "spann_elem_iter")
FAIL = 0x01


def _cases(golden):
    return sorted(f[:-4] for f in os.listdir(golden) if f.endswith(".npz"))


RAW_CASES = [(GOLDEN, c) for c in _cases(GOLDEN)] + [(GOLDEN_ELEM, c) for c in _cases(GOLDEN_ELEM)]
PQ_CASES = _cases(GOLDEN_PQ)
ITER_CASES = [(GOLDEN_ITER, GOLDEN, c) for c in _cases(GOLDEN_ITER)] + \
             [(GOLDEN_ELEM_ITER, GOLDEN_ELEM, c) for c in _cases(GOLDEN_ELEM_ITER)]


def member_devices(n):
    return [i % torch.cuda.device_count() for i in range(n)]


def reachable(devices, i, o):
    """Whether member i reads member o's cache: the same device, or one peer access reaches"""
    a, b = devices[i], devices[o]
    return a == b or torch.cuda.can_device_access_peer(a, b)


@pytest.fixture
def spann_group(tmp_path):
    """B200SpannGroup.load of a fixture's files written with ini values, members on member_devices(n); closed after"""
    opened = []

    def load(files, values=None, n=2, sub="index", devices=None):
        folder = str(tmp_path / sub)
        write_folder(files, folder, values or {})
        gr = capi.B200SpannGroup.load(folder, member_devices(n) if devices is None else devices)
        gr.devices = member_devices(n) if devices is None else list(devices)
        opened.append(gr)
        return gr

    yield load
    for gr in opened:
        gr.close()


def assign(folder, order, budget, n):
    """group_cache_warm's assignment restated: walk the ranking, each list to the member with the most budget left
    (ties: the lower index) when that member holds it whole, else skipped"""
    left = [budget] * n
    lists, owners = [], []
    for l in order:
        o = max(range(n), key=lambda i: (left[i], -i))
        if left[o] < list_bytes(folder, l):
            continue
        lists.append(l)
        owners.append(o)
        left[o] -= list_bytes(folder, l)
    return lists, owners


def assert_members_gathered(gr, folder, head_ids, head_dists, owner_of):
    """Each member's gathered bytes and rounds over its slice and the lists it does not cache itself; its peer bytes
    within them (all of them when every chosen list sits on a reachable peer)"""
    n = len(gr.members)
    nq = len(head_ids)
    per = -(-nq // n)
    for i, m in enumerate(gr.members):
        b, e = i * per, min((i + 1) * per, nq)
        if b >= e:
            continue
        per_query = [{l for l in chosen_lists(folder, h, d) if owner_of.get(l) != i}
                     for h, d in zip(head_ids[b:e], head_dists[b:e])]
        want = gather_rounds(folder, per_query)
        gathered, peer = int(m.get_param("B200.LastGatherBytes")), int(m.get_param("B200.LastPeerGatherBytes"))
        assert gathered == sum(want), i
        assert int(m.get_param("B200.LastGatherRounds")) == len(want), i
        assert 0 <= peer <= gathered, i
        union = set().union(*per_query)
        from_peers = {l for l in union if l in owner_of and reachable(gr.devices, i, owner_of[l])}
        if union == from_peers:
            assert peer == gathered, i
        if not from_peers:
            assert peer == 0, i


def assert_group_search(gr, g, folder, key, head_key, owner_of, ks=KS, w_of=None):
    for k in ks:
        ids, dists, stats = gr.search(g["queries"], k, want_stats=True)
        assert np.array_equal(ids, g["ids_%s_%d" % (key, k)]), (key, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (key, k)].view(np.int32)), (key, k)
        assert stats.dtype == np.int64 and (stats[:, 0] > 0).any(), (key, k)
        hk = w_of(k) if w_of else k
        assert_members_gathered(gr, folder, g["head_ids_%s_%d" % (head_key, hk)], g["head_dists_%s_%d" % (head_key, hk)],
                                owner_of)


def assignments(gr, g, folder, head_ids, head_dists):
    """No cache, a warmed cache at all_list_bytes / (2n) per member, every list on member 1, lists dealt alternately:
    each installed in turn and yielded as {list: owner}"""
    n, nl = len(gr.members), len(folder.lists)
    gr.cache_lists([], [])
    yield {}
    budget = all_list_bytes(folder) // (2 * n)
    lists, owners = gr.cache_warm(g["queries"], budget)
    assert (lists.tolist(), owners.tolist()) == assign(folder, ranking(folder, head_ids, head_dists, None), budget, n)
    yield dict(zip(lists.tolist(), owners.tolist()))
    gr.cache_lists(range(nl), [1] * nl)
    for i, m in enumerate(gr.members):
        assert int(m.get_param("B200.PostingCacheLists")) == (nl if i == 1 else 0)
        want_peer = nl if i != 1 and reachable(gr.devices, i, 1) else 0
        assert int(m.get_param("B200.PostingPeerLists")) == want_peer, i
    yield {l: 1 for l in range(nl)}
    gr.cache_lists(range(nl), [l % n for l in range(nl)])
    yield {l: l % n for l in range(nl)}


@pytest.mark.parametrize("golden,case", RAW_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("n", [2, 3])
def test_group_search_equals_reference(golden, case, pname, n, spann_group):
    g, files = _fixture(golden, case)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    gr = spann_group(files, PARAMS[pname], n)
    if _refused_truncation(folder):
        with pytest.raises(capi.SptagB200Error) as e:
            gr.search(g["queries"], 10)
        assert e.value.code == LACK_OF_INPUTS
        return
    hid, hd = g["head_ids_%s_10" % pname], g["head_dists_%s_10" % pname]
    for owner_of in assignments(gr, g, folder, hid, hd):
        assert_group_search(gr, g, folder, pname, pname, owner_of)
        if owner_of and set(owner_of.values()) == {1} and reachable(gr.devices, 0, 1):
            m0 = gr.members[0]
            assert int(m0.get_param("B200.LastPeerGatherBytes")) == int(m0.get_param("B200.LastGatherBytes")) > 0


@pytest.mark.parametrize("case", PQ_CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [2, 3])
def test_group_pq_search_equals_reference(case, pname, mode, n, spann_group):
    g, files = _fixture(GOLDEN_PQ, case)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    gr = spann_group(files, dict(PARAMS[pname], EnableADC="true" if mode == "adc" else "false"), n)
    w = folder.internal
    for owner_of in assignments(gr, g, folder, g["head_ids_%s_%d" % (mode, w)], g["head_dists_%s_%d" % (mode, w)]):
        assert_group_search(gr, g, folder, "%s_%s" % (mode, pname), mode, owner_of, w_of=lambda k: max(k, w))
        ids, dists, stats = gr.search(g["queries"], 10, want_stats=True)
        _, _, st = oracle_spann_pq.search(folder, oracle_spann_pq.folder_quantizer(files), g["queries"],
                                          g["head_ids_%s_%d" % (mode, max(10, w))],
                                          g["head_dists_%s_%d" % (mode, max(10, w))], 10, mode == "adc")
        assert np.array_equal(stats, st)


@pytest.mark.parametrize("golden", [GOLDEN, GOLDEN_ELEM])
def test_warm_assignment(golden, spann_group):
    """group_cache_warm's (lists, owners) at budgets 0, one byte below the first-ranked list (it fits no member), half
    of it, a quarter and a half of all list bytes, and more than all of them, with 2 and 3 members"""
    for case in _cases(golden)[:2]:
        g, files = _fixture(golden, case)
        folder = oracle_spann.SpannFolder(files)
        q, hid, hd = g["queries"], g["head_ids_default_10"], g["head_dists_default_10"]
        order = ranking(folder, hid, hd, None)
        first, total = list_bytes(folder, order[0]), all_list_bytes(folder)
        for n in (2, 3):
            gr = spann_group(files, n=n, sub="%s_%d" % (case, n))
            for budget in (0, first - 1, first // 2, total // 4, total // 2, total + 1):
                lists, owners = gr.cache_warm(q, budget)
                want = assign(folder, order, budget, n)
                assert (lists.tolist(), owners.tolist()) == want, (case, n, budget)
                if budget == first - 1:
                    assert order[0] not in want[0]
                assert len(set(want[0])) == len(want[0])
                for i, m in enumerate(gr.members):
                    mine = [l for l, o in zip(*want) if o == i]
                    assert int(m.get_param("B200.PostingCacheLists")) == len(mine)
                    assert int(m.get_param("B200.PostingCacheBytes")) == sum(list_bytes(folder, l) for l in mine)
                ids, dists = gr.search(q, 10)
                assert np.array_equal(ids, g["ids_default_10"]), budget
                assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32)), budget


@pytest.mark.parametrize("golden_iter,golden,case", ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
def test_member_iterators_read_peer_lists(golden_iter, golden, case, pname, sname, spann_group):
    """Every list cached on member 1: member 0's iterators gather their lists from it"""
    gi = np.load(os.path.join(golden_iter, case + ".npz"))
    src = np.load(os.path.join(golden, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    folder = oracle_spann.SpannFolder(files, ITER_PARAMS[pname])
    if _refused_truncation(folder) or not applies(case, pname):
        pytest.skip("truncated lists of the rearranged layout: refused on either placement")
    gr = spann_group(files, ITER_PARAMS[pname])
    nl = len(folder.lists)
    gr.cache_lists(range(nl), [1] * nl)
    m0 = gr.members[0]
    q = schedule_queries(src["queries"], sname)
    it = m0.iterators(q)
    try:
        sched, want = expected(gi, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
    finally:
        it.close()
    assert_calls_equal(got, want, (case, pname, sname))
    if reachable(gr.devices, 0, 1):
        assert int(m0.get_param("B200.LastPeerGatherBytes")) == int(m0.get_param("B200.LastGatherBytes"))


def test_installs_while_two_threads_search(spann_group):
    g, files = _fixture(GOLDEN, "spann_i8_l2_2k_16")
    folder = oracle_spann.SpannFolder(files)
    nl = len(folder.lists)
    gr = spann_group(files)
    q = g["queries"]
    want = {k: (g["ids_default_%d" % k], g["dists_default_%d" % k].view(np.int32)) for k in (10, 100)}
    sets = [(range(nl), [1] * nl), (range(nl), [l % 2 for l in range(nl)])]
    errors = []
    done = threading.Event()

    def run(k):
        try:
            for _ in range(30):
                ids, dists = gr.search(q, k)
                assert np.array_equal(ids, want[k][0])
                assert np.array_equal(dists.view(np.int32), want[k][1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    def install():
        try:
            i = 0
            while not done.is_set() or i < len(sets):
                gr.cache_lists(*sets[i % len(sets)])
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


def test_stage_growth_moves_every_pool(spann_group):
    """B200.PostingStageBytes raised after an install re-installs each member's cache with a larger stage, so every pool
    moves; the peer tables follow and results stay the reference's"""
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    folder = oracle_spann.SpannFolder(files)
    nl = len(folder.lists)
    gr = spann_group(files, n=3)
    gr.set_param("B200.PostingStageBytes", 0)
    owner_of = {l: l % 3 for l in range(nl)}
    gr.cache_lists(list(owner_of), list(owner_of.values()))
    hid, hd = g["head_ids_default_10"], g["head_dists_default_10"]
    for stage in (0, DEFAULT_STAGE, 2 * DEFAULT_STAGE):
        gr.set_param("B200.PostingStageBytes", stage)
        ids, dists = gr.search(g["queries"], 10)
        assert np.array_equal(ids, g["ids_default_10"]), stage
        assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32)), stage
        for i, m in enumerate(gr.members):
            assert m.get_param("B200.PostingStageBytes") == str(stage)
            assert int(m.get_param("B200.PostingCacheLists")) == sum(1 for o in owner_of.values() if o == i)
        per = -(-len(hid) // 3)
        for i, m in enumerate(gr.members):
            per_query = [{l for l in chosen_lists(folder, h, d) if owner_of[l] != i}
                         for h, d in zip(hid[i * per:(i + 1) * per], hd[i * per:(i + 1) * per])]
            assert int(m.get_param("B200.LastGatherBytes")) == sum(gather_rounds(folder, per_query, stage)), (stage, i)


def test_refusals(spann_group, tmp_path):
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    folder = oracle_spann.SpannFolder(files)
    nl = len(folder.lists)
    L = capi.lib()
    path = str(tmp_path / "plain")
    write_folder(files, path)
    h = C.c_void_p()

    def load(devs):
        d = np.asarray(devs, np.int32)
        return L.sptag_b200_spann_group_load(os.fsencode(path), d.ctypes.data if len(d) else None, len(d), C.byref(h))

    assert load([]) == LACK_OF_INPUTS
    assert load([0] * 17) == LACK_OF_INPUTS
    assert load([torch.cuda.device_count()]) == FAIL
    assert load([-1]) == FAIL
    assert L.sptag_b200_spann_group_load(os.fsencode(path), None, 2, C.byref(h)) == LACK_OF_INPUTS
    # the folder refusals of sptag_b200_spann_load_ex, with its codes
    for key in ("EnableDataCompression", "EnableDeltaEncoding"):
        bad = str(tmp_path / key)
        write_folder(files, bad, {key: "true"})
        o = capi.SpannLoadOptions(C.sizeof(capi.SpannLoadOptions), capi.POSTING_PLACEMENTS["host"])
        single = L.sptag_b200_spann_load_ex(os.fsencode(bad), 0, C.byref(o), C.byref(h))
        d = np.zeros(2, np.int32)
        assert single == LACK_OF_INPUTS
        assert L.sptag_b200_spann_group_load(os.fsencode(bad), d.ctypes.data, 2, C.byref(h)) == single, key
    missing = np.zeros(2, np.int32)
    assert L.sptag_b200_spann_group_load(os.fsencode(str(tmp_path / "none")), missing.ctypes.data, 2, C.byref(h)) == \
        L.sptag_b200_spann_load_ex(os.fsencode(str(tmp_path / "none")), 0, None, C.byref(h))

    gr = spann_group(files)
    m0 = gr.members[0]
    q = g["queries"]
    n = C.c_int32()
    one = np.zeros(1, np.int32)
    assert L.sptag_b200_spann_cache_lists(m0._h, one.ctypes.data, 1) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_cache_warm(m0._h, q.ctypes.data, len(q), -1, None, 0, C.byref(n)) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_group_member(gr._h, 2, C.byref(h)) == LACK_OF_INPUTS
    assert L.sptag_b200_spann_group_member(gr._h, -1, C.byref(h)) == LACK_OF_INPUTS

    def lists(ls, os_):
        a, b = np.asarray(ls, np.int32), np.asarray(os_, np.int32)
        return L.sptag_b200_spann_group_cache_lists(gr._h, a.ctypes.data, b.ctypes.data, len(a))

    gr.cache_lists([0, 2], [1, 0])
    for ls, os_ in (([nl], [0]), ([-1], [0]), ([3, 5, 3], [0, 1, 1]), ([3], [2]), ([3], [-1])):
        assert lists(ls, os_) == LACK_OF_INPUTS, (ls, os_)
    assert [int(m.get_param("B200.PostingCacheLists")) for m in gr.members] == [1, 1]  # a refused call changes nothing
    assert lists([], []) == 0
    assert [int(m.get_param("B200.PostingCacheLists")) for m in gr.members] == [0, 0]

    # members whose search parameters differ: refused until they agree again
    for name, value in (("MaxDistRatio", "1.5"), ("SearchInternalResultNum", "32"), ("SearchPostingPageLimit", "1"),
                        ("MaxCheck", "1024")):
        back = m0.get_param(name)
        assert back != value, name
        m0.set_param(name, value)
        with pytest.raises(capi.SptagB200Error) as e:
            gr.search(q, 10)
        assert e.value.code == LACK_OF_INPUTS, name
        gr.set_param(name, back)
    with pytest.raises(capi.SptagB200Error):
        gr.set_param("B200.PostingCacheLists", 1)

    # destroying a member does nothing: the group owns it
    L.sptag_b200_spann_destroy(m0._h)
    ids, dists = gr.search(q, 10)
    assert np.array_equal(ids, g["ids_default_10"])
    assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32))
    assert gr.members[0].get_param("B200.PostingPlacement") == "host"
    assert int(gr.members[1].get_param("B200.PostingHostBytes")) == int(m0.get_param("B200.PostingHostBytes")) > 0


@pytest.mark.skipif(torch.cuda.device_count() < 2 or not torch.cuda.can_device_access_peer(0, 1),
                    reason="needs two devices with peer access")
def test_peers_on_different_devices(spann_group):
    g, files = _fixture(GOLDEN, "spann_l2_3k_16")
    folder = oracle_spann.SpannFolder(files)
    nl = len(folder.lists)
    gr = spann_group(files, devices=[0, 1])
    gr.cache_lists(range(nl), [1] * nl)
    assert int(gr.members[0].get_param("B200.PostingPeerLists")) == nl
    assert_group_search(gr, g, folder, "default", "default", {l: 1 for l in range(nl)})
    m0 = gr.members[0]
    assert int(m0.get_param("B200.LastPeerGatherBytes")) == int(m0.get_param("B200.LastGatherBytes")) > 0
