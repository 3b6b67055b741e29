"""SPANN iterators with the posting lists in HBM (sptag_b200_spann_iterator_*) against the unmodified reference's
GetIterator + Next, recorded in tests/golden/spann_iter: counts, ids, distance bits and RelaxedMono of every call for every
case, parameter set and schedule.  Also: head batches 1 and 1024, a growing batch request, SearchInternalResultNum changed
between calls (against the plain-Python restatement, tests/oracle_spann_iterator.py), forced dedup table growth, hashed head
visited sets, 1 and 1 000 iterators, searches and other iterators between calls, two threads, the refusals, and (where
its driver was built) the reference itself on the folder the device loaded."""
import ctypes
import os
import subprocess
import threading

import numpy as np
import pytest

import oracle_spann
import oracle_spann_iterator
from golden.make_golden_spann import write_folder
from golden.make_golden_spann_iterator import PARAMS, SHORT, applies, schedule_queries
from sptag_b200 import capi
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_iter")
REF_DRIVER = os.path.join(HERE, "cpp", "spann_iter_ref")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
LACK_OF_INPUTS = 0x13


def _fixture(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    src = np.load(os.path.join(HERE, "golden", "spann", case + ".npz"))
    return g, src["queries"], oracle_spann.fixture_files(src)


def _load(files, tmp_path, values=None, **params):
    write_folder(files, str(tmp_path), values or {})
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    for k, v in params.items():
        s.set_param(k.replace("__", "."), v)
    return s


def run(s, queries, sched):
    it = s.iterators(queries)
    try:
        return [it.next(int(b)) for b in sched]
    finally:
        it.close()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
def test_iterators_equal_reference(case, pname, sname, tmp_path):
    g, q, files = _fixture(case)
    s = _load(files, tmp_path, PARAMS[pname])
    try:
        q = schedule_queries(q, sname)
        if not applies(case, pname):
            it = s.iterators(q)
            with pytest.raises(capi.SptagB200Error) as e:
                it.next(10)
            assert e.value.code == LACK_OF_INPUTS
            it.close()
            return
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        assert_calls_equal(run(s, q, sched), want, (case, pname, sname))
        assert int(s.get_param("B200.LastIteratorDedupBytes")) > 0
    finally:
        s.close()


def _restate(files, values, queries, sched, hb, internal_at=None):
    """SpannIterator per query; internal_at: {call index: SearchInternalResultNum set before that call}"""
    folder = oracle_spann.SpannFolder(files, values)
    head = oracle_spann_iterator.head_oracle(files)
    its = [oracle_spann_iterator.SpannIterator(folder, head, qq, hb) for qq in queries]
    out = []
    for c, b in enumerate(sched):
        if internal_at and c in internal_at:
            folder.internal = internal_at[c]
        r = [it.next(b) for it in its]
        out.append((np.array([x[0] for x in r], np.int32), np.stack([x[1] for x in r]), np.stack([x[2] for x in r]),
                    np.array([x[3] for x in r], bool)))
    for it in its:
        it.close()
    return out


@pytest.mark.parametrize("hb,internal", [(1, 64), (1024, 1024)])
def test_head_batch_extremes_and_a_growing_batch(hb, internal, tmp_path):
    """Head batches 1 and 1024; Next(8) then Next(40): the second call is capped by the first's result count."""
    _, q, files = _fixture("spann_l2_3k_16")
    q = q[:8]
    sched = (8, 40, 5, 30)
    s = _load(files, tmp_path, {"SearchInternalResultNum": str(internal)}, IterativeSearchHeadBatch=hb)
    try:
        got = run(s, q, sched)
        if hb == 1:
            assert int(s.get_param("B200.LastIteratorRounds")) > 0
    finally:
        s.close()
    assert_calls_equal(got, _restate(files, {"SearchInternalResultNum": str(internal)}, q, sched, hb), hb)


def test_internal_result_num_changed_between_calls(tmp_path):
    _, q, files = _fixture("spann_i8_l2_2k_16")
    q = q[:8]
    sched = (300, 300, 300, 300)  # a call loads several head batches: RelaxedMono turns on once the limit is 8
    s = _load(files, tmp_path, {"IterativeSearchHeadBatch": "8"})
    try:
        it = s.iterators(q)
        got = []
        for c, b in enumerate(sched):
            if c == 1:
                s.set_param("SearchInternalResultNum", 8)
            if c == 3:
                s.set_param("SearchInternalResultNum", 64)
            got.append(it.next(b))
        it.close()
    finally:
        s.close()
    want = _restate(files, {"IterativeSearchHeadBatch": "8"}, q, sched, 8, {1: 8, 3: 64})
    assert not want[0][3].any() and want[1][3].any()
    assert_calls_equal(got, want, "internal")


@pytest.mark.parametrize("params", [{"B200__SpannDedupEntries": 64},
                                    {"B200__IteratorVisitedSet": 1, "B200__IteratorVisitedHashEntries": 64}],
                         ids=["dedup_growth", "hashed_head"])
@pytest.mark.parametrize("case", ["spann_l2_3k_16", "spann_cos_rearr_2k_24"])
def test_small_tables_give_identical_results(case, params, tmp_path):
    g, q, files = _fixture(case)
    s = _load(files, tmp_path, **params)
    try:
        for sname in ("short", "scan"):
            qq = schedule_queries(q, sname)
            sched, want = expected(g, "default_" + sname, len(qq))
            assert_calls_equal(run(s, qq, sched), want, (case, params, sname))
            if "B200__SpannDedupEntries" in params:  # the tables grew past their first 64 entries
                assert int(s.get_param("B200.LastIteratorDedupBytes")) > len(qq) * 64 * 4
    finally:
        s.close()


@pytest.mark.parametrize("nq", [1, 1000])
def test_one_and_a_thousand_iterators(nq, tmp_path):
    g, q, files = _fixture("spann_l2_heads_2k_16")
    sched, want = expected(g, "default_short", len(q))
    rows = np.arange(nq) % len(q)
    s = _load(files, tmp_path)
    try:
        got = run(s, q[rows], sched)
    finally:
        s.close()
    assert_calls_equal(got, [tuple(x[rows] for x in w) for w in want], nq)


def test_searches_and_other_iterators_between_calls(tmp_path):
    g, q, files = _fixture("spann_l2_3k_16")
    sched, want = expected(g, "hb4_short", len(q))
    s = _load(files, tmp_path, {"IterativeSearchHeadBatch": "4"})
    try:
        a, b = s.iterators(q), s.iterators(q)
        got_a, got_b = [], []
        for bt in sched:
            got_a.append(a.next(int(bt)))
            s.search(q, 10)
            got_b.append(b.next(int(bt)))
            s.search(q[:5], 100)
        a.close()
        b.close()
    finally:
        s.close()
    assert_calls_equal(got_a, want, "a")
    assert_calls_equal(got_b, want, "b")


def test_two_threads_each_with_an_iterator(tmp_path):
    g, q, files = _fixture("spann_i8_l2_2k_16")
    sched, w = expected(g, "default_short", len(q))  # NpzFile: read in one thread
    s = _load(files, tmp_path)
    errors = []

    def work():
        try:
            for _ in range(3):
                assert_calls_equal(run(s, q, sched), w, "thread")
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=work) for _ in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    s.close()
    assert not errors, errors


def test_refusals(tmp_path):
    _, q, files = _fixture("spann_l2_3k_16")
    s = _load(files, tmp_path)
    L = capi.lib()
    try:
        it = s.iterators(q[:2])
        for batch in (0, 1025):
            with pytest.raises(capi.SptagB200Error) as e:
                it.next(batch)
            assert e.value.code == LACK_OF_INPUTS
        ids = np.empty((2, 4), np.int32)
        dists = np.empty((2, 4), np.float32)
        assert L.sptag_b200_spann_iterator_next(it._it, 4, None, dists.ctypes.data, None, None) == LACK_OF_INPUTS
        assert L.sptag_b200_spann_iterator_next(None, 4, ids.ctypes.data, dists.ctypes.data, None, None) != 0
        it.close()
        out = ctypes.c_void_p()
        assert L.sptag_b200_spann_iterator_open(s._h, None, 2, ctypes.byref(out)) == LACK_OF_INPUTS
        for name, value in (("IterativeSearchHeadBatch", 0), ("IterativeSearchHeadBatch", 1025),
                            ("B200.SpannDedupEntries", 100), ("B200.SpannDedupEntries", 32),
                            ("B200.LastIteratorRounds", 1), ("B200.LastIteratorDedupBytes", 1)):
            with pytest.raises(capi.SptagB200Error) as e:
                s.set_param(name, value)
            assert e.value.code == LACK_OF_INPUTS, name
        # a head batch above SearchInternalResultNum: the reference's page buffers would overflow
        s.set_param("SearchInternalResultNum", 16)
        it = s.iterators(q[:2])
        with pytest.raises(capi.SptagB200Error) as e:
            it.next(10)
        assert e.value.code == LACK_OF_INPUTS
        it.close()
        assert s.get_param("IterativeSearchHeadBatch") == "32"
    finally:
        s.close()


@pytest.mark.parametrize("case", CASES)
def test_reference_on_the_same_folder(case, tmp_path):
    """Where the reference driver was built, the reference itself iterates the folder the device loaded."""
    if not os.path.exists(REF_DRIVER):
        pytest.skip("tests/cpp/spann_iter_ref is built only where oracle/_ref exists")
    _, q, files = _fixture(case)
    folder = str(tmp_path / "index")
    s = _load(files, folder)
    try:
        qf, pre = str(tmp_path / "q.bin"), str(tmp_path / "r")
        q.tofile(qf)
        subprocess.check_call([REF_DRIVER, folder, qf, str(len(q)), pre, ",".join(map(str, SHORT))])
        counts = np.fromfile(pre + ".counts", np.int32).reshape(len(SHORT), len(q))
        relaxed = np.fromfile(pre + ".relaxed", np.uint8).reshape(len(SHORT), len(q))
        ids, dists = np.fromfile(pre + ".ids", np.int32), np.fromfile(pre + ".dists", np.float32)
        want, at = [], 0
        for c, b in enumerate(SHORT):
            n = len(q) * b
            want.append((counts[c], ids[at:at + n].reshape(len(q), b), dists[at:at + n].reshape(len(q), b),
                         relaxed[c].astype(bool)))
            at += n
        assert_calls_equal(run(s, q, SHORT), want, case)
    finally:
        s.close()
