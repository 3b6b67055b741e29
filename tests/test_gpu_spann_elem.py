"""SPANN search and SPANN iterators on uint8, int16 and integer-cosine rows whose size is not a multiple of 16 bytes, with
the posting lists in HBM and in pinned host memory (the default stage and B200.PostingStageBytes 0), against the unmodified
reference's results recorded in tests/golden/spann_elem and spann_elem_iter: ids and distance bits of every case, parameter
set and K, the counters against the plain-Python restatement (tests/oracle_spann.py), the gathered bytes and rounds, and
every GetIterator + Next call.  On int8 and uint8 rows every returned posting element's distance is also checked against
its exact integer value, computed here from the posting file's row, so that a misread stride, padded row or id fails even
where the oracle shares the mistake.  Each case asserts which posting-kernel instantiation ran (B200.LastPostingKernel),
and the file as a whole runs all 8 posting-scan and all 8 posting-step instantiations."""
import os
import sys

import numpy as np
import pytest

import oracle_spann
from golden.make_golden_spann import KS, PARAMS, write_folder
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from sptag_b200 import capi
from test_gpu_spann_host import DEFAULT_STAGE, _assert_gathered
from test_oracle_pin_spann_iterator import assert_calls_equal, expected

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_elem")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_elem_iter")
GOLDEN_OLD = os.path.join(HERE, "golden", "spann")
GOLDEN_OLD_ITER = os.path.join(HERE, "golden", "spann_iter")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
ITER_CASES = sorted(f[:-4] for f in os.listdir(GOLDEN_ITER) if f.endswith(".npz"))
# the (metric, type) pairs tests/golden/spann already covers: float L2, float cosine, int8 L2
OLD_CASES = ("spann_l2_3k_16", "spann_cos_rearr_2k_24", "spann_i8_l2_2k_16")
LACK_OF_INPUTS = 0x13
ELEM = {"Float": 0, "Int8": 1, "UInt8": 2, "Int16": 3}
BASE = {"Int8": 127, "UInt8": 255}  # Utils::GetBase: cosine distance = base^2 - dot on these types
# placement -> (posting_placement, B200.PostingStageBytes)
PLACEMENTS = {"device": ("device", None), "host": ("host", DEFAULT_STAGE), "host_stage0": ("host", 0)}
ALL_KERNELS = {"sptag_b200::(anonymous namespace)::spann_%s_kernel<%s, %d>" % (kind, cos, e)
               for kind in ("scan", "iter_step") for cos in ("false", "true") for e in range(4)}
_RAN = {}  # kernel name -> the tests that named it


@pytest.fixture
def spann(tmp_path):
    """load(files, values, placement) of a fixture's folder; every handle is closed after the test"""
    opened = []

    def load(files, values, placement):
        kind, stage = PLACEMENTS[placement]
        folder = str(tmp_path / ("index%d" % len(opened)))
        write_folder(files, folder, values)
        s = capi.B200SpannIndex.load(folder, 0, posting_placement=kind)
        opened.append(s)
        if stage is not None:
            s.set_param("B200.PostingStageBytes", stage)
        return s

    yield load
    for s in opened:
        s.close()


def _base(files):
    return oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())["Base"]


def predicted(kind, files):
    base = _base(files)
    return "sptag_b200::(anonymous namespace)::spann_%s_kernel<%s, %d>" % (
        kind, "true" if base["DistCalcMethod"] == "Cosine" else "false", ELEM[base["ValueType"]])


def _assert_kernel(s, kind, files, request):
    name = s.get_param("B200.LastPostingKernel")
    assert name == predicted(kind, files), name
    _RAN.setdefault(name, []).append(request.node.name)


def _refused_truncation(folder):
    return folder.rearranged and any(folder.searched(l) < folder.lists[l][0] for l in range(len(folder.lists)))


_ROWS = {}


def posting_rows(case, folder):
    """{id: row as int64} of every element of every list (all of a list, whatever the page limit)"""
    if case not in _ROWS:
        rows = {}
        for l, (cnt, _, _, _) in enumerate(folder.lists):
            for i in range(cnt):
                vid, row = folder.element(l, i, cnt)
                rows[vid] = np.frombuffer(row, folder.dtype).astype(np.int64)
        _ROWS[case] = rows
    return _ROWS[case]


def assert_exact_distances(case, files, q, ids, dists):
    """int8 / uint8: a returned posting element's distance is its exact integer L2 or base^2 - dot (both below 2^24 at
    these dimensions, so the float holds them exactly), from the row in the posting file and the query"""
    vt = _base(files)["ValueType"]
    if vt not in BASE:
        return 0
    folder = oracle_spann.SpannFolder(files)
    rows = posting_rows(case, folder)
    q = np.asarray(q).astype(np.int64)
    checked = 0
    for i in range(len(q)):
        for vid, d in zip(ids[i].tolist(), dists[i].tolist()):
            if vid < 0 or vid not in rows:
                continue
            r = rows[vid]
            exact = int(((q[i] - r) ** 2).sum()) if folder.metric == 0 else BASE[vt] ** 2 - int((q[i] * r).sum())
            assert abs(exact) < 2**24
            assert np.float32(d) == np.float32(exact), (case, i, vid, d, exact)
            checked += 1
    return checked


_STATS = {}


def oracle_stats(case, folder, pname, k, g):
    key = (case, pname, k)
    if key not in _STATS:
        hid, hd = g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)]
        _STATS[key] = oracle_spann.search(folder, g["queries"], hid, hd, k)[2]
    return _STATS[key]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("placement", sorted(PLACEMENTS))
def test_search_equals_reference(case, pname, placement, spann, request):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(g)
    s = spann(files, PARAMS[pname], placement)
    q = g["queries"]
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _refused_truncation(folder):
        with pytest.raises(capi.SptagB200Error) as e:
            s.search(q, 10)
        assert e.value.code == LACK_OF_INPUTS
        return
    stage = PLACEMENTS[placement][1]
    checked = 0
    for k in KS:
        ids, dists, stats = s.search(q, k, want_stats=True)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (case, pname, placement, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (case, pname, placement, k)
        assert np.array_equal(stats, oracle_stats(case, folder, pname, k, g)), (case, pname, placement, k)
        if stage is not None:
            _assert_gathered(s, folder, g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)], stage)
        checked += assert_exact_distances(case, files, q, ids, dists)
    assert checked > 0 or _base(files)["ValueType"] not in BASE
    _assert_kernel(s, "scan", files, request)


@pytest.mark.parametrize("case", ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
@pytest.mark.parametrize("placement", ["device", "host"])
def test_iterators_equal_reference(case, pname, sname, placement, spann, request):
    g = np.load(os.path.join(GOLDEN_ITER, case + ".npz"))
    src = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(src)
    q = schedule_queries(src["queries"], sname)
    refused = _refused_truncation(oracle_spann.SpannFolder(files, ITER_PARAMS[pname]))
    if not applies(case, pname) and not refused:
        pytest.skip("no recorded calls (the pages set is not run on the rearranged layout), and no list is truncated")
    s = spann(files, ITER_PARAMS[pname], placement)
    it = s.iterators(q)
    try:
        if refused:
            with pytest.raises(capi.SptagB200Error) as e:
                it.next(10)
            assert e.value.code == LACK_OF_INPUTS
            return
        sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
        got = [it.next(int(b)) for b in sched]
    finally:
        it.close()
    assert_calls_equal(got, want, (case, pname, sname, placement))
    for counts, ids, dists, _ in got:
        assert_exact_distances(case, files, q, ids, dists)
    _assert_kernel(s, "iter_step", files, request)


@pytest.mark.parametrize("case", OLD_CASES)
def test_older_fixtures_name_their_kernels(case, spann, request):
    """One search and one iterator schedule on each (metric, type) pair the older fixtures cover, so that this file runs
    every posting-kernel instantiation"""
    g = np.load(os.path.join(GOLDEN_OLD, case + ".npz"))
    files = oracle_spann.fixture_files(g)
    s = spann(files, {}, "device")
    ids, dists = s.search(g["queries"], 10)
    assert np.array_equal(ids, g["ids_default_10"])
    assert np.array_equal(dists.view(np.int32), g["dists_default_10"].view(np.int32))
    _assert_kernel(s, "scan", files, request)
    gi = np.load(os.path.join(GOLDEN_OLD_ITER, case + ".npz"))
    q = schedule_queries(g["queries"], "short")
    sched, want = expected(gi, "default_short", len(q))
    it = s.iterators(q)
    try:
        got = [it.next(int(b)) for b in sched]
    finally:
        it.close()
    assert_calls_equal(got, want, case)
    _assert_kernel(s, "iter_step", files, request)


def test_every_posting_kernel_is_named(request):
    """The case matrix predicts all 16 instantiations (a deleted case names the one that lost it); where this file ran in
    full, each of them was launched and named by some case"""
    want = set()
    for golden, cases in ((GOLDEN, CASES), (GOLDEN_OLD, OLD_CASES)):
        for case in cases:
            files = oracle_spann.fixture_files(np.load(os.path.join(golden, case + ".npz")))
            want |= {predicted("scan", files), predicted("iter_step", files)}
    assert want == ALL_KERNELS, sorted(ALL_KERNELS - want)
    mine = [i for i in request.session.items if i.module is sys.modules[__name__] and i is not request.node]
    full = len(mine) == len(CASES) * len(PARAMS) * len(PLACEMENTS) + len(ITER_CASES) * len(ITER_PARAMS) * 4 + len(OLD_CASES)
    if not full:
        pytest.skip("only part of this file ran")
    for name in sorted(_RAN):
        print("%s: %d cases, e.g. %s" % (name, len(_RAN[name]), _RAN[name][0]))
    assert set(_RAN) == ALL_KERNELS, sorted(ALL_KERNELS - set(_RAN))
