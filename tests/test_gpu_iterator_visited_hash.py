"""GPU tests of iterators on hashed visited sets (B200.IteratorVisitedSet = 1): each open iterator query owns a hash
table that grows, instead of a bitmap over the whole index.  A query that reaches its table's limit suspends, its table
grows (or becomes a bitmap) and the call resumes, so every call must return exactly what the bitmap iterators return:
ids, distance bits, result counts and relaxedMono, call by call.

Three modes run the checks: the bitmap, the hashed set at its default size, and the hashed set at 64 entries, where
nearly every query suspends, grows and, in a scan to exhaustion, converts to a bitmap.
"""
import os

import numpy as np
import pytest

import test_gpu_iterator as tgi
import test_gpu_parity as tgp
import test_gpu_visited_hash as tvh
import test_oracle_pin as pin
from conftest import data_folder
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

MODES = {"bitmap": {"B200.IteratorVisitedSet": 0},
         "hash": {"B200.IteratorVisitedSet": 1},
         "hash64": {"B200.IteratorVisitedSet": 1, "B200.IteratorVisitedHashEntries": 64}}
HASHED = ("hash", "hash64")
GOLDEN_BKT = ["algo_line_bkt", "bkt_cos_1500_20", "bkt_l2_2k_16", "bkt_l2_dups_1k_12"]


def set_mode(idx, mode):
    for k, v in MODES[mode].items():
        idx.set_param(k, v)


def suspensions(idx):
    step, trees = idx.get_param("B200.LastIteratorSuspensions").split(",")
    return int(step), int(trees)


def bitmap_bytes(n, nq):
    return nq * (((n + 1 + 31) // 32 + 3) // 4 * 4) * 4


def same(a, b, tag):
    """Two Next results (counts, ids, dists, relaxed) are identical."""
    assert np.array_equal(a[0], b[0]), tag
    assert np.array_equal(a[1], b[1]), tag
    assert np.array_equal(np.ascontiguousarray(a[2]).view(np.int32), np.ascontiguousarray(b[2]).view(np.int32)), tag
    assert np.array_equal(np.asarray(a[3], bool), np.asarray(b[3], bool)), tag


def queries_for(q, nq, seed=5):
    """nq queries from a fixture's queries: repeated, with a small perturbation after the first copy."""
    reps = -(-nq // q.shape[0])
    out = np.concatenate([q] * reps)[:nq].copy()
    rng = np.random.default_rng(seed)
    out[q.shape[0]:] += rng.standard_normal(out[q.shape[0]:].shape).astype(np.float32) * np.float32(0.01)
    return np.ascontiguousarray(out)


# ---- 1. the reference's own ResultIterator outputs -------------------------------------------------------------------
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", pin.iterator_golden_cases())
def test_golden_iterator_outputs(mode, name, monkeypatch):
    orig = B200Index.create

    def made(*args, **kwargs):
        idx = orig(*args, **kwargs)
        set_mode(idx, mode)
        return idx

    monkeypatch.setattr(B200Index, "create", made)
    pin.check_iterator_golden(name, tgi._DeviceIteratorBatch)


# ---- 2. hashed equals bitmap: batches, budgets, scans to exhaustion --------------------------------------------------
def _scan(make_index, q, mc, schedule, exhaust, sd=None):
    """Runs the schedule, or (exhaust) Next(1000) until every iterator is dry, in the three modes; returns per mode the
    suspension counts seen, the visited bytes after the last call and the growths of the last call.  (The first call
    sizes the result arena, so a scan to exhaustion starts on fresh iterators.)"""
    assert not (schedule and exhaust)
    seen = {}
    ref = None
    for mode in ("bitmap",) + HASHED:
        idx = make_index()
        try:
            set_mode(idx, mode)
            idx.set_param("MaxCheck", mc)
            its = idx.iterators(q, search_deleted=sd)
            got, susp = [], [0, 0]
            for b in schedule:
                got.append(its.next(b))
                s = suspensions(idx)
                susp = [susp[0] + s[0], susp[1] + s[1]]
            while exhaust:
                got.append(its.next(1000))
                s = suspensions(idx)
                susp = [susp[0] + s[0], susp[1] + s[1]]
                if ref is None and got[-1][0].sum() == 0:
                    break
                if ref is not None and len(got) == len(ref):
                    break
            seen[mode] = (susp, int(idx.get_param("B200.LastIteratorVisitedBytes")), int(idx.get_param("B200.LastIteratorGrowths")))
            its.close()
        finally:
            idx.close()
        if ref is None:
            ref = got
        else:
            assert len(got) == len(ref), mode
            for c, (a, b) in enumerate(zip(got, ref)):
                same(a, b, (mode, mc, c))
    return seen


def test_golden_sets_hashed_equals_bitmap():
    any_step = any_trees = False
    for name in GOLDEN_BKT:
        s, t = _golden_set_scans(name)
        any_step |= s
        any_trees |= t
    assert any_step and any_trees, "both resume paths ran"


def _golden_set_scans(name):
    g = np.load(os.path.join(tvh.GOLDEN, name + ".npz"))
    n = g["vectors"].shape[0]
    any_step = any_trees = False
    for nq in (1, 10, 1024):
        q = queries_for(np.ascontiguousarray(g["queries"]), nq)
        for mc in (16, 8192):
            seen = _scan(lambda: tvh.golden_index(name)[2], q, mc, [10, 10, 5, 7, 10], exhaust=False)
            assert seen["hash"][1] > 0
            any_step |= seen["hash64"][0][0] > 0
            any_trees |= seen["hash64"][0][1] > 0
            if nq <= 10:
                seen = _scan(lambda: tvh.golden_index(name)[2], q, mc, [], exhaust=True)
                any_step |= seen["hash64"][0][0] > 0
                any_trees |= seen["hash64"][0][1] > 0
            if nq == 1:
                # scanned dry: the table grew until it converted to a bitmap (or stopped below the bitmap's size), and
                # the buffers it left behind were freed
                assert seen["hash64"][1] <= bitmap_bytes(n, nq), (name, nq, mc, seen)
    return any_step, any_trees


@pytest.mark.parametrize("name", ["bkt_l2_20k_32", "bkt_cos_10k_128", "bkt_l2_3k_30", "bkt_l2_dups", "bkt2_l2_6k_32"])
def test_reference_built_sets_hashed_equals_bitmap(name):
    folder = data_folder(name)
    q0 = np.load(os.path.join(folder, "queries.npy"))
    for nq in (10, 1024):
        q = queries_for(np.ascontiguousarray(q0[:64]), nq)
        for mc in (16, 8192):
            _scan(lambda: B200Index.load(folder), q, mc, [10, 10, 5, 7, 10, 3, 10, 1, 4], exhaust=False)
    _scan(lambda: B200Index.load(folder), np.ascontiguousarray(q0[:4]), 256, [], exhaust=True)


# ---- 3. SearchIndexIterativeFromNeareast, then more calls ------------------------------------------------------------
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt_cos_1500_20", "bkt_l2_dups_1k_12"])
def test_nearest_first_hashed_equals_bitmap(name):
    g = np.load(os.path.join(tvh.GOLDEN, name + ".npz"))
    q = queries_for(np.ascontiguousarray(g["queries"]), 40)
    for k in (1, 10, 1024):
        ref = None
        for mode in ("bitmap",) + HASHED:
            idx = tvh.golden_index(name)[2]
            try:
                set_mode(idx, mode)
                idx.set_param("MaxCheck", 8192)
                its = idx.iterators(q)
                got = [its.next_from_nearest(k)]
                growths_first = int(idx.get_param("B200.LastIteratorGrowths"))
                got += [its.next_from_nearest(k) for _ in range(3)]
                its.close()
            finally:
                idx.close()
            if mode == "hash64" and k == 1:
                # the first search filled its table and ran again on a larger one (at larger k the tables are sized for
                # the k x (degree + 1) seeds, which leaves room for the whole search on these small sets)
                assert growths_first > 0
            if ref is None:
                ref = got
                continue
            for c, (a, b) in enumerate(zip(got, ref)):
                assert np.array_equal(a[0], b[0]), (mode, k, c)
                assert np.array_equal(a[1], b[1]), (mode, k, c)
                assert np.array_equal(a[2].view(np.int32), b[2].view(np.int32)), (mode, k, c)


# ---- 4. tombstones ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["bkt_l2_2k_16", "bkt_l2_dups_1k_12"])
def test_tombstones_hashed_equals_bitmap(name):
    g = np.load(os.path.join(tvh.GOLDEN, name + ".npz"))
    n = g["vectors"].shape[0]
    dead = np.nonzero(np.random.default_rng(11).random(n) < 0.3)[0].astype(np.int32)

    def make():
        idx = tvh.golden_index(name)[2]
        idx.delete(dead)
        return idx

    q = queries_for(np.ascontiguousarray(g["queries"]), 10)
    for sd in (False, True):
        for mc in (16, 8192):
            _scan(make, q, mc, [10, 10, 5, 7, 10], exhaust=False, sd=sd)
            _scan(make, q, mc, [], exhaust=True, sd=sd)


# ---- 5. auto: the hashed set when the bitmaps do not fit -------------------------------------------------------------
def test_auto_falls_back_to_hashed_iterators_when_the_bitmaps_do_not_fit():
    """8M vectors: 1 MB of bitmap per iterator query, 2 GB for 2048 queries.  With less than that left free, auto opens
    the batch on hash tables; its calls equal those of bitmap iterators opened in batches of 256."""
    import torch
    n, nq = 8000000, 2048
    idx, x = tvh._random_graph_index(n, 8, 3)
    q = np.ascontiguousarray(x[:: n // nq][:nq] + np.float32(0.01))
    schedule = [10, 10, 25]
    hold = None
    try:
        idx.set_param("B200.IteratorVisitedSet", 0)
        want = [[] for _ in schedule]
        for s in range(0, nq, 256):
            its = idx.iterators(q[s:s + 256])
            for c, b in enumerate(schedule):
                want[c].append(its.next(b))
            its.close()
        want = [tuple(np.concatenate([w[i] for w in ws]) for i in range(4)) for ws in want]
        idx.set_param("B200.IteratorVisitedSet", -1)
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        hold = torch.empty(free - (768 << 20), dtype=torch.uint8, device="cuda")  # room for the tables, not the bitmaps
        its = idx.iterators(q)
        for c, b in enumerate(schedule):
            same(its.next(b), want[c], c)
            assert int(idx.get_param("B200.LastIteratorVisitedBytes")) < bitmap_bytes(n, nq) // 8
        its.close()
    finally:
        del hold
        torch.cuda.empty_cache()
        idx.close()


# ---- 6. hashed iterator memory does not grow with the index ----------------------------------------------------------
def test_hashed_iterator_memory_does_not_grow_with_the_index():
    q = None
    held = []
    for n in (5000, 80000):
        idx, x = tvh._flat_index(n, 1)
        try:
            if q is None:
                q = np.ascontiguousarray(x[:16])
            idx.set_param("B200.IteratorVisitedSet", 1)
            its = idx.iterators(q)
            its.next(10)
            held.append(int(idx.get_param("B200.LastIteratorVisitedBytes")))
            its.close()
        finally:
            idx.close()
    assert held[0] == held[1] > 0


# ---- 7. parameters ---------------------------------------------------------------------------------------------------
def test_iterator_parameter_checks():
    g, files, idx = tvh.golden_index("algo_line_bkt")
    try:
        assert idx.get_param("B200.IteratorVisitedSet") == "-1"
        assert idx.get_param("B200.IteratorVisitedHashEntries") == "0"
        for name, bad in (("B200.IteratorVisitedSet", 2), ("B200.IteratorVisitedSet", -2),
                          ("B200.IteratorVisitedHashEntries", 100), ("B200.IteratorVisitedHashEntries", 32),
                          ("B200.IteratorVisitedHashEntries", 1 << 31)):
            with pytest.raises(capi.SptagB200Error):
                idx.set_param(name, bad)
        idx.set_param("B200.IteratorVisitedHashEntries", 4096)
        assert idx.get_param("B200.IteratorVisitedHashEntries") == "4096"
        for name in ("B200.LastIteratorSuspensions", "B200.LastIteratorGrowths", "B200.LastIteratorVisitedBytes"):
            idx.get_param(name)
            with pytest.raises(capi.SptagB200Error):
                idx.set_param(name, 1)  # read-only
        # an open iterator keeps the mode it was opened with; the search's B200.VisitedSet is not involved
        idx.set_param("B200.IteratorVisitedSet", 1)
        its = idx.iterators(np.zeros((2, 10), np.float32))
        idx.set_param("B200.IteratorVisitedSet", 0)
        its.next(5)
        assert int(idx.get_param("B200.LastIteratorVisitedBytes")) == 2 * 4096 * 4
        assert idx.get_param("B200.VisitedSet") == "-1"
        its.close()
    finally:
        idx.close()
