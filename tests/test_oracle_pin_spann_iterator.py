"""The plain-Python SPANN iterator restatement (tests/oracle_spann_iterator.py) against the unmodified reference's
GetIterator + Next on every fixture of tests/golden/spann_iter: counts, ids, distance bits and RelaxedMono of every call.
CPU only."""
import os

import numpy as np
import pytest

import oracle_spann
import oracle_spann_iterator
from golden.make_golden_spann_iterator import PARAMS, SHORT, applies, schedule_queries

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_iter")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def _load(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    src = np.load(os.path.join(HERE, "golden", "spann", case + ".npz"))
    return g, src, oracle_spann.fixture_files(src)


def restate(files, values, queries, sched, cov=None):
    """SpannIterator per query over the schedule -> per call (counts [nq], ids [nq, b], dists [nq, b], relaxed [nq])"""
    folder = oracle_spann.SpannFolder(files, values)
    ssd = oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())["BuildSSDIndex"]
    hb = int(values.get("IterativeSearchHeadBatch", ssd.get("IterativeSearchHeadBatch", "32")))
    head = oracle_spann_iterator.head_oracle(files)
    its = [oracle_spann_iterator.SpannIterator(folder, head, q, hb) for q in queries]
    calls = []
    for b in sched:
        out = [it.next(int(b)) for it in its]
        calls.append((np.array([o[0] for o in out], np.int32), np.stack([o[1] for o in out]),
                      np.stack([o[2] for o in out]), np.array([o[3] for o in out], bool)))
    for it in its:
        if cov is not None:
            for k, v in it.cov.items():
                cov[k] = cov.get(k, 0) + v
        it.close()
    return calls


def expected(g, key, nq):
    """The fixture's calls for parameter set + schedule `key`, in restate's layout"""
    sched = g["sched_" + key]
    ids, dists = g["ids_" + key], g["dists_" + key]
    out, at = [], 0
    for c, b in enumerate(sched):
        n = nq * int(b)
        out.append((g["counts_" + key][c], ids[at:at + n].reshape(nq, b), dists[at:at + n].reshape(nq, b),
                    g["relaxed_" + key][c].astype(bool)))
        at += n
    return sched, out


def assert_calls_equal(got, want, what):
    assert len(got) == len(want), what
    for c, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a[0], b[0]), (what, c, "counts")
        assert np.array_equal(a[1], b[1]), (what, c, "ids")
        assert np.array_equal(a[2].view(np.int32), b[2].view(np.int32)), (what, c, "dists")
        assert np.array_equal(a[3], b[3]), (what, c, "relaxed")


_COV = {}


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
def test_restatement_equals_reference(case, pname, sname):
    if not applies(case, pname):
        pytest.skip("truncated lists of the rearranged layout: the device refuses them")
    g, src, files = _load(case)
    q = schedule_queries(src["queries"], sname)
    sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
    cov = _COV.setdefault((case, pname, sname), {})
    cov.clear()
    got = restate(files, PARAMS[pname], q, sched, cov)
    assert_calls_equal(got, want, (case, pname, sname))


def test_fixtures_cover_the_iterator_paths():
    """Across the fixtures: the last-element quirk, a refill inside a call, a deduper skip of an id loaded in an earlier
    head batch, RelaxedMono turning on, head exhaustion (a call with fewer than batch, then 0) and a truncated list."""
    cov = {}
    for case in CASES:
        g, src, files = _load(case)
        for pname in PARAMS:
            if not applies(case, pname):
                continue
            key = (case, pname, "short")
            if key not in _COV:  # the restatement test did not run first
                _COV[key] = {}
                restate(files, PARAMS[pname], src["queries"], SHORT, _COV[key])
            for k, v in _COV[key].items():
                cov[k] = cov.get(k, 0) + v
            for sname in ("short", "scan"):
                nm = "%s_%s" % (pname, sname)
                cov["relaxed"] = cov.get("relaxed", 0) + int(g["relaxed_" + nm].sum())
                counts, sched = g["counts_" + nm], g["sched_" + nm]
                for c in range(1, len(sched)):
                    cov["exhausted"] = cov.get("exhausted", 0) + int(
                        ((counts[c - 1] > 0) & (counts[c - 1] < sched[c - 1]) & (counts[c] == 0)).sum())
    for k in ("quirk", "refill_mid_call", "dedup_across_batches", "truncated", "relaxed", "exhausted"):
        assert cov.get(k, 0) > 0, (k, cov)
