"""The plain-Python SPANN restatements (tests/oracle_spann.py, tests/oracle_spann_iterator.py) against the unmodified
reference on uint8, int16 and integer-cosine rows whose size is not a multiple of 16 bytes (tests/golden/spann_elem and
spann_elem_iter, written by tests/golden/make_golden_spann_elem.py): SearchIndex's ids and distance bits for every case,
parameter set and K, and every GetIterator + Next call.  Also what the fixtures must keep covering.  CPU only."""
import os

import numpy as np
import pytest

import oracle_spann
from golden.make_golden_spann import KS, PARAMS
from golden.make_golden_spann_iterator import PARAMS as ITER_PARAMS
from golden.make_golden_spann_iterator import applies, schedule_queries
from test_oracle_pin_spann_iterator import assert_calls_equal, expected, restate

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_elem")
GOLDEN_ITER = os.path.join(HERE, "golden", "spann_elem_iter")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
ITER_CASES = sorted(f[:-4] for f in os.listdir(GOLDEN_ITER) if f.endswith(".npz"))
# (value type, metric) of the posting kernels that no tests/golden/spann fixture runs
NEW_PAIRS = {("UInt8", "L2"), ("UInt8", "Cosine"), ("Int8", "Cosine"), ("Int16", "L2"), ("Int16", "Cosine")}


def _fixture(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    return g, oracle_spann.fixture_files(g)


def _pair(files):
    base = oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())["Base"]
    return base["ValueType"], base["DistCalcMethod"]


def _truncated_rearranged(folder):
    return folder.rearranged and any(folder.searched(l) < folder.lists[l][0] for l in range(len(folder.lists)))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_restatement_equals_reference(case, pname):
    g, files = _fixture(case)
    assert int(g["ref_isa"]) == 16  # the AVX-512 int16 rounding tree, the one the oracle and the device restate
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    if _truncated_rearranged(folder):
        pytest.skip("truncated lists of the rearranged layout: the device refuses them (tests/test_gpu_spann_elem.py)")
    q = g["queries"]
    for k in KS:
        ids, dists, _ = oracle_spann.search(folder, q, g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)], k)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (case, pname, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (case, pname, k)


@pytest.mark.parametrize("case", ITER_CASES)
@pytest.mark.parametrize("pname", sorted(ITER_PARAMS))
@pytest.mark.parametrize("sname", ["short", "scan"])
def test_iterator_restatement_equals_reference(case, pname, sname):
    if not applies(case, pname):
        pytest.skip("truncated lists of the rearranged layout: the device refuses them")
    g = np.load(os.path.join(GOLDEN_ITER, case + ".npz"))
    src, files = _fixture(case)
    q = schedule_queries(src["queries"], sname)
    sched, want = expected(g, "%s_%s" % (pname, sname), len(q))
    assert_calls_equal(restate(files, ITER_PARAMS[pname], q, sched), want, (case, pname, sname))


def test_fixtures_cover_types_padding_layouts_pruning_truncation_and_int16_range():
    """Every (type, metric) pair the older SPANN fixtures miss, each with padded rows; both layouts; MaxDistRatio 1.5
    dropping postings and the page limit truncating a plain list; int16 L2 differences whose squares pass 2^24 (where
    float sums of squares start to round).  Deleting a case fails this."""
    assert CASES == ITER_CASES
    pairs, layouts = set(), set()
    pruned = truncated = wide = False
    for case in CASES:
        g, files = _fixture(case)
        pairs.add(_pair(files))
        f0 = oracle_spann.SpannFolder(files)
        assert f0.row_bytes % 16 != 0, (case, f0.row_bytes)
        layouts.add(f0.rearranged)
        fp = oracle_spann.SpannFolder(files, PARAMS["pages"])
        truncated |= not f0.rearranged and any(fp.searched(l) < f0.searched(l) for l in range(len(f0.lists)))
        fr = oracle_spann.SpannFolder(files, PARAMS["ratio"])
        k = 10
        a = oracle_spann.search(f0, g["queries"], g["head_ids_default_%d" % k], g["head_dists_default_%d" % k], k)[2]
        b = oracle_spann.search(fr, g["queries"], g["head_ids_ratio_%d" % k], g["head_dists_ratio_%d" % k], k)[2]
        pruned |= bool((b[:, 0] < a[:, 0]).any())
        if _pair(files) == ("Int16", "L2"):
            rows = np.stack([np.frombuffer(f0.element(l, i, f0.lists[l][0])[1], np.int16)
                             for l in range(len(f0.lists)) for i in range(f0.lists[l][0])]).astype(np.int64)
            q = g["queries"].astype(np.int64)
            wide = bool((((q[:, None, :] - rows[None, :, :]) ** 2) > 2**24).any())
    assert NEW_PAIRS <= pairs, NEW_PAIRS - pairs
    assert layouts == {False, True}
    assert pruned and truncated and wide, (pruned, truncated, wide)
