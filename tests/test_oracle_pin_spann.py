"""The plain-Python SPANN restatement (tests/oracle_spann.py) against the unmodified reference's SPANN::Index::SearchIndex
on every fixture of tests/golden/spann, every K and every parameter set.  CPU only."""
import os

import numpy as np
import pytest

import oracle_spann
from golden.make_golden_spann import KS, PARAMS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spann")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_restatement_equals_reference(case, pname):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    folder = oracle_spann.SpannFolder(oracle_spann.fixture_files(g), PARAMS[pname])
    if folder.rearranged and any(folder.searched(l) < folder.lists[l][0] for l in range(len(folder.lists))):
        pytest.skip("truncated lists of the rearranged layout: the device refuses them (tests/test_gpu_spann.py)")
    q = g["queries"]
    for k in KS:
        ids, dists, _ = oracle_spann.search(folder, q, g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)], k)
        assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (case, pname, k)
        assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (case, pname, k)


def test_fixtures_cover_pruning_truncation_and_head_ids():
    """The parameter sets change what is read: MaxDistRatio drops postings, the page limit truncates plain lists.  Some
    reference result holds one id twice (a head result and the same vector in a posting list: the deduper is not seeded
    with the head results), and some head result is translated to (-1, MaxDist)."""
    pruned = truncated = repeated = no_vector = False
    for case in CASES:
        g = np.load(os.path.join(GOLDEN, case + ".npz"))
        files = oracle_spann.fixture_files(g)
        f0 = oracle_spann.SpannFolder(files)
        fp = oracle_spann.SpannFolder(files, PARAMS["pages"])
        truncated |= not f0.rearranged and any(fp.searched(l) < f0.searched(l) for l in range(len(f0.lists)))
        for k in KS:
            a = oracle_spann.search(f0, g["queries"], g["head_ids_default_%d" % k], g["head_dists_default_%d" % k], k)[2]
            fr = oracle_spann.SpannFolder(files, PARAMS["ratio"])
            b = oracle_spann.search(fr, g["queries"], g["head_ids_ratio_%d" % k], g["head_dists_ratio_%d" % k], k)[2]
            pruned |= bool((b[:, 0] < a[:, 0]).any())
            for p in PARAMS:
                ids = g["ids_%s_%d" % (p, k)]
                repeated |= any(len(set(r[r >= 0].tolist())) < int((r >= 0).sum()) for r in ids)
                head = g["head_ids_%s_%d" % (p, k)]
                no_vector |= bool((f0.translate[head[head >= 0]] == oracle_spann.INT_MAX).any())
    assert pruned and truncated and repeated and no_vector
