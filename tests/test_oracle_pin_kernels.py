"""CPU tests: pin the C restatement (oracle/sptag_oracle.c) to the reference where no other fixture does -- KD-trees over
cosine rows of float, int8, uint8 and int16, a uint8 L2 KD-tree and a uint8 cosine BKT -- with committed outputs of the
unmodified reference (tests/golden/kernels, generator tests/golden/make_golden_kernels.py).  The GPU case matrix
(tests/test_gpu_kernel_coverage.py) compares the device with this oracle on the same combinations, so without these pins
it would prove nothing there.  No reference is needed at test time."""
import glob
import os

import numpy as np
import pytest

import reflib
import test_oracle_pin as pin

KERNELS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kernels")


def kernel_golden_cases():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(KERNELS, "*.npz")))


def test_fixtures_cover_the_unpinned_combinations():
    seen = set()
    for name in kernel_golden_cases():
        g = np.load(os.path.join(KERNELS, name + ".npz"))
        p = dict(zip(g["param_names"].tolist(), g["param_values"].tolist()))
        seen.add((p["IndexAlgoType"], p["ValueType"], p["DistCalcMethod"]))
        caps = {max(int(mc) // 16, int(k)) for k, mc in g["runs"].tolist()}
        # every m_Results tier of the kernels, and the unordered HBM result set (K > 32)
        assert {0 if c <= 512 else 1 if c <= 1024 else 2 for c in caps} == {0, 1, 2}, name
        assert any(int(k) > 32 for k, _ in g["runs"].tolist()), name
    assert seen >= {("KDT", "Float", "Cosine"), ("KDT", "Int8", "Cosine"), ("KDT", "UInt8", "Cosine"),
                    ("KDT", "Int16", "Cosine"), ("KDT", "UInt8", "L2"), ("BKT", "UInt8", "Cosine")}


@pytest.mark.parametrize("name", kernel_golden_cases())
def test_oracle_matches_reference_kernel_golden(oracle_lib, name):
    g = np.load(os.path.join(KERNELS, name + ".npz"))
    files = reflib.IndexFiles.__new__(reflib.IndexFiles)
    pin._files_from_npz(files, g)
    q = g["queries"]
    for i, (k, mc) in enumerate(g["runs"].tolist()):
        o = reflib.OracleIndex(files)
        o.max_check = int(mc)
        ids, dists, stats = o.search(q, int(k))
        assert np.array_equal(ids, g["ref_ids_%d" % i]), (name, k, mc)
        assert np.array_equal(dists.view(np.int32), g["ref_dists_%d" % i].view(np.int32)), (name, k, mc)
        st = g["ref_stats_%d" % i]
        assert np.array_equal(stats[:, reflib.ST_CHECKED], st[:, 0]), (name, k, mc)
        assert np.array_equal(stats[:, reflib.ST_TREE_CHECKED], st[:, 1]), (name, k, mc)
        assert np.array_equal(stats[:, reflib.ST_NG_LEFT], st[:, 2]), (name, k, mc)
        assert np.array_equal(stats[:, reflib.ST_SPT_LEFT], st[:, 3]), (name, k, mc)
