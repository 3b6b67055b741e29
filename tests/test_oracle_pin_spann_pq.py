"""The plain-Python restatement of SPANN search on quantized indexes (tests/oracle_spann_pq.py) against the unmodified
reference's SPANN::Index<std::uint8_t>::SearchIndex on every fixture of tests/golden/spann_pq, every K, every parameter set
and both distances (SDC and ADC).  CPU only."""
import os

import numpy as np
import pytest

import oracle_spann
import oracle_spann_pq
from golden.make_golden_spann import KS, PARAMS
from golden.make_golden_spann_pq import MODES

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spann_pq")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
def test_restatement_equals_reference(case, pname, mode):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = oracle_spann.fixture_files(g)
    folder = oracle_spann.SpannFolder(files, PARAMS[pname])
    quant = oracle_spann_pq.folder_quantizer(files)
    assert folder.row_bytes == quant.m and folder.vis == quant.m + 4  # M code bytes + the id
    for k in KS:
        w = max(k, folder.internal)
        ids, dists, _ = oracle_spann_pq.search(folder, quant, g["queries"], g["head_ids_%s_%d" % (mode, w)],
                                               g["head_dists_%s_%d" % (mode, w)], k, mode == "adc")
        key = "%s_%s_%d" % (mode, pname, k)
        assert np.array_equal(ids, g["ids_" + key]), (case, key)
        assert np.array_equal(dists.view(np.int32), g["dists_" + key].view(np.int32)), (case, key)


def test_fixtures_cover_both_layouts_pruning_and_distinct_distances():
    """One case has plain lists in one file, the other rearranged lists in two; MaxDistRatio drops postings; SDC and ADC
    give different distances, and the reference's ValueType for the folders is UInt8 (the code rows it was built on)."""
    layouts, pruned, differ = set(), False, False
    for case in CASES:
        g = np.load(os.path.join(GOLDEN, case + ".npz"))
        files = oracle_spann.fixture_files(g)
        f0 = oracle_spann.SpannFolder(files)
        assert oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())["Base"]["ValueType"] == "UInt8"
        layouts.add((f0.rearranged, "SPTAGFullList.bin_1" in files))
        fr = oracle_spann.SpannFolder(files, PARAMS["ratio"])
        quant = oracle_spann_pq.folder_quantizer(files)
        a = oracle_spann_pq.search(f0, quant, g["queries"], g["head_ids_sdc_64"], g["head_dists_sdc_64"], 10, False)[2]
        b = oracle_spann_pq.search(fr, quant, g["queries"], g["head_ids_sdc_64"], g["head_dists_sdc_64"], 10, False)[2]
        pruned |= bool((b[:, 0] < a[:, 0]).any())
        differ |= not np.array_equal(g["dists_sdc_default_10"], g["dists_adc_default_10"])
    assert layouts == {(False, False), (True, True)} and pruned and differ
