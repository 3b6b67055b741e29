"""SPANN search with the posting lists in HBM (sptag_b200_spann_*) against the unmodified reference's
SPANN::Index::SearchIndex, recorded in tests/golden/spann: ids and distance bits for every case, K and parameter set, the
counters against the plain-Python restatement (tests/oracle_spann.py), parameter changes between batches, two threads on
one handle, the refusals, and (where its driver was built) the reference itself on the folder the device loaded."""
import os
import subprocess
import threading

import numpy as np
import pytest

import oracle_spann
from golden.make_golden_spann import KS, PARAMS, write_folder
from sptag_b200 import capi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann")
# the unmodified reference's SPANN search (tests/cpp/spann_ref.cpp), built by __graft_entry__.build() where oracle/_ref is
REF_DRIVER = os.path.join(HERE, "cpp", "spann_ref")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def _fixture(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    return g, oracle_spann.fixture_files(g)


def _refused_truncation(files, values):
    f = oracle_spann.SpannFolder(files, values)
    return f.rearranged and any(f.searched(l) < f.lists[l][0] for l in range(len(f.lists)))


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
def test_spann_search_equals_reference(case, pname, tmp_path):
    g, files = _fixture(case)
    write_folder(files, str(tmp_path), PARAMS[pname])
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        q = g["queries"]
        if _refused_truncation(files, PARAMS[pname]):
            with pytest.raises(capi.SptagB200Error) as e:
                s.search(q, 10)
            assert e.value.code == 0x13
            return
        folder = oracle_spann.SpannFolder(files, PARAMS[pname])
        for k in KS:
            ids, dists, stats = s.search(q, k, want_stats=True)
            assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (case, pname, k)
            assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (case, pname, k)
            _, _, st = oracle_spann.search(folder, q, g["head_ids_%s_%d" % (pname, k)], g["head_dists_%s_%d" % (pname, k)], k)
            assert np.array_equal(stats, st), (case, pname, k)
    finally:
        s.close()


@pytest.mark.parametrize("case", CASES)
def test_reference_on_the_same_folder(case, tmp_path):
    """Where the reference driver was built, the reference itself searches the folder the device loaded."""
    if not os.path.exists(REF_DRIVER):
        pytest.skip("tests/cpp/spann_ref is built only where oracle/_ref exists")
    g, files = _fixture(case)
    folder = str(tmp_path / "index")
    write_folder(files, folder)
    q = g["queries"]
    qf = str(tmp_path / "q.bin")
    q.tofile(qf)
    s = capi.B200SpannIndex.load(folder, 0)
    try:
        for k in (10, 100):
            pre = str(tmp_path / "r")
            subprocess.check_call([REF_DRIVER, "search", folder, qf, str(len(q)), str(k), pre])
            ids, dists = s.search(q, k)
            assert np.array_equal(ids, np.fromfile(pre + ".ids", np.int32).reshape(len(q), k))
            assert np.array_equal(dists.view(np.int32), np.fromfile(pre + ".dists", np.int32).reshape(len(q), k))
    finally:
        s.close()


def test_set_param_between_batches(tmp_path):
    g, files = _fixture("spann_l2_3k_16")
    # PostingVectorLimit 1 lets SearchPostingPageLimit alone decide the truncation (as in the "pages" parameter set)
    write_folder(files, str(tmp_path), {"PostingVectorLimit": "1"})
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        q = g["queries"]
        for pname, values in (("ratio", {"MaxDistRatio": "1.5"}), ("default", {"MaxDistRatio": "10000"}),
                              ("pages", {"SearchPostingPageLimit": "1"}), ("default", {"SearchPostingPageLimit": "12"})):
            for name, v in values.items():
                s.set_param(name, v)
            for k in (10, 100):
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, g["ids_%s_%d" % (pname, k)]), (pname, k)
                assert np.array_equal(dists.view(np.int32), g["dists_%s_%d" % (pname, k)].view(np.int32)), (pname, k)
        s.set_param("SearchPostingPageLimit", 1)
        assert s.get_param("SearchPostingPageLimit") == "1"
        assert s.get_param("MaxCheck") == "4096"
        assert int(s.get_param("PostingBytes")) > 0
        with pytest.raises(capi.SptagB200Error):
            s.set_param("PostingBytes", 1)
    finally:
        s.close()


def test_two_threads_on_one_handle(tmp_path):
    g, files = _fixture("spann_i8_l2_2k_16")
    write_folder(files, str(tmp_path))
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    q = g["queries"]
    want = {k: (g["ids_default_%d" % k], g["dists_default_%d" % k].view(np.int32)) for k in (10, 100)}  # NpzFile: one thread
    errors = []

    def run(k):
        try:
            for _ in range(20):
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, want[k][0])
                assert np.array_equal(dists.view(np.int32), want[k][1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=run, args=(k,)) for k in (10, 100)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    s.close()
    assert not errors, errors


@pytest.mark.parametrize("key,value", [("EnableDataCompression", "true"), ("EnableDeltaEncoding", "true"),
                                       ("QuantizerFilePath", "quantizer.bin")])
def test_refuses_compression_delta_encoding_and_quantizers(key, value, tmp_path):
    _, files = _fixture("spann_l2_3k_16")
    write_folder(files, str(tmp_path), {key: value})
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.load(str(tmp_path), 0)
    assert e.value.code == 0x13


def test_ini_names_are_case_insensitive(tmp_path):
    """IniReader lower-cases and trims names (SimpleIniReader.cpp:55-120): a hand-edited key is still refused."""
    _, files = _fixture("spann_l2_3k_16")
    write_folder(files, str(tmp_path))
    ini = tmp_path / "indexloader.ini"
    ini.write_text(ini.read_text().replace("EnableDataCompression=false", "enabledatacompression = true"))
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.load(str(tmp_path), 0)
    assert e.value.code == 0x13
