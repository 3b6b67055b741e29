"""SPANN search on PQ/OPQ-quantized indexes (sptag_b200_spann_* on a folder with [Base] QuantizerFilePath) against the
unmodified reference's SPANN::Index<std::uint8_t>::SearchIndex, recorded in tests/golden/spann_pq: ids and distance bits
for every case, parameter set, K and distance (SDC, ADC), the counters against the plain-Python restatement
(tests/oracle_spann_pq.py), EnableADC and the posting parameters changed between batches, two threads on one handle, the
refusals, and (where its driver was built) the reference itself on the folder the device loaded."""
import os
import subprocess
import threading

import numpy as np
import pytest

import oracle_spann
import oracle_spann_pq
from golden.make_golden_spann import KS, PARAMS, write_folder
from golden.make_golden_spann_pq import MODES
from sptag_b200 import capi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_pq")
# the unmodified reference's quantized SPANN search (tests/cpp/spann_pq_ref.cpp), built by __graft_entry__.build() where
# oracle/_ref is
REF_DRIVER = os.path.join(HERE, "cpp", "spann_pq_ref")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
LACK_OF_INPUTS = 0x13


def _fixture(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    return g, oracle_spann.fixture_files(g)


def _want(g, mode, pname, k):
    key = "%s_%s_%d" % (mode, pname, k)
    return g["ids_" + key], g["dists_" + key].view(np.int32)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("pname", sorted(PARAMS))
@pytest.mark.parametrize("mode", MODES)
def test_spann_pq_search_equals_reference(case, pname, mode, tmp_path):
    """ADC comes from the folder's [BuildSSDIndex] EnableADC here (SPANNIndex.cpp:73-76)"""
    g, files = _fixture(case)
    write_folder(files, str(tmp_path), dict(PARAMS[pname], EnableADC="true" if mode == "adc" else "false"))
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        assert s.get_param("EnableADC") == ("1" if mode == "adc" else "0")
        q = g["queries"]
        folder = oracle_spann.SpannFolder(files, PARAMS[pname])
        quant = oracle_spann_pq.folder_quantizer(files)
        for k in KS:
            ids, dists, stats = s.search(q, k, want_stats=True)
            want_ids, want_d = _want(g, mode, pname, k)
            assert np.array_equal(ids, want_ids), (case, pname, mode, k)
            assert np.array_equal(dists.view(np.int32), want_d), (case, pname, mode, k)
            w = max(k, folder.internal)
            _, _, st = oracle_spann_pq.search(folder, quant, q, g["head_ids_%s_%d" % (mode, w)],
                                              g["head_dists_%s_%d" % (mode, w)], k, mode == "adc")
            assert np.array_equal(stats, st), (case, pname, mode, k)
    finally:
        s.close()


@pytest.mark.parametrize("case", CASES)
def test_reference_on_the_same_folder(case, tmp_path):
    """Where the reference driver was built, the reference itself searches the folder the device loaded."""
    if not os.path.exists(REF_DRIVER):
        pytest.skip("tests/cpp/spann_pq_ref is built only where oracle/_ref exists")
    g, files = _fixture(case)
    folder = str(tmp_path / "index")
    write_folder(files, folder)
    q = g["queries"]
    qf = str(tmp_path / "q.bin")
    q.tofile(qf)
    s = capi.B200SpannIndex.load(folder, 0)
    try:
        for adc in (0, 1):
            s.set_param("EnableADC", adc)
            for k in (10, 100):
                pre = str(tmp_path / "r")
                subprocess.check_call([REF_DRIVER, "search", folder, qf, str(len(q)), str(k), str(adc), pre])
                ids, dists = s.search(q, k)
                assert np.array_equal(ids, np.fromfile(pre + ".ids", np.int32).reshape(len(q), k)), (adc, k)
                assert np.array_equal(dists.view(np.int32), np.fromfile(pre + ".dists", np.int32).reshape(len(q), k)), (adc, k)
    finally:
        s.close()


def test_set_param_between_batches(tmp_path):
    """EnableADC switches the head search and the posting scan together; the ratio and the page limit change what is read"""
    g, files = _fixture("spann_pq_f32_3k_16")
    write_folder(files, str(tmp_path), {"PostingVectorLimit": "1"})
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        q = g["queries"]
        steps = (("sdc", "ratio", {"MaxDistRatio": "1.5"}), ("adc", "ratio", {"EnableADC": "1"}),
                 ("adc", "default", {"MaxDistRatio": "10000"}), ("adc", "pages", {"SearchPostingPageLimit": "1"}),
                 ("sdc", "pages", {"EnableADC": "0"}), ("sdc", "default", {"SearchPostingPageLimit": "12"}))
        for mode, pname, values in steps:
            for name, v in values.items():
                s.set_param(name, v)
            for k in (10, 100):
                ids, dists = s.search(q, k)
                want_ids, want_d = _want(g, mode, pname, k)
                assert np.array_equal(ids, want_ids), (mode, pname, k)
                assert np.array_equal(dists.view(np.int32), want_d), (mode, pname, k)
        assert s.get_param("MaxCheck") == "4096"
    finally:
        s.close()


def test_posting_bytes_count_code_rows(tmp_path):
    """The lists hold M-byte code rows: PostingBytes is below what the raw rows alone would take"""
    g, files = _fixture("spann_pq_f32_3k_16")
    write_folder(files, str(tmp_path))
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        folder = oracle_spann.SpannFolder(files)
        total = sum(lst[0] for lst in folder.lists)
        raw_row = g["queries"].shape[1] * g["queries"].itemsize
        assert 0 < int(s.get_param("PostingBytes")) < total * raw_row
    finally:
        s.close()


def test_two_threads_on_one_handle(tmp_path):
    g, files = _fixture("spann_opq_i8_2k_24")
    write_folder(files, str(tmp_path), {"EnableADC": "true"})
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    q = g["queries"]
    want = {k: _want(g, "adc", "default", k) for k in (10, 100)}  # NpzFile: one thread
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


def _load_code(folder):
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.load(folder, 0)
    return e.value.code


def test_refuses_cosine_with_a_quantizer(tmp_path):
    """Quantized search is L2 only (PQQuantizer::CosineDistance is an error stub)"""
    _, files = _fixture("spann_pq_f32_3k_16")
    write_folder(files, str(tmp_path))
    ini = tmp_path / "indexloader.ini"
    text = ini.read_text()
    base = text.index("[Base]")
    at = text.index("DistCalcMethod=L2", base)
    ini.write_text(text[:at] + "DistCalcMethod=Cosine" + text[at + len("DistCalcMethod=L2"):])
    assert _load_code(str(tmp_path)) == LACK_OF_INPUTS


def test_refuses_a_quantizer_without_a_quantized_head(tmp_path):
    """A float SPANN folder with QuantizerFilePath set, and the quantizer file present: the head holds raw rows"""
    _, pq_files = _fixture("spann_pq_f32_3k_16")
    g = np.load(os.path.join(HERE, "golden", "spann", "spann_l2_3k_16.npz"))
    write_folder(oracle_spann.fixture_files(g), str(tmp_path), {"QuantizerFilePath": "quantizer.bin"})
    (tmp_path / "quantizer.bin").write_bytes(bytes(pq_files["quantizer.bin"]))
    assert _load_code(str(tmp_path)) == LACK_OF_INPUTS


def test_refuses_iterators(tmp_path):
    g, files = _fixture("spann_pq_f32_3k_16")
    write_folder(files, str(tmp_path))
    s = capi.B200SpannIndex.load(str(tmp_path), 0)
    try:
        with pytest.raises(capi.SptagB200Error) as e:
            s.iterators(g["queries"])
        assert e.value.code == LACK_OF_INPUTS
        ids, _ = s.search(g["queries"], 10)  # the handle still searches
        assert np.array_equal(ids, _want(g, "sdc", "default", 10)[0])
    finally:
        s.close()
