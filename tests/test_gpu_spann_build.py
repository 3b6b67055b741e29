"""SPANN's posting-list build on the device (sptag_b200_spann_build) against the unmodified reference's
ExtraFullGraphSearcher::BuildIndex, recorded in tests/golden/spann_build: from the folder as the stage finds it (no posting
files; with ExcludeHead false, the head-id file from before the stage) the device must write every file byte for byte,
count what the reference counts, and the built folder must search as the reference-built one does.  Also the refusals."""
import os

import numpy as np
import pytest

import oracle_spann
import oracle_spann_build
from golden.make_golden_spann import set_ini, write_folder
from sptag_b200 import capi

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "spann_build")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))
LACK_OF_INPUTS, MEMORY_OVERFLOW, EMPTY_DATA, DIMENSION_MISMATCH = 0x13, 0x12, 0x16, 0x17


def _stage_folder(g, folder, ini_values=None):
    """Writes the folder as the stage finds it; returns the fixture's files (the reference's output)"""
    files = oracle_spann.fixture_files(g)
    inp = {rel: arr for rel, arr in files.items() if not rel.startswith("SPTAGFullList.bin")}
    inp.update({key[4:]: g[key] for key in g.files if key.startswith("pre:")})
    write_folder(inp, folder, ini_values)
    return files


def _read_folder(folder):
    out = {}
    for dirpath, _, names in os.walk(folder):
        for nm in names:
            with open(os.path.join(dirpath, nm), "rb") as fh:
                out[os.path.relpath(os.path.join(dirpath, nm), folder)] = fh.read()
    return out


@pytest.mark.parametrize("case", CASES)
def test_build_writes_the_reference_files(case, tmp_path):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    built, ref = str(tmp_path / "built"), str(tmp_path / "ref")
    files = _stage_folder(g, built)
    before = _read_folder(built)
    stats = {}
    s = capi.B200SpannIndex.build(built, g["vectors"], stats=stats, device=0)
    try:
        after = _read_folder(built)
        assert sorted(after) == sorted(files), case
        for rel, blob in after.items():
            if rel.startswith("SPTAGFullList.bin") or rel == "SPTAGHeadVectorIDs.bin":
                assert blob == bytes(files[rel]), (case, rel)
            else:
                assert blob == before[rel], (case, rel)  # indexloader.ini and the head are not rewritten
        inp = {rel: np.frombuffer(b, np.uint8) for rel, b in before.items()}
        _, rejected, e_before, e_after = oracle_spann_build.build(inp, g["vectors"], g["head_ids"], g["head_dists"])
        n_heads = len(set(np.frombuffer(before["SPTAGHeadVectorIDs.bin"], np.uint64).tolist()) & set(range(len(g["vectors"]))))
        exclude = not any(k.startswith("pre:") for k in g.files)
        assert stats["searched"] == len(g["vectors"]) - (n_heads if exclude else 0)
        assert (stats["rng_rejected"], stats["edges_before_cut"], stats["edges_after_cut"]) == (
            int(g["rng_rejected"]), e_before, e_after), case
        # the built folder searches as the reference-built one does
        write_folder(files, ref)
        r = capi.B200SpannIndex.load(ref, 0)
        try:
            for k in (1, 10, 64):
                ids, dists = s.search(g["queries"], k)
                ids_r, dists_r = r.search(g["queries"], k)
                assert np.array_equal(ids, ids_r), (case, k)
                assert np.array_equal(dists.view(np.int32), dists_r.view(np.int32)), (case, k)
        finally:
            r.close()
    finally:
        s.close()


@pytest.mark.parametrize("case", ["build_cos_rearr_1k_24"])
def test_build_normalized_rows(case, tmp_path):
    """normalized = True takes the rows as they are: rows the caller normalised give the same files"""
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    files = _stage_folder(g, str(tmp_path))
    x = oracle_spann_build.normalize(g["vectors"], 1)
    capi.B200SpannIndex.build(str(tmp_path), x, normalized=True, device=0).close()
    with open(os.path.join(str(tmp_path), "SPTAGFullList.bin"), "rb") as fh:
        assert fh.read() == bytes(files["SPTAGFullList.bin"])


def _refused(g, folder, vectors, code, ini_values=None):
    _stage_folder(g, folder, ini_values)
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.build(folder, vectors, device=0)
    assert e.value.code == code, str(e.value)
    assert not os.path.exists(os.path.join(folder, "SPTAGFullList.bin"))


@pytest.mark.parametrize("key,value", [("EnableDataCompression", "true"), ("EnableDeltaEncoding", "true"),
                                       ("OutputEmptyReplicaID", "true"), ("QuantizerFilePath", "quantizer.bin"),
                                       ("ReplicaCount", "65")])
def test_build_refuses_what_it_does_not_reproduce(key, value, tmp_path):
    g = np.load(os.path.join(GOLDEN, "build_l2_1k_16.npz"))
    _refused(g, str(tmp_path), g["vectors"], LACK_OF_INPUTS, {key: value})


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_build_refuses_non_finite_rows(bad, tmp_path):
    g = np.load(os.path.join(GOLDEN, "build_l2_1k_16.npz"))
    x = g["vectors"].copy()
    x[1034, 5] = bad
    _refused(g, str(tmp_path), x, LACK_OF_INPUTS)


def test_build_refuses_empty_and_mismatched_input(tmp_path):
    g = np.load(os.path.join(GOLDEN, "build_l2_1k_16.npz"))
    _refused(g, str(tmp_path / "a"), g["vectors"][:0], EMPTY_DATA)
    _refused(g, str(tmp_path / "b"), np.ascontiguousarray(g["vectors"][:, :15]), DIMENSION_MISMATCH)


def test_build_refuses_more_edges_than_it_can_sort(tmp_path):
    """num x ReplicaCount above 2^31 - 1 edges: MemoryOverFlow before any row is read (the zero rows are never touched)"""
    g = np.load(os.path.join(GOLDEN, "build_i8_l2_2k_16.npz"))
    x = np.zeros((1 << 25, 16), np.int8)
    _refused(g, str(tmp_path), x, MEMORY_OVERFLOW, {"ReplicaCount": "64"})
