"""SPANN's posting-list build with a device budget (sptag_b200_spann_build_ex) against the reference's files in
tests/golden/spann_build.  Below the resident path's working set the streamed path runs: rows read from the caller's
buffer, edges held in a pinned host store and sorted in groups of lists.  At every budget the files must equal the
reference's byte for byte, the counts must equal the reference's, and the built folder must search as the reference-built
one does.  Also: the budget's floor, the path choice at -1, the caller's rows left untouched, and the refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import oracle_spann
import oracle_spann_build
from golden.make_golden_spann import write_folder
from sptag_b200 import capi
from test_gpu_spann_build import GOLDEN, CASES, _read_folder, _stage_folder

pytestmark = pytest.mark.gpu

FAIL, LACK_OF_INPUTS, MEMORY_OVERFLOW = 0x01, 0x13, 0x12
ITEMSIZE = {"Float": 4, "Int8": 1, "UInt8": 1, "Int16": 2}


def _ini(g):
    return oracle_spann.parse_ini(bytes(oracle_spann.fixture_files(g)["indexloader.ini"]).decode())


def _resident_floor(g):
    """The resident path's working set from the header's formula, without the sort's scratch: any budget below it
    takes the streamed path"""
    ini = _ini(g)
    n, dim = g["vectors"].shape
    replicas = int(ini["BuildSSDIndex"].get("ReplicaCount", "8"))
    k = int(ini["BuildSSDIndex"].get("InternalResultNum", "64"))
    row = dim * ITEMSIZE[ini["Base"]["ValueType"]]
    return n * row + 24 * n * replicas + min(n, 65536) * k * 8 + (64 << 20)


def _files_of(folder):
    return {rel: b for rel, b in _read_folder(folder).items()
            if rel.startswith("SPTAGFullList.bin") or rel == "SPTAGHeadVectorIDs.bin"}


def _posting_files(folder):
    return [f for f in os.listdir(folder) if f.startswith("SPTAGFullList.bin")]


def _refused(folder, vectors, budget, code):
    with pytest.raises(capi.SptagB200Error) as e:
        capi.B200SpannIndex.build(folder, vectors, device=0, budget_bytes=budget)
    assert e.value.code == code, str(e.value)
    assert not _posting_files(folder)
    return str(e.value)


def _check_build(g, case, folder, files, before, stats):
    """The files equal the reference's and the counts its counts"""
    built = _files_of(folder)
    assert sorted(built) == sorted(rel for rel in files if rel.startswith("SPTAGFullList.bin")
                                   or rel == "SPTAGHeadVectorIDs.bin"), case
    for rel, blob in built.items():
        assert blob == bytes(files[rel]), (case, rel)
    inp = {rel: np.frombuffer(b, np.uint8) for rel, b in before.items()}
    _, rejected, e_before, e_after = oracle_spann_build.build(inp, g["vectors"], g["head_ids"], g["head_dists"])
    n_heads = len(set(np.frombuffer(before["SPTAGHeadVectorIDs.bin"], np.uint64).tolist()) & set(range(len(g["vectors"]))))
    exclude = not any(k.startswith("pre:") for k in g.files)
    assert stats["searched"] == len(g["vectors"]) - (n_heads if exclude else 0)
    assert (stats["rng_rejected"], stats["edges_before_cut"], stats["edges_after_cut"]) == (
        int(g["rng_rejected"]), e_before, e_after), case


@pytest.mark.parametrize("case", CASES)
def test_streamed_build_writes_the_reference_files(case, tmp_path):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    n_files = int(_ini(g)["Base"].get("SSDIndexFileNum", "1"))
    row_bytes = g["vectors"].shape[1] * g["vectors"].itemsize
    # the floor: a budget that holds pass 1 but not pass 2 is refused after pass 1, with the minimum in the message
    probe = str(tmp_path / "probe")
    _stage_folder(g, probe)
    msg = _refused(probe, g["vectors"], 64 << 10, MEMORY_OVERFLOW)
    minimum = int(re.search(r"needs at least (\d+) bytes", msg).group(1))
    assert 64 << 10 < minimum < _resident_floor(g)
    below = str(tmp_path / "below")
    _stage_folder(g, below)
    assert "needs at least %d bytes" % minimum in _refused(below, g["vectors"], minimum - 1, MEMORY_OVERFLOW)

    # at the minimum (several row batches; many groups, so group boundaries inside files), and just below the resident
    # path's working set (one batch, few groups)
    for budget in (minimum, _resident_floor(g) - 1):
        folder = str(tmp_path / ("b%d" % budget))
        files = _stage_folder(g, folder)
        before = _read_folder(folder)
        stats = {}
        s = capi.B200SpannIndex.build(folder, g["vectors"], device=0, stats=stats, budget_bytes=budget)
        try:
            assert stats["streamed"] == 1, (case, budget, stats)
            _check_build(g, case, folder, files, before, stats)
            stored = stats["edges_before_cut"]
            assert stats["h2d_bytes"] == (len(g["vectors"]) * row_bytes + stats["edge_groups"] * 12 * stored
                                          + stats["edges_after_cut"] * row_bytes), stats
            assert stats["edge_groups"] >= n_files
            if budget != minimum:
                continue
            assert stats["row_batches"] >= 2 and stats["edge_groups"] >= 3, (case, stats)
            assert stats["edge_groups"] > n_files, (case, stats)  # some file holds several groups
            ref = str(tmp_path / "ref")
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


@pytest.mark.parametrize("case", CASES)
def test_auto_budget_takes_the_resident_path(case, tmp_path):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    files = _stage_folder(g, a)
    before = _read_folder(a)
    _stage_folder(g, b)
    stats = {}
    capi.B200SpannIndex.build(a, g["vectors"], device=0, stats=stats, budget_bytes=-1).close()
    assert (stats["streamed"], stats["row_batches"], stats["edge_groups"]) == (0, 1, 1), stats
    assert stats["h2d_bytes"] == g["vectors"].nbytes
    _check_build(g, case, a, files, before, stats)
    capi.B200SpannIndex.build(b, g["vectors"], device=0).close()
    assert _files_of(a) == _files_of(b)


def test_streamed_build_leaves_the_callers_rows(tmp_path):
    """Cosine rows the caller has not normalised are normalised on the device copies only"""
    g = np.load(os.path.join(GOLDEN, "build_cos_rearr_1k_24.npz"))
    x = g["vectors"].copy()
    assert not np.allclose(np.linalg.norm(x, axis=1), 1.0)
    files = _stage_folder(g, str(tmp_path))
    stats = {}
    capi.B200SpannIndex.build(str(tmp_path), x, device=0, stats=stats, budget_bytes=_resident_floor(g) - 1).close()
    assert stats["streamed"] == 1
    assert x.tobytes() == g["vectors"].tobytes()
    with open(os.path.join(str(tmp_path), "SPTAGFullList.bin"), "rb") as fh:
        assert fh.read() == bytes(files["SPTAGFullList.bin"])


def test_build_ex_refusals(tmp_path):
    g = np.load(os.path.join(GOLDEN, "build_l2_1k_16.npz"))
    x = g["vectors"]
    folder = str(tmp_path / "a")
    _stage_folder(g, folder)
    _refused(folder, x, -2, LACK_OF_INPUTS)
    o = capi.SpannBuildOptions(C.sizeof(capi.SpannBuildOptions) - 4, -1)
    rc = capi.lib().sptag_b200_spann_build_ex(os.fsencode(folder), x.ctypes.data, x.shape[0], x.shape[1], 0, 0,
                                              C.byref(o), None)
    assert rc == FAIL
    assert not _posting_files(folder)
    # a refusal of sptag_b200_spann_build is one here too, at any budget
    for i, budget in enumerate((-1, 1 << 20)):
        folder = str(tmp_path / ("c%d" % i))
        _stage_folder(g, folder, {"EnableDataCompression": "true"})
        _refused(folder, x, budget, LACK_OF_INPUTS)
