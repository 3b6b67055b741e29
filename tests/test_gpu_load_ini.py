"""GPU tests of how sptag_b200_load reads indexloader.ini: as VectorIndex::LoadIndex does (VectorIndex.cpp:617-681) with
Helper::IniReader (SimpleIniReader.cpp:40-135).  Section and parameter names are trimmed and matched case-insensitively,
and each name is read from its own section only: [Index] for the index (BKTIndex.cpp:21-31), [Quantizer] for the
quantizer file.  Results are compared bit for bit with the unmodified reference's golden outputs."""
import os

import numpy as np
import pytest

import test_oracle_pin_bfs as pin

pytestmark = pytest.mark.gpu


def write_index(tmp_path, name, edit=None, drop=()):
    """The golden index `name` as the reference saves it, its ini passed through edit(text)."""
    mk = pin.golden_module()
    g = np.load(os.path.join(pin.GOLDEN, name + ".npz"))
    ix = mk.index_from_npz(g)
    for key in drop:
        ix["params"].pop(key)
    folder = str(tmp_path / "idx")
    mk.write_folder(ix, folder)
    if edit is not None:
        ini = os.path.join(folder, "indexloader.ini")
        with open(ini) as f:
            text = f.read()
        with open(ini, "w") as f:
            f.write(edit(text))
    return g, folder


def check_golden(idx, g, mc, suffix=""):
    i = g["max_checks"].tolist().index(mc)
    ids, dists = idx.search(np.ascontiguousarray(g["queries"]), int(g["k"]))
    assert np.array_equal(ids, g["ref_ids" + suffix][i]), mc
    assert np.array_equal(dists.view(np.int32), g["ref_dists" + suffix][i].view(np.int32)), mc


def test_index_names_are_trimmed_and_case_insensitive(tmp_path):
    from sptag_b200 import B200Index
    g, folder = write_index(tmp_path, "bkt_l2_2k_16", drop=("MaxCheck",),
                            edit=lambda t: t.replace("[Index]\n", "[index]\n maxcheck = 64 \n"))
    idx = B200Index.load(folder, device=0)
    try:
        assert idx.get_param("MaxCheck") == "64"
        check_golden(idx, g, 64)
    finally:
        idx.close()


def test_index_parameters_of_another_section_are_not_read(tmp_path):
    from sptag_b200 import B200Index
    g, folder = write_index(tmp_path, "bkt_l2_2k_16", drop=("MaxCheck",), edit=lambda t: t + "\n[Other]\nMaxCheck=64\n")
    idx = B200Index.load(folder, device=0)
    try:
        assert idx.get_param("MaxCheck") == "8192"
        check_golden(idx, g, 8192)
    finally:
        idx.close()


def test_quantized_folder_reads_its_quantizer_section(tmp_path):
    from sptag_b200 import B200Index
    g, folder = write_index(tmp_path, os.path.join("quantized", "pq_f32_1200_16"))
    with open(os.path.join(folder, "indexloader.ini")) as f:
        assert f.read().startswith("[Quantizer]\nQuantizerFilePath=")
    idx = B200Index.load(folder, device=0)
    try:
        check_golden(idx, g, 8192, "_sdc")
    finally:
        idx.close()
