"""The plain-Python restatement of SPANN's posting-list build (tests/oracle_spann_build.py) against the unmodified
reference's ExtraFullGraphSearcher::BuildIndex on every fixture of tests/golden/spann_build: from the recorded head
results it must write every posting file (and the rewritten head-id file) byte for byte and count the same RNG
rejections.  CPU only."""
import os

import numpy as np
import pytest

import oracle_spann
import oracle_spann_build

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spann_build")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def stage_input(g):
    """The folder as the stage finds it: no posting files, and the head-id file from before the stage"""
    files = oracle_spann.fixture_files(g)
    inp = {rel: arr for rel, arr in files.items() if not rel.startswith("SPTAGFullList.bin")}
    inp.update({key[4:]: g[key] for key in g.files if key.startswith("pre:")})
    return files, inp


@pytest.mark.parametrize("case", CASES)
def test_restatement_writes_the_reference_files(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    files, inp = stage_input(g)
    out, rejected, before, after = oracle_spann_build.build(inp, g["vectors"], g["head_ids"], g["head_dists"])
    assert sorted(n for n in out if n.startswith("SPTAGFullList.bin")) == sorted(
        n for n in files if n.startswith("SPTAGFullList.bin"))
    for name, blob in out.items():
        assert blob == bytes(files[name]), (case, name)
    assert rejected == int(g["rng_rejected"]), case
    assert after <= before


def test_fixtures_cover_cut_ties_and_layouts():
    """Some list is cut, some list holds vectors at equal distance from its head, one case is rearranged, one writes
    several files, one rewrites the head-id file."""
    cut = ties = rearranged = files_many = rewrite = False
    for case in CASES:
        g = np.load(os.path.join(GOLDEN, case + ".npz"))
        files, inp = stage_input(g)
        _, _, before, after = oracle_spann_build.build(inp, g["vectors"], g["head_ids"], g["head_dists"])
        cut |= after < before
        ini = oracle_spann.parse_ini(bytes(files["indexloader.ini"]).decode())
        rearranged |= ini["BuildSSDIndex"]["EnablePostingListRearrange"].lower() == "true"
        files_many |= sum(n.startswith("SPTAGFullList.bin") for n in files) > 1
        rewrite |= any(k.startswith("pre:") for k in g.files)
        d = g["head_dists"][:, :4]
        ties |= bool((np.diff(np.sort(d, axis=None)) == 0).any() and len(np.unique(g["vectors"], axis=0)) < len(g["vectors"]))
    assert cut and ties and rearranged and files_many and rewrite
