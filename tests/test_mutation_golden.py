"""CPU test: the normalisation sptag_b200_add applies to Cosine rows (normalize_rows_kernel), restated in numpy, against
the rows the unmodified reference's AddIndex stored (tests/golden/mutation/*.npz, made by make_golden_mutation.py).

Utils::Normalize (CommonUtils.h:62-76): a double accumulator in element order, sqrt, then (T)(x / len * base) with
base = 1 for float and numeric_limits<T>::max() otherwise; the integer cast truncates toward zero."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mutation")
CASES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".npz"))


def normalize(rows):
    rows = np.asarray(rows)
    base = 1.0 if rows.dtype == np.float32 else float(np.iinfo(rows.dtype).max)
    x = rows.astype(np.float64)
    length = np.sqrt(np.cumsum(x * x, axis=1)[:, -1])  # element order; products of T values are exact in double
    out = np.empty_like(rows)
    for i in range(rows.shape[0]):
        if length[i] < 1e-6:
            v = 1.0 / np.sqrt(float(rows.shape[1])) * base
            y = np.full(rows.shape[1], v)
        else:
            y = x[i] / length[i] * base
        out[i] = y.astype(np.float32) if rows.dtype == np.float32 else np.trunc(y).astype(rows.dtype)
    return out


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("case", CASES)
def test_added_rows_are_normalised_like_the_reference(case):
    m = np.load(os.path.join(GOLDEN, case + ".npz"))
    src = m if "base_param_names" in m else np.load(os.path.join(os.path.dirname(GOLDEN), str(m["fixture"]) + ".npz"))
    key = "base_param_" if "base_param_names" in m else "param_"
    params = dict(zip(src[key + "names"].tolist(), src[key + "values"].tolist()))
    cosine = params["DistCalcMethod"] == "Cosine"
    a, b = m["batch_a"], m["batch_b"]
    if not cosine or int(m["normalized"]):  # stored as given
        assert np.array_equal(bits(m["added1"]), bits(a))
        assert np.array_equal(bits(m["added2"]), bits(b))
    else:
        assert np.array_equal(bits(m["added1"]), bits(normalize(a)))
        assert np.array_equal(bits(m["added2"]), bits(normalize(b)))


def test_fixtures_cover_the_mutation_sequence():
    for case in CASES:
        m = np.load(os.path.join(GOLDEN, case + ".npz"))
        n = m["graph1"].shape[0] - 200
        assert m["graph2"].shape[0] == n + 250
        codes = m["del_codes"]
        assert set(codes[:-1].tolist()) == {0, 0x14}  # live ids and repeats
        assert int(m["num_deleted2"]) == int((m["deleted2"] == 1).sum())
