"""GPU tests of the parameter surface of index and SPANN handles (sptag_b200_set_param / get_param,
sptag_b200_spann_set_param / get_param, and the ini keys sptag_b200_load and sptag_b200_spann_load hand to them), as
VectorIndex::SetParameter / GetParameter (BKTIndex.cpp:980-1025) and SPANN::Index::SetParameter / GetParameter
(SPANNIndex.cpp:1033-1073) define it: every name's default, a set / get round trip for every settable name, every
refusal and its code, and the ini keys.  The names are listed here, not read from the library, so that a name that
disappears or changes fails a test."""
import os

import numpy as np
import pytest

import oracle_spann
import test_oracle_pin_bfs as pin
from golden.make_golden_spann import write_folder as write_spann_folder
from sptag_b200 import B200Index, capi

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PARAM_NOT_FOUND, FAILED_PARSE_VALUE, LACK_OF_INPUTS = 0x10, 0x11, 0x13  # include/sptag_b200.h

# handle -> (golden fixture, prefix of its index arrays)
INDEXES = {"bkt": ("bkt_l2_2k_16", ""), "kdt": ("kdt_l2_2k_16", ""), "int8": ("mutation/bkt_cos_i8_1200_24", "base_"),
           "pq": ("quantized/pq_f32_1200_16", "")}
# settable name -> (default, a value to set, how get_param prints that value)
SETTABLE = {
    "MaxCheck": ("8192", "64", "64"),
    "MaxCheckForRefineGraph": ("8192", "100", "100"),
    "NumberOfInitialDynamicPivots": ("50", "30", "30"),
    "NumberOfOtherDynamicPivots": ("4", "7", "7"),
    "ThresholdOfNumberOfContinuousNoBetterPropagation": ("3", "5", "5"),
    "EnableBfs": ("0", "-2", "-2"),  # BKT only
    "AddCEF": ("500", "250", "250"),
    "CEF": ("1000", "900", "900"),
    "RNGFactor": ("1.000000", "1.25", "1.250000"),
    "SearchDeleted": ("0", "5", "1"),
    "EnableADC": ("0", "2", "1"),
    "B200.QueriesPerSM": ("0", "12", "12"),
    "B200.StageRows": ("0", "8", "8"),
    "B200.Stages": ("2", "1", "1"),
    "B200.NGCacheEntries": ("0", "16", "16"),
    "B200.SPTCacheEntries": ("0", "24", "24"),
    "B200.SimdWidth": ("16", "8", "8"),
    "B200.SlotScheme": ("0", "2", "2"),
    "B200.VisitedLog": ("-1", "1", "1"),
    "B200.VisitedLogEntries": ("0", "1024", "1024"),
    "B200.VisitedSet": ("-1", "1", "1"),
    "B200.VisitedHashEntries": ("0", "4096", "4096"),
    "B200.IteratorVisitedSet": ("-1", "0", "0"),
    "B200.IteratorVisitedHashEntries": ("0", "128", "128"),
    "B200.RowSketch": ("-1", "0", "0"),
}
# read-only name -> value on a handle that has run nothing
READ_ONLY = {"B200.RowsSkipped": "0", "B200.LastVisitedOverflows": "0", "B200.ScratchBytes": "256",
             "B200.LastIteratorSuspensions": "0,0", "B200.LastIteratorGrowths": "0", "B200.LastIteratorVisitedBytes": "0",
             "B200.LastRefineSearchUs": "0", "B200.LastRefineRebuildUs": "0"}
# the keys of the reference's [Index] section -> a value other than the default, and how get_param prints it
REF_KEYS = {"MaxCheck": ("1234", "1234"), "MaxCheckForRefineGraph": ("2345", "2345"),
            "NumberOfInitialDynamicPivots": ("31", "31"), "NumberOfOtherDynamicPivots": ("6", "6"),
            "ThresholdOfNumberOfContinuousNoBetterPropagation": ("9", "9"), "AddCEF": ("321", "321"),
            "CEF": ("654", "654"), "RNGFactor": ("1.5", "1.500000"), "EnableBfs": ("2", "2")}
# accepted-value sets of the checked names: (name, refused values, accepted values)
POW2 = (["32", "63", "100", "-64", str(1 << 31)], ["0", "64", str(1 << 30)])
INDEX_RANGES = [("B200.VisitedSet", ["-2", "2"], ["-1", "0", "1"]),
                ("B200.IteratorVisitedSet", ["-2", "2"], ["-1", "0", "1"]),
                ("B200.RowSketch", ["-2", "2"], ["-1", "0"]),
                ("B200.VisitedHashEntries",) + POW2,
                ("B200.IteratorVisitedHashEntries",) + POW2]

# the SPANN fixture, its [BuildHead] MaxCheck 4096
SPANN_CASE = "spann_l2_3k_16"
SPANN_HEAD = {"MaxCheck": ("4096", "512", "512"), "B200.IteratorVisitedSet": ("-1", "1", "1"),
              "B200.IteratorVisitedHashEntries": ("0", "256", "256")}
SPANN_SETTABLE = {"SearchInternalResultNum": ("64", "32", "32"), "SearchPostingPageLimit": ("12", "4", "4"),
                  "MaxDistRatio": ("10000.000000", "1.5", "1.500000"), "IterativeSearchHeadBatch": ("32", "16", "16"),
                  "B200.SpannDedupEntries": ("0", "1024", "1024")}
SPANN_READ_ONLY = {"B200.LastIteratorRounds": "0", "B200.LastIteratorDedupBytes": "0"}  # and PostingBytes
SPANN_RANGES = [("SearchInternalResultNum", ["-1", "2049"], ["0", "2048"]),
                ("SearchPostingPageLimit", ["-1", "2049"], ["0", "2048"]),
                ("IterativeSearchHeadBatch", ["0", "1025"], ["1", "1024"]),
                ("B200.SpannDedupEntries",) + POW2,
                ("B200.IteratorVisitedSet", ["2"], ["-1", "0", "1"]),
                ("B200.IteratorVisitedHashEntries", ["32"], ["0", "64"])]


def write_index(folder, case, params=None):
    """The golden index of `case` as the reference's SaveIndex lays it out, its [Index] keys updated by params."""
    mk = pin.golden_module()
    name, prefix = INDEXES[case]
    ix = mk.index_from_npz(np.load(os.path.join(GOLDEN, name + ".npz")), prefix)
    ix["params"].update(params or {})
    mk.write_folder(ix, folder)
    return folder


@pytest.fixture(params=sorted(INDEXES))
def index(request, tmp_path):
    idx = B200Index.load(write_index(str(tmp_path / "idx"), request.param), device=0)
    yield request.param, idx
    idx.close()


def write_spann(folder, head_max_check=None):
    g = np.load(os.path.join(GOLDEN, "spann", SPANN_CASE + ".npz"))
    write_spann_folder(oracle_spann.fixture_files(g), folder)
    if head_max_check is not None:
        ini = os.path.join(folder, "indexloader.ini")
        with open(ini) as f:
            text = f.read()
        head, rest = text.split("[BuildHead]\n", 1)
        assert "\nMaxCheck=4096\n" in rest.split("\n[", 1)[0]
        with open(ini, "w") as f:
            f.write(head + "[BuildHead]\n" + rest.replace("\nMaxCheck=4096\n", "\nMaxCheck=%s\n" % head_max_check, 1))
    return folder


@pytest.fixture
def spann(tmp_path):
    s = capi.B200SpannIndex.load(write_spann(str(tmp_path / "spann")), 0)
    yield s
    s.close()


def code(fn, *args):
    with pytest.raises(capi.SptagB200Error) as e:
        fn(*args)
    return e.value.code


def settable(case):
    return [n for n in SETTABLE if n != "EnableBfs" or case != "kdt"]


# ---- index handles ----------------------------------------------------------------------------------------------------
def test_defaults(index):
    case, idx = index
    for name in settable(case):
        assert idx.get_param(name) == SETTABLE[name][0], name
    for name, want in READ_ONLY.items():
        assert idx.get_param(name) == want, name


def test_round_trip(index):
    case, idx = index
    for name in settable(case):
        _, value, printed = SETTABLE[name]
        idx.set_param(name, value)
        assert idx.get_param(name) == printed, name
    if case == "bkt":
        idx.set_param("B200.RowSketch", 1)
        assert idx.get_param("B200.RowSketch") == "1"
    # integers: strtol base 10, trailing characters accepted; bool values: v != 0
    idx.set_param("MaxCheck", " 33abc")
    assert idx.get_param("MaxCheck") == "33"
    idx.set_param("SearchDeleted", "0")
    assert idx.get_param("SearchDeleted") == "0"
    idx.set_param("RNGFactor", "2e-1")
    assert idx.get_param("RNGFactor") == "0.200000"


def test_refusals(index):
    case, idx = index
    for name, refused, accepted in INDEX_RANGES:
        for v in refused:
            assert code(idx.set_param, name, v) == LACK_OF_INPUTS, (name, v)
            assert idx.get_param(name) == SETTABLE[name][0], (name, v)
        for v in accepted:
            idx.set_param(name, v)
            assert idx.get_param(name) == v, (name, v)
    for name in settable(case):
        for v in ("abc", ""):
            assert code(idx.set_param, name, v) == FAILED_PARSE_VALUE, (name, v)
    assert code(idx.get_param, "NoSuchParameter") == PARAM_NOT_FOUND
    assert code(idx.set_param, "NoSuchParameter", "1") == PARAM_NOT_FOUND
    if case == "kdt":  # EnableBfs is a BKT parameter
        assert code(idx.set_param, "EnableBfs", "1") == PARAM_NOT_FOUND
        assert code(idx.get_param, "EnableBfs") == PARAM_NOT_FOUND


def test_read_only_names_are_refused_as_read_only(index):
    _, idx = index
    for name, want in READ_ONLY.items():
        assert code(idx.set_param, name, "1") == LACK_OF_INPUTS, name
        assert idx.get_param(name) == want, name


@pytest.mark.parametrize("case", ["kdt", "int8", "pq"])
def test_row_sketch_on_is_refused_where_no_sketch_exists(case, tmp_path):
    idx = B200Index.load(write_index(str(tmp_path / "idx"), case), device=0)
    try:
        assert code(idx.set_param, "B200.RowSketch", "1") == LACK_OF_INPUTS
        assert idx.get_param("B200.RowSketch") == "-1"
        idx.set_param("B200.RowSketch", "0")
        assert idx.get_param("B200.RowSketch") == "0"
    finally:
        idx.close()


def test_names_are_case_insensitive(index):
    case, idx = index
    idx.set_param("maxcheck", "64")
    assert idx.get_param("MAXCHECK") == "64"
    assert idx.get_param("MaxCheck") == "64"
    idx.set_param("b200.visitedset", "1")
    assert idx.get_param("B200.VISITEDSET") == "1"
    assert code(idx.set_param, "b200.visitedset", "2") == LACK_OF_INPUTS
    assert idx.get_param("b200.lastiteratorsuspensions") == "0,0"
    assert code(idx.set_param, "B200.SCRATCHBYTES", "1") == LACK_OF_INPUTS
    if case == "kdt":
        assert code(idx.set_param, "enablebfs", "1") == PARAM_NOT_FOUND
    else:
        idx.set_param("enablebfs", "3")
        assert idx.get_param("EnableBfs") == "3"


def test_unknown_name_is_not_found_whatever_the_value(index):
    _, idx = index
    for v in ("abc", "", "1"):
        assert code(idx.set_param, "NoSuchParameter", v) == PARAM_NOT_FOUND, v
    assert code(idx.set_param, "MaxCheck", "abc") == FAILED_PARSE_VALUE


def test_rng_factor_takes_any_float(index):
    _, idx = index
    idx.set_param("RNGFactor", ".5")
    assert idx.get_param("RNGFactor") == "0.500000"
    assert code(idx.set_param, "RNGFactor", "abc") == FAILED_PARSE_VALUE
    assert idx.get_param("RNGFactor") == "0.500000"


@pytest.mark.parametrize("case", ["bkt", "kdt"])
def test_load_reads_every_reference_key(case, tmp_path):
    """sptag_b200_load sets the 9 keys of [Index] (BKTIndex.cpp:21-31); EnableBfs is ignored on a KDT folder."""
    folder = write_index(str(tmp_path / "idx"), case, {k: v for k, (v, _) in REF_KEYS.items()})
    idx = B200Index.load(folder, device=0)
    try:
        for name, (_, printed) in REF_KEYS.items():
            if case == "kdt" and name == "EnableBfs":
                assert code(idx.get_param, name) == PARAM_NOT_FOUND
            else:
                assert idx.get_param(name) == printed, name
    finally:
        idx.close()


def test_load_ignores_values_the_setter_refuses(tmp_path):
    """As LoadIndex ignores a failed ConvertStringTo: the folder loads and the parameter keeps its default."""
    idx = B200Index.load(write_index(str(tmp_path / "idx"), "bkt", {"MaxCheck": "abc", "CEF": "77"}), device=0)
    try:
        assert idx.get_param("MaxCheck") == "8192"
        assert idx.get_param("CEF") == "77"
    finally:
        idx.close()


# ---- SPANN handles ----------------------------------------------------------------------------------------------------
def test_spann_defaults_and_round_trip(spann):
    for table in (SPANN_HEAD, SPANN_SETTABLE):
        for name, (default, _, _) in table.items():
            assert spann.get_param(name) == default, name
    for name, want in SPANN_READ_ONLY.items():
        assert spann.get_param(name) == want, name
    assert int(spann.get_param("PostingBytes")) > 0
    for table in (SPANN_HEAD, SPANN_SETTABLE):
        for name, (_, value, printed) in table.items():
            spann.set_param(name, value)
            assert spann.get_param(name) == printed, name


def test_spann_refusals(spann):
    for name, refused, accepted in SPANN_RANGES:
        default = {**SPANN_HEAD, **SPANN_SETTABLE}[name][0]
        for v in refused:
            assert code(spann.set_param, name, v) == LACK_OF_INPUTS, (name, v)
            assert spann.get_param(name) == default, (name, v)
        for v in accepted:
            spann.set_param(name, v)
            assert spann.get_param(name) == v, (name, v)
    for name in list(SPANN_HEAD) + list(SPANN_SETTABLE):
        assert code(spann.set_param, name, "abc") == FAILED_PARSE_VALUE, name
    posting = spann.get_param("PostingBytes")
    for name in list(SPANN_READ_ONLY) + ["PostingBytes"]:
        assert code(spann.set_param, name, "1") == LACK_OF_INPUTS, name
    assert spann.get_param("PostingBytes") == posting
    # the head's other parameters are not the SPANN handle's
    for name in ("NoSuchParameter", "MaxCheckForRefineGraph", "B200.VisitedSet"):
        assert code(spann.set_param, name, "1") == PARAM_NOT_FOUND, name
        assert code(spann.set_param, name, "abc") == PARAM_NOT_FOUND, name
        assert code(spann.get_param, name) == PARAM_NOT_FOUND, name


def test_spann_names_are_case_insensitive(spann):
    spann.set_param("searchinternalresultnum", "32")
    assert spann.get_param("SEARCHINTERNALRESULTNUM") == "32"
    spann.set_param("maxcheck", "512")  # the head's
    assert spann.get_param("MAXCHECK") == "512"
    spann.set_param("b200.iteratorvisitedset", "1")
    assert spann.get_param("B200.IteratorVisitedSet") == "1"
    assert code(spann.set_param, "postingbytes", "1") == LACK_OF_INPUTS


def test_spann_load_hands_build_head_to_the_head(tmp_path):
    s = capi.B200SpannIndex.load(write_spann(str(tmp_path / "spann"), head_max_check=1234), 0)
    try:
        assert s.get_param("MaxCheck") == "1234"
    finally:
        s.close()
