"""Golden fixtures for SPANN search and SPANN iterators on uint8, int16 and integer-cosine rows whose size is not a multiple
of 16 bytes -- TEST INFRASTRUCTURE.

Builds five small SPANN indexes with the UNMODIFIED REFERENCE (tests/cpp/spann_elem_ref.cpp, linked with
oracle/_ref/libsptag_ref.so), the build recipe and clustered rows of make_golden_spann.py, one element type and metric per
case.  Every row size leaves padding before the 16-byte row stride the device packs rows at, and together the dimensions
end in every step width of the int16 distance (32, 16, 8, 4-wide steps and 1-wide tails):

  u8_l2_33          UInt8 L2, 33 x 1 byte (stride 48): odd, ends in a 1-wide tail
  u8_cos_rearr_44   UInt8 Cosine, 44 x 1 byte (stride 48), EnablePostingListRearrange; rows normalised to base 255
  i8_cos_17         Int8 Cosine, 17 x 1 byte (stride 32), two posting files; base 127
  i16_l2_63         Int16 L2, 63 x 2 bytes (stride 128): 32 + 16 + 8 + 4 + 3; values over most of +-32767, so differences
                    leave int16 and their squares pass 2^24
  i16_cos_rearr_45  Int16 Cosine, 45 x 2 bytes (stride 96), EnablePostingListRearrange; base 32767

Cosine rows and queries are normalised as the reference's callers do (Utils::Normalize, truncation toward zero).  The
rearranged layout stores a list's ids after its rows, at c * row_bytes: with these row sizes an id can start at a file
offset that is not a multiple of 4.

tests/golden/spann_elem/<case>.npz holds what make_golden_spann.py records (every file of the folder, the queries, the
reference's results and the head's results per parameter set of its PARAMS and K of its KS) and ref_isa, the SIMD width the
reference's DistanceUtils ran at (16: AVX-512, the only int16 rounding tree the device reproduces).
tests/golden/spann_elem_iter/<case>.npz holds what make_golden_spann_iterator.py records (its parameter sets, schedules
and layout) for these folders.  Running this twice writes byte-identical files (everything runs on one thread).
Run (where oracle/_ref exists):  python tests/golden/make_golden_spann_elem.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, HERE)

import make_golden_spann as mgs  # noqa: E402
import make_golden_spann_iterator as mgi  # noqa: E402
import reflib  # noqa: E402
from make_golden_kernels import _norm_u8  # noqa: E402
from make_test_data import _norm_i8, _norm_i16  # noqa: E402

OUT = os.path.join(HERE, "spann_elem")
OUT_ITER = os.path.join(HERE, "spann_elem_iter")

# case -> (value type, metric, rearranged, n, dim, posting files, seed)
CASES = {
    "u8_l2_33": ("UInt8", "L2", 0, 700, 33, 1, 21),
    "u8_cos_rearr_44": ("UInt8", "Cosine", 1, 700, 44, 1, 22),
    "i8_cos_17": ("Int8", "Cosine", 0, 700, 17, 2, 23),
    "i16_l2_63": ("Int16", "L2", 0, 500, 63, 1, 24),
    "i16_cos_rearr_45": ("Int16", "Cosine", 1, 500, 45, 1, 25),
}
NQ = 24
KB = 1024
CASE_BUDGET, TOTAL_BUDGET = 400 * KB, 2048 * KB


def data(vt, metric, n, dim, seed):
    """make_golden_spann's clustered float rows and queries (its first NQ queries: perturbed copies of rows, then fresh
    points), scaled to the element type's range; cosine rows and queries normalised with the type's base"""
    x, q = mgs.data("Float", "L2", n, dim, seed)
    x, q = x.astype(np.float64), q[:NQ].astype(np.float64)
    if vt == "UInt8":
        lo, hi = x.min(), x.max()
        x, q = [np.clip(np.rint((a - lo) / (hi - lo) * 255), 0, 255).astype(np.uint8) for a in (x, q)]
        return (_norm_u8(x), _norm_u8(q)) if metric == "Cosine" else (x, q)
    top, dtype, norm = {"Int8": (127, np.int8, _norm_i8), "Int16": (32767, np.int16, _norm_i16)}[vt]
    scale = top / np.abs(x).max()
    x, q = [np.clip(np.rint(a * scale), -top, top).astype(dtype) for a in (x, q)]
    return (norm(x), norm(q)) if metric == "Cosine" else (x, q)


def build_driver(out):
    src = os.path.join(TESTS, "cpp", "spann_elem_ref.cpp")
    ref_dir = os.path.join(os.path.dirname(TESTS), "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-include", "cstdint", "-I/root/reference/AnnService",
                           "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src, "-L" + ref_dir, "-lsptag_ref",
                           "-Wl,-rpath," + ref_dir])


def search_fixtures(drv, tmp):
    os.makedirs(OUT, exist_ok=True)
    isa = {512: 16, 256: 8, 128: 4, 0: 1}[int(reflib.ref().ref_isa())]  # vector bits -> floats per step
    assert isa == 16, "the reference's DistanceUtils ran at SIMD width %d, not AVX-512's 16" % isa
    for case, (vt, metric, rearr, n, dim, nfiles, seed) in CASES.items():
        x, q = data(vt, metric, n, dim, seed)
        assert (x.itemsize * dim) % 16 != 0, case
        xf, qf = os.path.join(tmp, "x.bin"), os.path.join(tmp, "q.bin")
        x.tofile(xf)
        q.tofile(qf)
        built = os.path.join(tmp, case)
        subprocess.check_call([drv, "build", built, vt, metric, str(rearr), str(n), str(dim), xf, str(nfiles), "1"])
        files = mgs.folder_files(built)
        out = {"file:" + rel: arr for rel, arr in files.items()}
        out["queries"] = q
        out["ref_isa"] = np.int32(isa)
        for pname, values in mgs.PARAMS.items():
            folder = os.path.join(tmp, case + "_" + pname)
            shutil.rmtree(folder, ignore_errors=True)
            mgs.write_folder(files, folder, values)
            for k in mgs.KS:
                pre = os.path.join(tmp, "r")
                subprocess.check_call([drv, "search", folder, qf, str(NQ), str(k), pre])
                w = max(k, 64)
                out["ids_%s_%d" % (pname, k)] = np.fromfile(pre + ".ids", np.int32).reshape(NQ, k)
                out["dists_%s_%d" % (pname, k)] = np.fromfile(pre + ".dists", np.float32).reshape(NQ, k)
                out["head_ids_%s_%d" % (pname, k)] = np.fromfile(pre + ".head_ids", np.int32).reshape(NQ, w)
                out["head_dists_%s_%d" % (pname, k)] = np.fromfile(pre + ".head_dists", np.float32).reshape(NQ, w)
        np.savez_compressed(os.path.join(OUT, case + ".npz"), **out)


def iterator_fixtures(drv, tmp):
    """make_golden_spann_iterator's parameter sets and schedules on the folders of OUT"""
    os.makedirs(OUT_ITER, exist_ok=True)
    for case in CASES:
        g = np.load(os.path.join(OUT, case + ".npz"))
        files = {key[5:]: g[key] for key in g.files if key.startswith("file:")}
        out = {}
        for pname, values in mgi.PARAMS.items():
            if not mgi.applies(case, pname):
                continue
            folder = os.path.join(tmp, case + "_iter_" + pname)
            mgs.write_folder(files, folder, values)
            for sname in ("short", "scan"):
                q = mgi.schedule_queries(g["queries"], sname)
                sched = list(mgi.SHORT) if sname == "short" else [mgi.SCAN_BATCH] * mgi.SCAN_CALLS
                counts, relaxed, ids, dists = mgi.run(drv, folder, q, sched, tmp)
                if sname == "scan":  # up to and including the first call that returns 0 for every query
                    done = np.nonzero(counts.sum(1) == 0)[0]
                    calls = int(done[0]) + 1 if len(done) else mgi.SCAN_CALLS
                    sched, counts, relaxed = sched[:calls], counts[:calls], relaxed[:calls]
                    ids, dists = ids[:calls * len(q) * mgi.SCAN_BATCH], dists[:calls * len(q) * mgi.SCAN_BATCH]
                key = "%s_%s" % (pname, sname)
                out["sched_" + key] = np.array(sched, np.int32)
                out["counts_" + key] = counts
                out["relaxed_" + key] = relaxed
                out["ids_" + key] = ids
                out["dists_" + key] = dists
        np.savez_compressed(os.path.join(OUT_ITER, case + ".npz"), **out)


def main():
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "spann_elem_ref")
        build_driver(drv)
        search_fixtures(drv, tmp)
        iterator_fixtures(drv, tmp)
    total = 0
    for d in (OUT, OUT_ITER):
        for case in CASES:
            size = os.path.getsize(os.path.join(d, case + ".npz"))
            total += size
            print("%s/%s.npz: %d bytes" % (os.path.basename(d), case, size))
            assert size < CASE_BUDGET, (d, case, size)
    print("total: %d bytes" % total)
    assert total < TOTAL_BUDGET, total


if __name__ == "__main__":
    sys.exit(main())
