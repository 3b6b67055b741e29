"""Golden fixtures for SPANN search on PQ/OPQ-quantized indexes -- TEST INFRASTRUCTURE.

Builds two small quantized SPANN indexes with the UNMODIFIED REFERENCE (tests/cpp/spann_pq_ref.cpp, linked with
oracle/_ref/libsptag_ref.so) and records SPANN::Index<std::uint8_t>::SearchIndex(QueryResult&) on them.  The quantizer is
trained by reflib.train_quantizer and the code rows are the reference's own QuantizeVector of the raw rows, as in
make_golden_quantized.py; the index is built on the codes (IndexBuilder's route for a quantized index):

  spann_pq_f32_3k_16     PQ over float rows, 3000 x 16, M 4, plain lists, one posting file
  spann_opq_i8_2k_24     OPQ over int8 rows, 2000 x 24, M 6, EnablePostingListRearrange, two posting files

The queries are raw vectors (make_golden_spann.data).  For the parameter sets of make_golden_spann.py (default, ratio,
pages), K in (1, 10, 64, 100) and both distances of the quantizer (sdc: the symmetric table, adc: SetQuantizerADC(true)),
tests/golden/spann_pq/<case>.npz holds ids_<mode>_<p>_<K> / dists_<mode>_<p>_<K> (the reference's results),
head_ids_<mode>_<W> / head_dists_<mode>_<W> (the head index's search at W = max(K, SearchInternalResultNum), head-local
ids, the same under every parameter set), every file of the folder (key "file:<path>") and the queries.
/root/reference is not needed to USE them.
Run (where oracle/_ref exists):  python tests/golden/make_golden_spann_pq.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
import reflib  # noqa: E402
from golden.make_golden_spann import KS, NQ, PARAMS, data, folder_files, write_folder  # noqa: E402,F401

OUT = os.path.join(HERE, "spann_pq")
MODES = ("sdc", "adc")

# case -> (raw value type, rearranged, n, dim, M, opq, posting files, seed)
CASES = {
    "spann_pq_f32_3k_16": ("Float", 0, 3000, 16, 4, False, 1, 31),
    "spann_opq_i8_2k_24": ("Int8", 1, 2000, 24, 6, True, 2, 32),
}


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "spann_pq_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def main():
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "spann_pq_ref")
        build_driver(drv)
        for case, (vt, rearr, n, dim, m, opq, nfiles, seed) in CASES.items():
            x, q = data(vt, "L2", n, dim, seed)
            rtype = reflib.VT_INT8 if vt == "Int8" else reflib.VT_FLOAT
            qz = reflib.train_quantizer(x.astype(np.float32), m=m, ks=256, opq=opq, rtype=rtype, seed=7, iters=3)
            qpath = os.path.join(tmp, "quantizer_src.bin")
            qz.write(qpath)
            codes = reflib.RefQuantizer(qpath).encode(x)
            cf, qf = os.path.join(tmp, "codes.bin"), os.path.join(tmp, "q.bin")
            codes.tofile(cf)
            q.tofile(qf)
            built = os.path.join(tmp, case)
            subprocess.check_call([drv, "build", built, qpath, str(rearr), str(n), str(m), cf, str(nfiles)])
            files = folder_files(built)
            out = {"file:" + rel: arr for rel, arr in files.items()}
            out["queries"] = q
            for pname, values in PARAMS.items():
                folder = os.path.join(tmp, case + "_" + pname)
                shutil.rmtree(folder, ignore_errors=True)
                write_folder(files, folder, values)
                for mode in MODES:
                    for k in KS:
                        pre = os.path.join(tmp, "r")
                        subprocess.check_call([drv, "search", folder, qf, str(NQ), str(k), str(MODES.index(mode)), pre])
                        w = max(k, 64)
                        key = "%s_%s_%d" % (mode, pname, k)
                        out["ids_" + key] = np.fromfile(pre + ".ids", np.int32).reshape(NQ, k)
                        out["dists_" + key] = np.fromfile(pre + ".dists", np.float32).reshape(NQ, k)
                        # the head search reads no posting parameter: one record per distance and width
                        for name, dt in (("head_ids", np.int32), ("head_dists", np.float32)):
                            got = np.fromfile(pre + "." + name, dt).reshape(NQ, w)
                            hkey = "%s_%s_%d" % (name, mode, w)
                            assert hkey not in out or np.array_equal(out[hkey].view(np.int32), got.view(np.int32)), hkey
                            out[hkey] = got
            path = os.path.join(OUT, case + ".npz")
            np.savez_compressed(path, **out)
            print("%s: %d bytes" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    sys.exit(main())
