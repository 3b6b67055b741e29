"""Golden fixtures for SPANN's posting-list build (the SSD stage of SPANN::Index::BuildIndex) -- TEST INFRASTRUCTURE.

Each case builds a small SPANN index with the UNMODIFIED REFERENCE (tests/cpp/spann_build_ref.cpp, linked with
oracle/_ref/libsptag_ref.so): SelectHead, BuildHead and BuildSSDIndex in one BuildIndex call, one thread, then SaveIndex.
The posting files are then deleted and the SSD stage alone (SelectHead and BuildHead off) runs again on that folder with
1 and with 8 threads; both must write files byte-identical to the full build's.  That is the claim the device build
rests on: given the head, the stage is a function of its inputs.

  build_l2_1k_16        float L2, 1200 x 16, ReplicaCount 8, plain lists, the default cut (180
                        elements at this row size; a tight blob of 400 rows makes lists longer than 118)
  build_cos_rearr_1k_24 float Cosine, 1200 x 24, rows NOT unit length, RNGFactor 1.5, ReplicaCount 6, rearranged lists
  build_i8_l2_2k_16     int8 L2, 2000 x 16, ReplicaCount 4, three posting files
  build_i16_l2_1k_20    int16 L2, 1500 x 20, ReplicaCount 5, ExcludeHead false (every vector is searched; the stage
                        rewrites the head-id file with MaxSize)
  build_l2_dups_1k_16   float L2, 1200 x 16 of 300 distinct rows (equal distances: the tonode order of ties),
                        ReplicaCount 4, PostingPageLimit 1 and PostingVectorLimit 1 (a heavy cut)

tests/golden/spann_build/<case>.npz holds:
  file:<path>     every file of the folder after the build (indexloader.ini with IndexDirectory blanked)
  pre:<path>      for ExcludeHead false: the head-id file as the stage finds it (each head's row id, recovered by
                  matching HeadIndex/vectors.bin against the rows; the full build itself overwrote it)
  vectors         the input rows (Cosine: before the stage normalises them)
  head_ids / head_dists  [n x InternalResultNum] the head index's SearchIndex for every row as the stage runs it
                  (MaxCheck of [BuildSSDIndex], Cosine rows normalised), head-local ids.  Only the results the RNG
                  selection examines are kept (it stops at ReplicaCount accepted heads, and the restatement
                  tests/oracle_spann_build.py tells where); the rest of each row is (-1, MaxDist), where the selection
                  stops too.  The generator checks that the restatement still writes the reference's files from them.
  rng_rejected    the RNG failed count ApproximateRNG logs
  queries         a few search queries (tests/test_gpu_spann_build.py searches the built folder with them)
/root/reference is not needed to USE the fixtures.
Run (where oracle/_ref exists):  python tests/golden/make_golden_spann_build.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "spann_build")
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_spann import folder_files  # noqa: E402
import oracle_spann_build  # noqa: E402

# case -> (value type, metric, n, dim, seed, duplicates, {Section.Name: value})
CASES = {
    # dups < 0: the first -dups rows lie in one tight blob, which makes some lists longer than 118 elements
    "build_l2_1k_16": ("Float", "L2", 1200, 16, 21, -400, {"BuildSSDIndex.ReplicaCount": "8"}),
    "build_cos_rearr_1k_24": ("Float", "Cosine", 1200, 24, 22, 0,
                              {"BuildSSDIndex.ReplicaCount": "6", "BuildSSDIndex.RNGFactor": "1.5",
                               "BuildSSDIndex.EnablePostingListRearrange": "true",
                               "BuildSSDIndex.SearchPostingPageLimit": "12"}),
    "build_i8_l2_2k_16": ("Int8", "L2", 2000, 16, 23, 0,
                          {"BuildSSDIndex.ReplicaCount": "4", "Base.SSDIndexFileNum": "3"}),
    "build_i16_l2_1k_20": ("Int16", "L2", 1500, 20, 24, 0,
                           {"BuildSSDIndex.ReplicaCount": "5", "BuildSSDIndex.ExcludeHead": "false"}),
    "build_l2_dups_1k_16": ("Float", "L2", 1200, 16, 25, 300,
                            {"BuildSSDIndex.ReplicaCount": "4", "BuildSSDIndex.PostingPageLimit": "1",
                             "BuildSSDIndex.PostingVectorLimit": "1"}),
}
INTERNAL = 64  # InternalResultNum (the default)
MAX_CHECK = 4096  # [BuildSSDIndex] MaxCheck (the default)
NQ = 16
DTYPES = {"Float": np.float32, "Int8": np.int8, "Int16": np.int16}


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "spann_build_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def data(vt, n, dim, seed, dups):
    """Clustered rows (posting lists of different lengths), `dups` > 0: n rows drawn from that many distinct ones.  Cosine
    rows are left at their length: the stage normalises them."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((40, dim)) * 3.0
    m = max(dups, 0) or n
    x = centres[rng.integers(0, 40, m)] + rng.standard_normal((m, dim))
    if dups < 0:
        x[:-dups] = centres[0] + 0.01 * rng.standard_normal((-dups, dim))
    if dups > 0:
        x = x[rng.integers(0, m, n)]
    q = centres[rng.integers(0, 40, NQ)] + rng.standard_normal((NQ, dim))
    if vt != "Float":
        scale = (127.0 if vt == "Int8" else 3000.0) / np.abs(x).max()
        lim = 127 if vt == "Int8" else 32767
        return (np.clip(np.rint(x * scale), -lim, lim).astype(DTYPES[vt]),
                np.clip(np.rint(q * scale), -lim, lim).astype(DTYPES[vt]))
    return x.astype(np.float32), q.astype(np.float32)


def posting_names(files):
    return sorted(rel for rel in files if rel.startswith("SPTAGFullList.bin"))


def head_row_ids(folder, x):
    """Each head's row id in x (the first row with its bytes), from HeadIndex/vectors.bin"""
    with open(os.path.join(folder, "HeadIndex", "vectors.bin"), "rb") as fh:
        rows, dim = np.frombuffer(fh.read(8), np.int32)
        heads = np.frombuffer(fh.read(), x.dtype).reshape(rows, dim)
    where = {x[i].tobytes(): i for i in range(len(x) - 1, -1, -1)}
    return np.array([where[h.tobytes()] for h in heads], np.uint64)


def main():
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "spann_build_ref")
        build_driver(drv)
        for case, (vt, metric, n, dim, seed, dups, params) in CASES.items():
            x, q = data(vt, n, dim, seed, dups)
            xf = os.path.join(tmp, "x.bin")
            x.tofile(xf)
            kv = ["%s=%s" % kv for kv in params.items()]
            built = os.path.join(tmp, case)
            shutil.rmtree(built, ignore_errors=True)
            subprocess.check_call([drv, "full", built, vt, metric, str(n), str(dim), xf, "1"] + kv)
            files = folder_files(built)
            exclude_head = params.get("BuildSSDIndex.ExcludeHead", "true") == "true"
            pre = {}
            if not exclude_head:
                pre["SPTAGHeadVectorIDs.bin"] = np.frombuffer(head_row_ids(built, x).tobytes(), np.uint8)
            rng_rejected = None
            for threads in (1, 8):
                # the SSD stage alone on the folder as the stage finds it
                for rel in posting_names(files):
                    os.remove(os.path.join(built, rel))
                for rel, arr in pre.items():
                    arr.tofile(os.path.join(built, rel))
                subprocess.check_call([drv, "ssd", built, vt, metric, str(n), str(dim), xf, str(threads)] + kv)
                with open(os.path.join(built, "rng.txt")) as fh:
                    rej = int(fh.read().split()[0])
                os.remove(os.path.join(built, "rng.txt"))
                again = folder_files(built)
                for rel in posting_names(files) + ["SPTAGHeadVectorIDs.bin"]:
                    assert np.array_equal(again[rel], files[rel]), (case, threads, rel)
                assert set(posting_names(again)) == set(posting_names(files)), case
                if threads == 1:
                    rng_rejected = rej
                assert rej == rng_rejected, (case, threads, rej, rng_rejected)
            pre_head = os.path.join(tmp, "h")
            subprocess.check_call([drv, "heads", built, vt, str(n), str(dim), xf, str(INTERNAL), str(MAX_CHECK),
                                   "1" if metric == "Cosine" else "0", pre_head])
            out = {"file:" + rel: arr for rel, arr in files.items()}
            out.update({"pre:" + rel: arr for rel, arr in pre.items()})
            out["vectors"] = x
            out["queries"] = q
            head_ids = np.fromfile(pre_head + ".ids", np.int32).reshape(n, INTERNAL)
            head_dists = np.fromfile(pre_head + ".dists", np.float32).reshape(n, INTERNAL)
            stage_in = {rel: arr for rel, arr in files.items() if rel not in posting_names(files)}
            stage_in.update(pre)
            read = np.zeros(n, np.int64)
            oracle_spann_build.build(stage_in, x, head_ids, head_dists, read=read)
            unread = np.arange(INTERNAL)[None, :] >= read[:, None]
            head_ids[unread] = -1
            head_dists[unread] = np.finfo(np.float32).max
            again, rej, _, _ = oracle_spann_build.build(stage_in, x, head_ids, head_dists)
            assert rej == rng_rejected and all(blob == files[name].tobytes() for name, blob in again.items()), case
            out["head_ids"] = head_ids
            out["head_dists"] = head_dists
            out["rng_rejected"] = np.array(rng_rejected, np.int64)
            path = os.path.join(OUT, case + ".npz")
            np.savez_compressed(path, **out)
            print("%s: %d bytes, %d posting files, %d RNG rejections" % (path, os.path.getsize(path),
                                                                         len(posting_names(files)), rng_rejected))


if __name__ == "__main__":
    sys.exit(main())
