"""Golden fixtures for SPANN search with the posting lists in HBM -- TEST INFRASTRUCTURE.

Builds three small SPANN indexes with the UNMODIFIED REFERENCE (tests/cpp/spann_ref.cpp, linked with
oracle/_ref/libsptag_ref.so) and records SPANN::Index<T>::SearchIndex(QueryResult&) on them:

  spann_l2_3k_16        float L2, 3000 x 16
  spann_cos_rearr_2k_24 float Cosine, 2000 x 24, EnablePostingListRearrange
  spann_i8_l2_2k_16     int8 L2, 2000 x 16, two posting files (SSDIndexFileNum 2)
  spann_l2_heads_2k_16  float L2, 2000 x 16, built with ExcludeHead false: every head vector is in posting lists too.
                        That build writes MaxSize ("no vector") for every head into SPTAGHeadVectorIDs.bin; the file is
                        rewritten with each head's own row id (found by matching HeadIndex/vectors.bin against the data),
                        except every fifth head, which keeps MaxSize.  So a head result and a posting element can carry
                        the same id (the deduper is not seeded with the head results, and the reference returns such an id
                        twice), and some head results become (-1, MaxDist)

for K in (1, 10, 64, 100) under three parameter sets, each a variant of the folder's indexloader.ini:

  default   the folder as built (MaxDistRatio 10000, SearchPostingPageLimit 12: nothing is truncated)
  ratio     MaxDistRatio 1.5: postings far from the nearest head are not read
  pages     SearchPostingPageLimit 1 and PostingVectorLimit 1: lists longer than one page are truncated

tests/golden/spann/<case>.npz holds every file of the folder (key "file:<path>", bytes), the queries, and per parameter
set p and K: ids_<p>_<K> / dists_<p>_<K> (the reference's results) and head_ids_<p>_<K> / head_dists_<p>_<K> (the head
index's search at W = max(K, SearchInternalResultNum), head-local ids, as SPANN runs it).  The reference's
SearchIndex(QueryResult&) reports no counters (it passes no SearchStats, SPANNIndex.cpp:236); tests/oracle_spann.py
restates them.  /root/reference is not needed to USE the fixtures.
Run (where oracle/_ref exists):  python tests/golden/make_golden_spann.py
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "spann")

# case -> (value type, metric, rearranged, n, dim, posting files, heads in posting lists, seed)
CASES = {
    "spann_l2_3k_16": ("Float", "L2", 0, 3000, 16, 1, 0, 11),
    "spann_cos_rearr_2k_24": ("Float", "Cosine", 1, 2000, 24, 1, 0, 12),
    "spann_i8_l2_2k_16": ("Int8", "L2", 0, 2000, 16, 2, 0, 13),
    "spann_l2_heads_2k_16": ("Float", "L2", 0, 2000, 16, 1, 1, 14),
}
KS = (1, 10, 64, 100)
PARAMS = {
    "default": {},
    "ratio": {"MaxDistRatio": "1.5"},
    "pages": {"SearchPostingPageLimit": "1", "PostingVectorLimit": "1"},
}
NQ = 32


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "spann_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def data(vt, metric, n, dim, seed):
    """Clustered rows (so that posting lists differ in length) and queries: perturbed copies of indexed rows and fresh
    points.  Cosine rows are unit length, as the reference expects."""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((40, dim)) * 3.0
    x = centres[rng.integers(0, 40, n)] + rng.standard_normal((n, dim))
    q = np.concatenate([x[rng.choice(n, NQ // 2, replace=False)] + 0.05 * rng.standard_normal((NQ // 2, dim)),
                        centres[rng.integers(0, 40, NQ - NQ // 2)] + rng.standard_normal((NQ - NQ // 2, dim))])
    if vt == "Int8":
        scale = 127.0 / np.abs(x).max()
        return (np.clip(np.rint(x * scale), -127, 127).astype(np.int8),
                np.clip(np.rint(q * scale), -127, 127).astype(np.int8))
    x, q = x.astype(np.float32), q.astype(np.float32)
    if metric == "Cosine":
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
    return x, q


def set_ini(text, values):
    """indexloader.ini with Name=Value replaced in whichever section holds the name (every name here is in exactly one)."""
    lines = text.split("\n")
    for name, value in values.items():
        hits = [i for i, ln in enumerate(lines) if ln.split("=", 1)[0] == name]
        assert len(hits) == 1, (name, hits)
        lines[hits[0]] = name + "=" + value
    return "\n".join(lines)


def folder_files(folder):
    files = {}
    for dirpath, _, names in os.walk(folder):
        for nm in sorted(names):
            path = os.path.join(dirpath, nm)
            with open(path, "rb") as fh:
                blob = fh.read()
            rel = os.path.relpath(path, folder)
            if rel == "indexloader.ini":  # the build's own directory is no part of the index
                blob = set_ini(blob.decode(), {"IndexDirectory": ""}).encode()
            files[rel] = np.frombuffer(blob, np.uint8)
    return files


def restore_head_ids(folder, x):
    """SPTAGHeadVectorIDs.bin with each head's row id in x (every fifth head keeps MaxSize)"""
    with open(os.path.join(folder, "HeadIndex", "vectors.bin"), "rb") as fh:
        rows, dim = np.frombuffer(fh.read(8), np.int32)
        heads = np.frombuffer(fh.read(), x.dtype).reshape(rows, dim)
    where = {x[i].tobytes(): i for i in range(len(x) - 1, -1, -1)}  # the first row with these bytes
    ids = np.array([where[h.tobytes()] for h in heads], np.uint64)
    ids[::5] = np.uint64(2**31 - 1)
    ids.tofile(os.path.join(folder, "SPTAGHeadVectorIDs.bin"))


def write_folder(files, folder, ini_values=None):
    """The folder of a fixture under `folder`, its indexloader.ini changed by ini_values.  IndexDirectory names `folder`:
    the reference's LoadIndex reads the posting files from there (ExtraFullGraphSearcher.h:166)."""
    ini_values = dict(ini_values or {}, IndexDirectory=os.path.abspath(folder))
    for rel, arr in files.items():
        path = os.path.join(folder, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        blob = arr.tobytes()
        if rel == "indexloader.ini":
            blob = set_ini(blob.decode(), ini_values).encode()
        with open(path, "wb") as fh:
            fh.write(blob)


def main():
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "spann_ref")
        build_driver(drv)
        for case, (vt, metric, rearr, n, dim, nfiles, heads_in_lists, seed) in CASES.items():
            x, q = data(vt, metric, n, dim, seed)
            xf, qf = os.path.join(tmp, "x.bin"), os.path.join(tmp, "q.bin")
            x.tofile(xf)
            q.tofile(qf)
            built = os.path.join(tmp, case)
            subprocess.check_call([drv, "build", built, vt, metric, str(rearr), str(n), str(dim), xf, str(nfiles),
                                   "0" if heads_in_lists else "1"])
            if heads_in_lists:
                restore_head_ids(built, x)
            files = folder_files(built)
            out = {"file:" + rel: arr for rel, arr in files.items()}
            out["queries"] = q
            for pname, values in PARAMS.items():
                folder = os.path.join(tmp, case + "_" + pname)
                shutil.rmtree(folder, ignore_errors=True)
                write_folder(files, folder, values)
                for k in KS:
                    pre = os.path.join(tmp, "r")
                    subprocess.check_call([drv, "search", folder, qf, str(NQ), str(k), pre])
                    w = max(k, 64)
                    out["ids_%s_%d" % (pname, k)] = np.fromfile(pre + ".ids", np.int32).reshape(NQ, k)
                    out["dists_%s_%d" % (pname, k)] = np.fromfile(pre + ".dists", np.float32).reshape(NQ, k)
                    out["head_ids_%s_%d" % (pname, k)] = np.fromfile(pre + ".head_ids", np.int32).reshape(NQ, w)
                    out["head_dists_%s_%d" % (pname, k)] = np.fromfile(pre + ".head_dists", np.float32).reshape(NQ, w)
            path = os.path.join(OUT, case + ".npz")
            np.savez_compressed(path, **out)
            print("%s: %d bytes" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    sys.exit(main())
