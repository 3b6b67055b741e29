"""Golden fixtures for SPANN iterators (GetIterator + ResultIterator::Next) -- TEST INFRASTRUCTURE.

Runs the UNMODIFIED REFERENCE (tests/cpp/spann_iter_ref.cpp, linked with oracle/_ref/libsptag_ref.so) on the four SPANN
folders of tests/golden/spann (their files are read from those fixtures, not stored again) under four parameter sets,
each a variant of the folder's indexloader.ini:

  default   the folder as built (IterativeSearchHeadBatch 32, SearchInternalResultNum 64)
  hb4       IterativeSearchHeadBatch 4: the head is asked for its next batch many times within one call
  relaxed   SearchInternalResultNum 8 and IterativeSearchHeadBatch 8: RelaxedMono turns on after the first load
  pages     SearchPostingPageLimit 1 and PostingVectorLimit 1: lists longer than one page are truncated (plain layouts
            only: the device refuses truncated lists of the rearranged layout)

and two schedules of Next(batch) calls on fresh iterators:

  short     Next(64), Next(64), Next(16), Next(16), Next(1) on every query
  scan      Next(50) on the first SCAN_NQ queries until a call returns 0 for all of them, at most SCAN_CALLS calls

tests/golden/spann_iter/<case>.npz holds, per parameter set p and schedule s: sched_<p>_<s> (the batches),
counts_<p>_<s> [calls x nq] (resultNum), relaxed_<p>_<s> [calls x nq] (GetRelaxedMono()), and ids_<p>_<s> /
dists_<p>_<s>: the calls' [nq x batch] blocks one after another, the first resultNum results then (-1, MaxDist).  The
queries are those of tests/golden/spann/<case>.npz.  Running this twice writes byte-identical files.
Run (where oracle/_ref exists):  python tests/golden/make_golden_spann_iterator.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(HERE, "spann")
OUT = os.path.join(HERE, "spann_iter")

CASES = ("spann_l2_3k_16", "spann_cos_rearr_2k_24", "spann_i8_l2_2k_16", "spann_l2_heads_2k_16")
PARAMS = {
    "default": {},
    "hb4": {"IterativeSearchHeadBatch": "4"},
    "relaxed": {"SearchInternalResultNum": "8", "IterativeSearchHeadBatch": "8"},
    "pages": {"SearchPostingPageLimit": "1", "PostingVectorLimit": "1"},
}
SHORT = (64, 64, 16, 16, 1)
SCAN_BATCH, SCAN_NQ, SCAN_CALLS = 50, 8, 90


def applies(case, pname):
    """The pages set truncates lists, which the device refuses for the rearranged layout"""
    return not (pname == "pages" and "rearr" in case)


def schedule_queries(q, sname):
    return q if sname == "short" else q[:SCAN_NQ]


def run(drv, folder, q, sched, tmp):
    """The reference's iterate mode -> (counts [calls, nq], relaxed [calls, nq], ids, dists (flat blocks))"""
    qf, pre = os.path.join(tmp, "q.bin"), os.path.join(tmp, "it")
    q.tofile(qf)
    subprocess.check_call([drv, folder, qf, str(len(q)), pre, ",".join(map(str, sched))])
    counts = np.fromfile(pre + ".counts", np.int32).reshape(len(sched), len(q))
    relaxed = np.fromfile(pre + ".relaxed", np.uint8).reshape(len(sched), len(q))
    return counts, relaxed, np.fromfile(pre + ".ids", np.int32), np.fromfile(pre + ".dists", np.float32)


def build_driver(out):
    src = os.path.join(ROOT, "tests", "cpp", "spann_iter_ref.cpp")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-fopenmp", "-w", "-include", "cstdint",
                           "-I/root/reference/AnnService", "-I/root/reference/ThirdParty/zstd/lib", "-o", out, src,
                           "-L" + ref_dir, "-lsptag_ref", "-Wl,-rpath," + ref_dir])


def main():
    from make_golden_spann import write_folder  # run as a script from tests/golden
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        drv = os.path.join(tmp, "spann_iter_ref")
        build_driver(drv)
        for case in CASES:
            g = np.load(os.path.join(SRC, case + ".npz"))
            files = {key[5:]: g[key] for key in g.files if key.startswith("file:")}
            out = {}
            for pname, values in PARAMS.items():
                if not applies(case, pname):
                    continue
                folder = os.path.join(tmp, case + "_" + pname)
                write_folder(files, folder, values)
                for sname in ("short", "scan"):
                    q = schedule_queries(g["queries"], sname)
                    sched = list(SHORT) if sname == "short" else [SCAN_BATCH] * SCAN_CALLS
                    counts, relaxed, ids, dists = run(drv, folder, q, sched, tmp)
                    if sname == "scan":  # up to and including the first call that returns 0 for every query
                        done = np.nonzero(counts.sum(1) == 0)[0]
                        calls = int(done[0]) + 1 if len(done) else SCAN_CALLS
                        sched, counts, relaxed = sched[:calls], counts[:calls], relaxed[:calls]
                        ids, dists = ids[:calls * len(q) * SCAN_BATCH], dists[:calls * len(q) * SCAN_BATCH]
                    key = "%s_%s" % (pname, sname)
                    out["sched_" + key] = np.array(sched, np.int32)
                    out["counts_" + key] = counts
                    out["relaxed_" + key] = relaxed
                    out["ids_" + key] = ids
                    out["dists_" + key] = dists
            path = os.path.join(OUT, case + ".npz")
            np.savez_compressed(path, **out)
            print("%s: %d bytes" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    sys.exit(main())
