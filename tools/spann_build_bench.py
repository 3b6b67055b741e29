#!/usr/bin/env python
"""spann_build_bench.py -- SPANN's posting-list build (the SSD stage of SPANN::Index::BuildIndex) on the device against
the reference.

For each --sizes entry: clustered float32 rows of tools/spann_bench.py (seeded), a head from the reference's SelectHead +
BuildHead (tests/cpp/spann_build_ref head, --threads host threads, not timed), then on copies of that folder:
  reference  the SSD stage alone (spann_build_ref ssd, SelectHead and BuildHead off, --threads host threads): wall time
  device     sptag_b200_spann_build (capi.B200SpannIndex.build): device ms of the head searches, the RNG selection and the
             sort, host ms of writing the files (bounded by the disk, reported apart), and the call's wall time
and compares every posting file byte for byte (SHA-256 of each file).  The card's name and power limit are read in the
same call.  Writes nothing in the tree: the folders go to a temporary directory.  One JSON line per size.

    python tools/spann_build_bench.py --sizes 200000 1000000 --dim 128
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from spann_bench import card, data  # noqa: E402

DRIVER = os.path.join(ROOT, "tests", "cpp", "spann_build_ref")


def digests(folder):
    out = {}
    for nm in sorted(os.listdir(folder)):
        if nm.startswith("SPTAGFullList.bin") or nm == "SPTAGHeadVectorIDs.bin":
            h = hashlib.sha256()
            with open(os.path.join(folder, nm), "rb") as fh:
                for chunk in iter(lambda: fh.read(64 << 20), b""):
                    h.update(chunk)
            out[nm] = (os.path.getsize(os.path.join(folder, nm)), h.hexdigest())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[200000, 1000000])
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--tmp", default=None, help="directory for the folders (default: the system's temporary directory)")
    a = ap.parse_args()
    if not os.path.exists(DRIVER):
        sys.exit("tests/cpp/spann_build_ref is missing: run __graft_entry__.build() where the reference sources exist")
    from sptag_b200 import capi
    for n in a.sizes:
        x, _ = data(n, a.dim, 2)
        res = {"card": card(), "n": n, "dim": a.dim, "metric": "L2", "dtype": "f32", "host_threads": a.threads}
        with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
            xf, head = os.path.join(tmp, "x.bin"), os.path.join(tmp, "head")
            x.tofile(xf)
            t0 = time.perf_counter()
            subprocess.check_call([DRIVER, "head", head, "Float", "L2", str(n), str(a.dim), xf, str(a.threads)],
                                  stdout=subprocess.DEVNULL)
            res["reference_head_s"] = round(time.perf_counter() - t0, 1)
            ref, dev = os.path.join(tmp, "ref"), os.path.join(tmp, "dev")
            shutil.copytree(head, ref)
            subprocess.check_call([DRIVER, "ssd", ref, "Float", "L2", str(n), str(a.dim), xf, str(a.threads)],
                                  stdout=subprocess.DEVNULL)
            with open(os.path.join(ref, "rng.txt")) as fh:
                rej, ref_ms = fh.read().split()
            ref_d = digests(ref)
            shutil.rmtree(ref)
            shutil.copytree(head, dev)
            stats = {}
            t0 = time.perf_counter()
            s = capi.B200SpannIndex.build(dev, x, device=0, stats=stats)
            wall = time.perf_counter() - t0
            s.close()
            dev_d = digests(dev)
        phases = {k: round(stats[k + "_us"] / 1000.0, 1) for k in ("search", "rng", "sort", "write")}
        dev_stage_ms = sum(phases.values())
        res.update({
            "reference_ssd_s": round(float(ref_ms) / 1000.0, 2),
            "reference_vectors_per_s": round(n / (float(ref_ms) / 1000.0), 1),
            "device_ms": phases,
            "device_stage_s": round(dev_stage_ms / 1000.0, 2),
            "device_vectors_per_s": round(n / (dev_stage_ms / 1000.0), 1),
            "device_vectors_per_s_without_write": round(n / ((dev_stage_ms - phases["write"]) / 1000.0), 1),
            "device_call_s": round(wall, 2),
            "searched": stats["searched"], "rng_rejected": stats["rng_rejected"],
            "reference_rng_rejected": int(rej),
            "edges_before_cut": stats["edges_before_cut"], "edges_after_cut": stats["edges_after_cut"],
            "posting_bytes": sum(v[0] for k, v in dev_d.items() if k.startswith("SPTAGFullList.bin")),
            "files_identical": dev_d == ref_d and len(ref_d) > 1,
        })
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
