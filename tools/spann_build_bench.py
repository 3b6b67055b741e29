#!/usr/bin/env python
"""spann_build_bench.py -- SPANN's posting-list build (the SSD stage of SPANN::Index::BuildIndex) on the device: the
resident path against the streamed path, and against the reference.

For each --sizes entry: clustered float32 rows of tools/spann_bench.py (seeded) and a head, then on copies of that folder:
  reference  (sizes <= --reference-max only) the SSD stage alone (spann_build_ref ssd, SelectHead and BuildHead off,
             --threads host threads): wall time
  resident   sptag_b200_spann_build (capi.B200SpannIndex.build): rows and edges in HBM
  streamed   sptag_b200_spann_build_ex at --budget device bytes: rows read from host memory, edges in a pinned host store,
             sorted and written in groups of lists
The device arms run alternately, --repeat times each; every run's files must be byte-identical (SHA-256 of each file),
and the reference's too where it runs.  Reported per arm (the median run): device ms of the head searches, the RNG
selection and the sort, host ms of the rest (the write; on the streamed path also the edge passes and the row gathers),
the row batches, edge groups and host-to-device bytes, and the call's wall time.  One more streamed run under
torch.profiler splits the streamed path's pass 2 into device time per kernel family and host-to-device copy time.
The head: up to --reference-max rows the reference's SelectHead + BuildHead (tests/cpp/spann_build_ref head, not
timed); above it the reference's head build does not fit one run, so the head is a seeded 10 % sample of the rows with
a BKT + RNG graph from tools/gpu_index_builder.py (not timed), and the equality check is between the device arms.
The card's name and power limit are read in the same call.  Writes nothing in the tree: the folders go to a temporary
directory.  One JSON line per size.

    python tools/spann_build_bench.py --sizes 200000 1000000 --dim 128 --budget 268435456
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


SPANN_INI = """[Index]
IndexAlgoType=SPANN
ValueType=Float

[Base]
ValueType=Float
DistCalcMethod=L2
IndexAlgoType=BKT
Dim={dim}
HeadVectorIDs=SPTAGHeadVectorIDs.bin
HeadIndexFolder=HeadIndex
SSDIndex=SPTAGFullList.bin
SSDIndexFileNum=1

[BuildSSDIndex]
isExecute=true
BuildSsdIndex=true
"""


def sample_head(x, folder, seed=11):
    """A SPANN folder whose head is a seeded 10 % sample of the rows, indexed with tools/gpu_index_builder.py"""
    import numpy as np
    import torch
    import gpu_index_builder as gib
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(len(x), max(1, len(x) // 10), replace=False))
    hx = np.ascontiguousarray(x[ids])
    nodes, starts, graph = gib.build_index(torch.from_numpy(hx).cuda(), metric="L2")
    torch.cuda.synchronize()
    gib.save_index_folder(os.path.join(folder, "HeadIndex"), hx, graph, nodes, starts, "L2")
    ids.astype(np.uint64).tofile(os.path.join(folder, "SPTAGHeadVectorIDs.bin"))
    with open(os.path.join(folder, "indexloader.ini"), "w") as f:
        f.write(SPANN_INI.format(dim=x.shape[1]))


def run_arm(capi, head, folder, x, budget):
    shutil.copytree(head, folder)
    stats = {}
    t0 = time.perf_counter()
    s = capi.B200SpannIndex.build(folder, x, device=0, stats=stats, budget_bytes=budget)
    wall = time.perf_counter() - t0
    s.close()
    d = digests(folder)
    shutil.rmtree(folder)
    stats["call_s"] = round(wall, 2)
    return stats, d


def profile_streamed(capi, head, folder, x, budget):
    """Device time of the streamed build's kernels by family, and of its host-to-device copies, in ms"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fam = {"edge passes (select)": ("spann_edge_flag", "DeviceSelect", "DeviceCompact"),
           "sort": ("DeviceRadixSort", "Onesweep", "RadixSort"), "gather": ("spann_row_gather",),
           "image": ("spann_posting_image",), "search": ("search_kernel",), "rng": ("spann_rng_select",)}
    torch.zeros(1, device="cuda")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_arm(capi, head, folder, x, budget)
    out = {k: 0.0 for k in fam}
    out["h2d copies"] = out["other"] = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
        if t <= 0:
            continue
        if "HtoD" in e.key:
            out["h2d copies"] += t
            continue
        for k, names in fam.items():
            if any(n in e.key for n in names):
                out[k] += t
                break
        else:
            out["other"] += t
    return {k: round(v, 1) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[200000, 1000000])
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--budget", type=int, default=256 << 20, help="the streamed arm's device budget in bytes")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--reference-max", type=int, default=200000)
    ap.add_argument("--tmp", default=None, help="directory for the folders (default: the system's temporary directory)")
    a = ap.parse_args()
    from sptag_b200 import capi
    for n in a.sizes:
        x, _ = data(n, a.dim, 2)
        reference = n <= a.reference_max
        if reference and not os.path.exists(DRIVER):
            sys.exit("tests/cpp/spann_build_ref is missing: run __graft_entry__.build() where the reference sources exist")
        res = {"card": card(), "n": n, "dim": a.dim, "metric": "L2", "dtype": "f32", "budget": a.budget,
               "head": "reference" if reference else "sample"}
        with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
            xf, head = os.path.join(tmp, "x.bin"), os.path.join(tmp, "head")
            t0 = time.perf_counter()
            if reference:
                x.tofile(xf)
                subprocess.check_call([DRIVER, "head", head, "Float", "L2", str(n), str(a.dim), xf, str(a.threads)],
                                      stdout=subprocess.DEVNULL)
            else:
                os.makedirs(head)
                sample_head(x, head)
            res["head_s"] = round(time.perf_counter() - t0, 1)
            digest_set = []
            if reference:
                ref = os.path.join(tmp, "ref")
                shutil.copytree(head, ref)
                subprocess.check_call([DRIVER, "ssd", ref, "Float", "L2", str(n), str(a.dim), xf, str(a.threads)],
                                      stdout=subprocess.DEVNULL)
                with open(os.path.join(ref, "rng.txt")) as fh:
                    rej, ref_ms = fh.read().split()
                digest_set.append(digests(ref))
                shutil.rmtree(ref)
                res.update({"reference_ssd_s": round(float(ref_ms) / 1000.0, 2), "reference_rng_rejected": int(rej),
                            "reference_vectors_per_s": round(n / (float(ref_ms) / 1000.0), 1)})
            runs = {"resident": [], "streamed": []}
            for _ in range(a.repeat):
                for arm, budget in (("resident", None), ("streamed", a.budget)):
                    st, d = run_arm(capi, head, os.path.join(tmp, arm), x, budget)
                    runs[arm].append(st)
                    digest_set.append(d)
            res["streamed_pass2_device_ms"] = profile_streamed(capi, head, os.path.join(tmp, "prof"), x, a.budget)
        for arm, rs in runs.items():
            rs.sort(key=lambda r: r["call_s"])
            st = rs[len(rs) // 2]
            phases = {k: round(st[k + "_us"] / 1000.0, 1) for k in ("search", "rng", "sort", "write")}
            res[arm] = {"ms": phases, "stage_s": round(sum(phases.values()) / 1000.0, 2),
                        "call_s": [r["call_s"] for r in rs],
                        "vectors_per_s": round(n / (sum(phases.values()) / 1000.0), 1)}
            for k in ("streamed", "row_batches", "edge_groups", "h2d_bytes"):
                if k in st:
                    res[arm][k] = st[k]
        st = runs["streamed"][0]
        res.update({
            "streamed_over_resident_stage": round(res["streamed"]["stage_s"] / max(res["resident"]["stage_s"], 1e-9), 2),
            "edge_store_bytes": 12 * st["edges_before_cut"],
            "h2d_bytes_streamed": {"rows": n * a.dim * 4, "edge_passes": st["edge_groups"] * 12 * st["edges_before_cut"],
                                   "gathered_rows": st["edges_after_cut"] * a.dim * 4},
            "searched": st["searched"], "rng_rejected": st["rng_rejected"],
            "edges_before_cut": st["edges_before_cut"], "edges_after_cut": st["edges_after_cut"],
            "posting_bytes": sum(v[0] for k, v in digest_set[0].items() if k.startswith("SPTAGFullList.bin")),
            "files_identical": all(d == digest_set[0] for d in digest_set) and len(digest_set[0]) > 1,
        })
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
