"""Generate tests/golden/kernels/*.npz (TEST INFRASTRUCTURE): the reference's own search outputs on the combinations whose
kernels only they reach -- KD-trees over cosine rows of every element type, uint8 KD-trees, and uint8 cosine BKT.

Each fixture holds a small index BUILT BY THE UNMODIFIED REFERENCE (oracle/_ref/libsptag_ref.so: BuildIndex, SaveIndex),
flattened to arrays, its queries (cosine queries normalised as the reference's callers do: Utils::Normalize, truncation
toward zero), and for each (K, MaxCheck) of `runs` the reference's ids, distances and WorkSpace counters
(m_iNumberOfCheckedLeaves, m_iNumberOfTreeCheckedLeaves, NGQueue.size(), SPTQueue.size()).  The runs cross the
m_Results tiers of the kernels: max(MaxCheck / 16, K) at or below 512, in 513-1024 and in 1025-2048, with K above 32.
/root/reference is not needed to USE the fixtures (tests/test_oracle_pin_kernels.py, tests/test_gpu_kernel_coverage.py).
Run (where oracle/_ref exists):  python tests/golden/make_golden_kernels.py [name ...]
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import reflib  # noqa: E402
from make_test_data import _int8_lowrank, _int16_lowrank, _norm_i8, _norm_i16, _uint8_lowrank  # noqa: E402

OUT = os.path.join(HERE, "kernels")
N, NQ, INT_DIM, FLOAT_DIM = 800, 24, 44, 27
RUNS = [(10, 8192), (40, 1024), (200, 16384), (64, 32768)]
PARAMS = "NeighborhoodSize=16"


def _norm_u8(x):
    # Utils::Normalize for uint8 (CommonUtils.h:62-76): base = 255, truncation toward zero
    v = x.astype(np.float64)
    n = np.sqrt((v * v).sum(1, keepdims=True))
    return np.trunc(v / n * 255).astype(np.uint8)


CASES = {
    # name: (algo, metric, data, queries)
    "kdt_cos_f32_27": ("KDT", "Cosine", lambda: reflib.gen_lowrank(N, FLOAT_DIM, 6, 301),
                       lambda: reflib.normalize_rows(reflib.gen_lowrank(NQ, FLOAT_DIM, 6, 302))),
    "kdt_cos_i8_44": ("KDT", "Cosine", lambda: _int8_lowrank(N, INT_DIM, 8, 303), lambda: _norm_i8(_int8_lowrank(NQ, INT_DIM, 8, 304))),
    "kdt_cos_u8_44": ("KDT", "Cosine", lambda: _uint8_lowrank(N, INT_DIM, 8, 305),
                      lambda: _norm_u8(_uint8_lowrank(NQ, INT_DIM, 8, 306))),
    "kdt_cos_i16_44": ("KDT", "Cosine", lambda: _int16_lowrank(N, INT_DIM, 8, 307),
                       lambda: _norm_i16(_int16_lowrank(NQ, INT_DIM, 8, 308))),
    "kdt_l2_u8_44": ("KDT", "L2", lambda: _uint8_lowrank(N, INT_DIM, 8, 309), lambda: _uint8_lowrank(NQ, INT_DIM, 8, 310)),
    "bkt_cos_u8_44": ("BKT", "Cosine", lambda: _uint8_lowrank(N, INT_DIM, 8, 311),
                      lambda: _norm_u8(_uint8_lowrank(NQ, INT_DIM, 8, 312))),
}


def make(name):
    algo, metric, gen_data, gen_q = CASES[name]
    data = np.ascontiguousarray(gen_data())
    q = np.ascontiguousarray(gen_q())
    with tempfile.TemporaryDirectory() as tmp:
        reflib.RefIndex.build(algo, data, metric, threads=8, params=PARAMS).save(tmp)
        files = reflib.IndexFiles(tmp)
        r = reflib.RefIndex.load(tmp)
        assert r.enable_stats() == 0
        names = sorted(files.params)
        out = dict(param_names=np.array(names), param_values=np.array([files.params[n] for n in names]),
                   vectors=files.vectors, graph=files.graph, tree_starts=files.tree_starts, nodes=files.nodes, queries=q,
                   runs=np.array(RUNS, np.int32), ref_isa=np.int32(reflib.ref().ref_isa()))
        for i, (k, mc) in enumerate(RUNS):
            r.set_param("MaxCheck", mc)
            ids = np.empty((NQ, k), np.int32)
            dists = np.empty((NQ, k), np.float32)
            stats = np.empty((NQ, 4), np.int32)
            for j in range(NQ):
                ids[j], dists[j], stats[j] = r.search_one_stats(q[j], k)
            out["ref_ids_%d" % i], out["ref_dists_%d" % i], out["ref_stats_%d" % i] = ids, dists, stats
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print("golden", name, data.shape, os.path.getsize(path))


if __name__ == "__main__":
    for nm in (sys.argv[1:] or CASES):
        make(nm)
