"""The C restatement with EnableBfs (TEST INFRASTRUCTURE).

oracle/sptag_oracle.c restates the default tree seeding only.  This module builds build/oracle_bfs/libsptag_oracle_bfs.so
from an unchanged copy of it in which bkt_init_search_trees is renamed bkt_init_search_trees_default, followed by
tests/oracle_bfs.c, which defines bkt_init_search_trees with the breadth-first branch (BKTree.h:703-758) and falls back
to the default at EnableBfs = 0.  Everything else -- distances, heaps, the search loops, refine, iterators -- is the
pinned restatement itself, compiled with oracle/Makefile's flags.  OracleBfsIndex is reflib.OracleIndex on that library.
"""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

import reflib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SRC = os.path.join(ROOT, "oracle", "sptag_oracle.c")
BFS_SRC = os.path.join(ROOT, "tests", "oracle_bfs.c")
OUT_DIR = os.path.join(ROOT, "build", "oracle_bfs")
LIB = os.path.join(OUT_DIR, "libsptag_oracle_bfs.so")
# oracle/Makefile's `port` flags: the same compiler settings keep every distance bit-identical to the pinned library
FLAGS = ["-std=c11", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-Wall", "-Wextra"]
DEFAULT_DEF = "static void bkt_init_search_trees(const qctx_t* c, ws_t* ws)\n"


def build():
    """(Re)build the library when its sources or flags differ from what it was built from."""
    with open(ORACLE_SRC) as f:
        src = f.read()
    with open(BFS_SRC) as f:
        bfs = f.read()
    digest = hashlib.sha256("\0".join([src, bfs] + FLAGS).encode()).hexdigest()
    stamp = LIB + ".srchash"
    if os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as f:
            if f.read().strip() == digest:
                return LIB
    if src.count(DEFAULT_DEF) != 1:
        raise RuntimeError("oracle/sptag_oracle.c: the definition of bkt_init_search_trees was not found")
    combined = src.replace(DEFAULT_DEF, "static void bkt_init_search_trees(const qctx_t* c, ws_t* ws);\n"
                                        "static void bkt_init_search_trees_default(const qctx_t* c, ws_t* ws)\n")
    combined += '\n#line 1 "tests/oracle_bfs.c"\n' + bfs
    os.makedirs(OUT_DIR, exist_ok=True)
    gen = os.path.join(OUT_DIR, "sptag_oracle_bfs.c")
    with open(gen, "w") as f:
        f.write(combined)
    tmp = LIB + ".tmp%d" % os.getpid()
    subprocess.check_call(["gcc"] + FLAGS + ["-I", os.path.join(ROOT, "oracle"), "-o", tmp, gen, "-lm"])
    os.replace(tmp, LIB)
    with open(stamp, "w") as f:
        f.write(digest + "\n")
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.ora_set_bfs.argtypes = [C.c_int32]
        L.ora_search_batch.argtypes = [C.POINTER(reflib._OraIndex), C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.ora_refine_nodes.argtypes = [C.POINTER(reflib._OraIndex), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.ora_iter_open.restype = C.c_void_p
        L.ora_iter_open.argtypes = [C.POINTER(reflib._OraIndex), C.c_void_p]
        L.ora_iter_next.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.ora_iter_close.argtypes = [C.c_void_p]
        L.ora_iter_next_from_nearest.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class OracleBfsIndex(reflib.OracleIndex):
    """reflib.OracleIndex with EnableBfs = `bfs` (BKTree::m_bfs).  The quantizer tables come from the pinned library."""

    def __init__(self, files, bfs=0, simd_width=16):
        super().__init__(files, simd_width)
        self.bfs = int(bfs)

    def search(self, queries, k, threads=0, want_stats=True):
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        stats = np.zeros((nq, reflib.ORA_ST_COUNT), np.int32)
        s = self._struct()
        lib().ora_set_bfs(self.bfs)
        rc = lib().ora_search_batch(C.byref(s), queries.ctypes.data, nq, k, ids.ctypes.data, dists.ctypes.data,
                                    stats.ctypes.data if want_stats else None, threads)
        assert rc == 0
        return ids, dists, stats

    def refine_nodes(self, first, num, cef, neighborhood=32, rng_factor=1.0, threads=0):
        rows = np.empty((num, neighborhood), np.int32)
        ids = np.empty((num, cef + 1), np.int32)
        dists = np.empty((num, cef + 1), np.float32)
        s = self._struct()
        lib().ora_set_bfs(self.bfs)
        rc = lib().ora_refine_nodes(C.byref(s), first, num, cef, neighborhood, rng_factor, rows.ctypes.data,
                                    ids.ctypes.data, dists.ctypes.data, threads)
        assert rc == 0
        return rows, ids, dists

    def iterator(self, query):
        return _BfsIterator(self, np.ascontiguousarray(query))


class _BfsIterator:
    """ResultIterator / SearchIndexIterativeFromNeareast; the seeding reads EnableBfs at the first call"""

    def __init__(self, oindex, query):
        self.oindex, self.query = oindex, query
        self.struct = oindex._struct()
        self.h = lib().ora_iter_open(C.byref(self.struct), query.ctypes.data)
        if not self.h:
            raise RuntimeError("ora_iter_open: unsupported index kind")

    def next(self, batch):
        ids = np.empty(batch, np.int32)
        dists = np.empty(batch, np.float32)
        relaxed = C.c_int32()
        lib().ora_set_bfs(self.oindex.bfs)
        count = lib().ora_iter_next(self.h, batch, ids.ctypes.data, dists.ctypes.data, C.byref(relaxed))
        return count, ids, dists, bool(relaxed.value)

    def next_from_nearest(self, k):
        ids = np.empty(k, np.int32)
        dists = np.empty(k, np.float32)
        lib().ora_set_bfs(self.oindex.bfs)
        ok = lib().ora_iter_next_from_nearest(self.h, k, ids.ctypes.data, dists.ctypes.data)
        assert ok >= 0
        return bool(ok), ids, dists

    def close(self):
        if self.h:
            lib().ora_iter_close(self.h)
            self.h = None
