"""ctypes binding of libsptag_b200 (include/sptag_b200.h).

This is plumbing for tests and bench.py: every call goes through the C ABI, exactly the entry
points a C++/cgo/JNI host would bind.  There is no fallback -- if the CUDA library is missing or
the device is not an H100 (sm_90) the calls raise.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SPTAG_B200_LIB", os.path.join(_HERE, "lib", "libsptag_b200.so"))

STATS_PER_QUERY = 8
ST_CHECKED, ST_TREE_CHECKED, ST_NG_LEFT, ST_SPT_LEFT, ST_NDIST, ST_NEXPAND, ST_NTREE, ST_FLAGS = range(8)

VT_INT8, VT_UINT8, VT_INT16, VT_FLOAT = 0, 1, 2, 3
METRIC_L2, METRIC_COSINE, METRIC_IP = 0, 1, 2
ALGO_BKT, ALGO_KDT = 0, 1

EXPORTS = [
    "sptag_b200_create", "sptag_b200_load", "sptag_b200_destroy", "sptag_b200_set_param", "sptag_b200_set_quantizer",
    "sptag_b200_quantize", "sptag_b200_search_filtered",
    "sptag_b200_get_param", "sptag_b200_search", "sptag_b200_search_device", "sptag_b200_distance_batch",
    "sptag_b200_merge_topk", "sptag_b200_last_kernel_ms", "sptag_b200_launch_count",
    "sptag_b200_num_vectors", "sptag_b200_dim", "sptag_b200_value_type", "sptag_b200_metric",
    "sptag_b200_algo", "sptag_b200_last_error", "sptag_b200_refine_graph", "sptag_b200_get_graph",
    "sptag_b200_graph_degree", "sptag_b200_iterator_open", "sptag_b200_iterator_next", "sptag_b200_iterator_close",
    "sptag_b200_iterator_next_from_nearest", "sptag_b200_search_ex", "sptag_b200_iterator_open_ex",
    "sptag_b200_refine_search", "sptag_b200_refine_schedule", "sptag_b200_rebuild_graph", "sptag_b200_group_create", "sptag_b200_group_search",
    "sptag_b200_group_destroy", "sptag_b200_add", "sptag_b200_delete", "sptag_b200_delete_vectors", "sptag_b200_save",
    "sptag_b200_num_deleted",
]


class IndexDesc(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("device", C.c_int32), ("algo", C.c_int32),
                ("value_type", C.c_int32), ("metric", C.c_int32), ("num_vectors", C.c_int32),
                ("dim", C.c_int32), ("graph_degree", C.c_int32), ("vectors", C.c_void_p),
                ("graph", C.c_void_p), ("tree_num", C.c_int32), ("node_count", C.c_int32),
                ("tree_starts", C.c_void_p), ("tree_nodes", C.c_void_p), ("deleted", C.c_void_p),
                ("num_deleted", C.c_int32), ("id_offset", C.c_int32)]


class SearchOptions(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("search_deleted", C.c_int32), ("max_check", C.c_int32),
                ("allowed", C.c_void_p)]


class SptagB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("sptag_b200 error 0x%04x: %s" % (code, msg))
        self.code = code


_lib = None


def lib():
    """Load libsptag_b200.so; raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SptagB200Error(1, "CUDA library %s is missing -- build it with __graft_entry__.build(); "
                                    "there is no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.sptag_b200_create.argtypes = [C.POINTER(IndexDesc), C.POINTER(C.c_void_p)]
        L.sptag_b200_load.argtypes = [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_set_quantizer.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.sptag_b200_quantize.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
        L.sptag_b200_destroy.argtypes = [C.c_void_p]
        L.sptag_b200_destroy.restype = None
        L.sptag_b200_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.sptag_b200_get_param.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int32]
        L.sptag_b200_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_search_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(SearchOptions), C.c_void_p,
                                           C.c_void_p, C.c_void_p]
        L.sptag_b200_iterator_open_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_refine_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sptag_b200_refine_schedule.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_float, C.c_float]
        L.sptag_b200_rebuild_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.sptag_b200_group_create.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_group_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.sptag_b200_group_destroy.argtypes = [C.c_void_p]
        L.sptag_b200_group_destroy.restype = None
        L.sptag_b200_search_filtered.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                                 C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_search_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_distance_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
        L.sptag_b200_merge_topk.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_refine_graph.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.sptag_b200_get_graph.argtypes = [C.c_void_p, C.c_void_p]
        L.sptag_b200_graph_degree.argtypes = [C.c_void_p]
        L.sptag_b200_iterator_open.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_iterator_next.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_iterator_next_from_nearest.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_iterator_close.argtypes = [C.c_void_p]
        L.sptag_b200_iterator_close.restype = None
        L.sptag_b200_add.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
        L.sptag_b200_delete.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
        L.sptag_b200_delete_vectors.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.sptag_b200_save.argtypes = [C.c_void_p, C.c_char_p]
        L.sptag_b200_num_deleted.argtypes = [C.c_void_p]
        L.sptag_b200_last_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        L.sptag_b200_launch_count.restype = C.c_int64
        for f in ("num_vectors", "dim", "value_type", "metric", "algo"):
            getattr(L, "sptag_b200_" + f).argtypes = [C.c_void_p]
        L.sptag_b200_last_error.restype = C.c_char_p
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise SptagB200Error(rc, lib().sptag_b200_last_error().decode(errors="replace"))


class B200Index:
    """Handle to a device-resident index (the product side of VectorIndex for the search path)."""

    def __init__(self, handle):
        self._h = C.c_void_p(handle)

    # -- construction ---------------------------------------------------------------------------
    @classmethod
    def load(cls, folder, device=-1, id_offset=0):
        """VectorIndex::LoadIndex(folder) for the search path."""
        h = C.c_void_p()
        _check(lib().sptag_b200_load(os.fsencode(folder), device, id_offset, C.byref(h)))
        return cls(h.value)

    @classmethod
    def create(cls, *, algo, value_type, metric, vectors, graph, tree_starts, tree_nodes, deleted=None,
               num_deleted=0, device=-1, id_offset=0):
        vectors = np.ascontiguousarray(vectors)
        graph = np.ascontiguousarray(graph, dtype=np.int32)
        tree_starts = np.ascontiguousarray(tree_starts, dtype=np.int32)
        tree_nodes = np.ascontiguousarray(tree_nodes)
        d = IndexDesc()
        d.struct_size = C.sizeof(IndexDesc)
        d.device = device
        d.algo, d.value_type, d.metric = algo, value_type, metric
        d.num_vectors, d.dim = vectors.shape
        d.graph_degree = graph.shape[1]
        d.vectors = vectors.ctypes.data
        d.graph = graph.ctypes.data
        d.tree_num = tree_starts.shape[0]
        d.node_count = tree_nodes.shape[0]
        d.tree_starts = tree_starts.ctypes.data
        d.tree_nodes = tree_nodes.ctypes.data
        if deleted is not None and num_deleted > 0:
            deleted = np.ascontiguousarray(deleted, dtype=np.int8)
            d.deleted = deleted.ctypes.data
            d.num_deleted = num_deleted
        d.id_offset = id_offset
        h = C.c_void_p()
        _check(lib().sptag_b200_create(C.byref(d), C.byref(h)))
        return cls(h.value)

    def close(self):
        if self._h:
            lib().sptag_b200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- facts / parameters ---------------------------------------------------------------------
    @property
    def num_vectors(self):
        return lib().sptag_b200_num_vectors(self._h)

    @property
    def dim(self):
        return lib().sptag_b200_dim(self._h)

    @property
    def metric(self):
        return lib().sptag_b200_metric(self._h)

    def set_param(self, name, value):
        """VectorIndex::SetParameter (same names as the reference's ini file)."""
        _check(lib().sptag_b200_set_param(self._h, name.encode(), str(value).encode()))

    def set_quantizer(self, blob):
        """VectorIndex::LoadQuantizer: blob = bytes of a reference quantizer file."""
        buf = (C.c_char * len(blob)).from_buffer_copy(blob)
        _check(lib().sptag_b200_set_quantizer(self._h, buf, len(blob)))

    def quantize(self, raw, m):
        """VectorIndex::QuantizeVector: raw vectors -> [n, m] uint8 codes."""
        raw = np.ascontiguousarray(raw)
        out = np.empty((raw.shape[0], m), np.uint8)
        _check(lib().sptag_b200_quantize(self._h, raw.ctypes.data, raw.shape[0], out.ctypes.data))
        return out

    def get_param(self, name):
        buf = C.create_string_buffer(64)
        _check(lib().sptag_b200_get_param(self._h, name.encode(), buf, 64))
        return buf.value.decode()

    # -- search ---------------------------------------------------------------------------------
    def search(self, queries, k, want_stats=False, out_ids=None, out_dists=None, search_deleted=None, max_check=0,
               allowed=None):
        """VectorIndex::SearchIndex(batch) with HOST buffers (numpy or pinned torch memory viewed as numpy).
        search_deleted / max_check / allowed: the per-call arguments (sptag_b200_search_ex); all None/0 = sptag_b200_search."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = out_ids if out_ids is not None else np.empty((nq, k), np.int32)
        dists = out_dists if out_dists is not None else np.empty((nq, k), np.float32)
        stats = np.zeros((nq, STATS_PER_QUERY), np.int32) if want_stats else None
        if search_deleted is None and not max_check and allowed is None:
            _check(lib().sptag_b200_search(self._h, queries.ctypes.data, nq, k, ids.ctypes.data, dists.ctypes.data,
                                           stats.ctypes.data if want_stats else None))
        else:
            if allowed is not None:
                allowed = np.ascontiguousarray(allowed, dtype=np.uint8)
            o = SearchOptions(C.sizeof(SearchOptions), 1 if search_deleted else 0, int(max_check),
                              allowed.ctypes.data if allowed is not None else None)
            _check(lib().sptag_b200_search_ex(self._h, queries.ctypes.data, nq, k, C.byref(o), ids.ctypes.data,
                                              dists.ctypes.data, stats.ctypes.data if want_stats else None))
        return (ids, dists, stats) if want_stats else (ids, dists)

    def search_filtered(self, queries, k, allowed, max_check=0, want_stats=False):
        """VectorIndex::SearchIndexWithFilter for a batch; allowed = uint8 [N], 0 = filtered out."""
        queries = np.ascontiguousarray(queries)
        allowed = np.ascontiguousarray(allowed, dtype=np.uint8)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        stats = np.zeros((nq, STATS_PER_QUERY), np.int32) if want_stats else None
        _check(lib().sptag_b200_search_filtered(self._h, queries.ctypes.data, nq, k, allowed.ctypes.data, max_check,
                                                ids.ctypes.data, dists.ctypes.data,
                                                stats.ctypes.data if want_stats else None))
        return (ids, dists, stats) if want_stats else (ids, dists)

    def refine_search(self, queries, k, search_deleted=False):
        """VectorIndex::RefineSearchIndex for a batch of host query vectors (MaxCheckForRefineGraph, searchDuplicated = false)."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        _check(lib().sptag_b200_refine_search(self._h, queries.ctypes.data, nq, k, 1 if search_deleted else 0,
                                              ids.ctypes.data, dists.ctypes.data))
        return ids, dists

    def search_device(self, d_queries_ptr, nq, k, d_ids_ptr, d_dists_ptr, d_stats_ptr=0, stream=0):
        """Same call with device pointers (e.g. torch tensor .data_ptr()), stream-ordered, no sync."""
        _check(lib().sptag_b200_search_device(self._h, d_queries_ptr, nq, k, d_ids_ptr, d_dists_ptr,
                                              d_stats_ptr or None, stream or None))

    def refine_graph(self, cef, first=0, num=None, neighborhood=None, rng_factor=1.0, install=False,
                     want_rows=True, want_results=False):
        """One NeighborhoodGraph::RefineNode pass (RefineSearchIndex + RebuildNeighbors) on the device.
        -> rows [num, neighborhood] (or None), and with want_results also the (ids, dists) refine-search lists."""
        num = self.num_vectors - first if num is None else num
        neighborhood = self.graph_degree if neighborhood is None else neighborhood
        rows = np.empty((num, neighborhood), np.int32) if want_rows else None
        ids = np.empty((num, cef + 1), np.int32) if want_results else None
        dists = np.empty((num, cef + 1), np.float32) if want_results else None
        _check(lib().sptag_b200_refine_graph(self._h, first, num, cef, neighborhood, rng_factor,
                                             rows.ctypes.data if want_rows else None,
                                             ids.ctypes.data if want_results else None,
                                             dists.ctypes.data if want_results else None, 1 if install else 0))
        return (rows, ids, dists) if want_results else rows

    def refine_schedule(self, refine_iterations=2, cef=1000, cef_scale=2.0, neighborhood=32, neighborhood_scale=2.0,
                        rng_factor=1.0):
        """NeighborhoodGraph::RefineGraph (NeighborhoodGraph.h:460-492) on the device; the graph is replaced in place."""
        _check(lib().sptag_b200_refine_schedule(self._h, refine_iterations, cef, cef_scale, neighborhood,
                                                neighborhood_scale, rng_factor))

    def rebuild_graph(self, install=False):
        """NeighborhoodGraph::RebuildGraph (EnableRebuild's in-degree repair, NeighborhoodGraph.h:404-456) in its
        single-thread order; the index's rows must hold 2 x N candidates.  -> new rows [n, N]."""
        rows = np.empty((self.num_vectors, self.graph_degree // 2), np.int32)
        _check(lib().sptag_b200_rebuild_graph(self._h, rows.ctypes.data, 1 if install else 0))
        return rows

    @property
    def graph_degree(self):
        return lib().sptag_b200_graph_degree(self._h)

    def get_graph(self):
        g = np.empty((self.num_vectors, self.graph_degree), np.int32)
        _check(lib().sptag_b200_get_graph(self._h, g.ctypes.data))
        return g

    def iterators(self, queries, search_deleted=None):
        """VectorIndex::GetIterator for every query of a batch -> B200Iterators (next(batch) / close())."""
        return B200Iterators(self, queries, search_deleted)

    def save_graph(self, path):
        """NeighborhoodGraph::SaveGraph (NeighborhoodGraph.h:606-615): int32 rows, int32 cols, rows x cols int32 --
        the index's current (e.g. device-refined) graph as a graph.bin the reference's LoadIndex reads."""
        g = self.get_graph()
        with open(path, "wb") as f:
            np.array([g.shape[0], g.shape[1]], np.int32).tofile(f)
            g.tofile(f)
        return g

    # -- mutation -------------------------------------------------------------------------------
    def add(self, vectors, normalized=False):
        """VectorIndex::AddIndex: appends the rows and links them into the graph on the device -> the first new id."""
        vectors = np.ascontiguousarray(vectors)
        first = C.c_int32()
        _check(lib().sptag_b200_add(self._h, vectors.ctypes.data, vectors.shape[0], vectors.shape[1],
                                    1 if normalized else 0, C.byref(first)))
        return first.value

    def delete(self, ids):
        """VectorIndex::DeleteIndex(id) per id -> int32 ErrorCodes (0 Success, 0x14 VectorNotFound)."""
        ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
        codes = np.empty(ids.shape[0], np.int32)
        _check(lib().sptag_b200_delete(self._h, ids.ctypes.data, ids.shape[0], codes.ctypes.data))
        return codes

    def delete_vectors(self, vectors):
        """VectorIndex::DeleteIndex(vectors, num) in its single-thread order."""
        vectors = np.ascontiguousarray(vectors)
        _check(lib().sptag_b200_delete_vectors(self._h, vectors.ctypes.data, vectors.shape[0]))

    def save(self, folder):
        """VectorIndex::SaveIndex(folder): a folder both the reference's LoadIndex and B200Index.load read."""
        _check(lib().sptag_b200_save(self._h, os.fsencode(folder)))

    @property
    def num_deleted(self):
        return lib().sptag_b200_num_deleted(self._h)

    def distance_batch(self, queries, ids):
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty(ids.shape, np.float32)
        _check(lib().sptag_b200_distance_batch(self._h, queries.ctypes.data, queries.shape[0], ids.ctypes.data,
                                               ids.shape[1], out.ctypes.data))
        return out

    def last_kernel_ms(self):
        ms = C.c_float()
        _check(lib().sptag_b200_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value


class B200Iterators:
    """A batch of ResultIterators (ResultIterator.cpp): one resumable search per query, state resident in HBM."""

    def __init__(self, index, queries, search_deleted=None):
        queries = np.ascontiguousarray(queries)
        self.index = index           # the handle must outlive the iterators
        self.nq = queries.shape[0]
        h = C.c_void_p()
        if search_deleted is None:
            _check(lib().sptag_b200_iterator_open(index._h, queries.ctypes.data, self.nq, C.byref(h)))
        else:
            _check(lib().sptag_b200_iterator_open_ex(index._h, queries.ctypes.data, self.nq, 1 if search_deleted else 0,
                                                     C.byref(h)))
        self._it = h

    def next(self, batch):
        """ResultIterator::Next(batch) for every query -> (counts [nq], ids [nq, batch], dists [nq, batch], relaxed [nq])."""
        ids = np.empty((self.nq, batch), np.int32)
        dists = np.empty((self.nq, batch), np.float32)
        counts = np.empty(self.nq, np.int32)
        relaxed = np.empty(self.nq, np.uint8)
        _check(lib().sptag_b200_iterator_next(self._it, batch, ids.ctypes.data, dists.ctypes.data, counts.ctypes.data,
                                              relaxed.ctypes.data))
        return counts, ids, dists, relaxed.astype(bool)

    def next_from_nearest(self, k):
        """SearchIndexIterativeFromNeareast for every query -> (found [nq] bool, ids [nq, k], dists [nq, k])."""
        ids = np.empty((self.nq, k), np.int32)
        dists = np.empty((self.nq, k), np.float32)
        found = np.empty(self.nq, np.uint8)
        _check(lib().sptag_b200_iterator_next_from_nearest(self._it, k, ids.ctypes.data, dists.ctypes.data,
                                                           found.ctypes.data))
        return found.astype(bool), ids, dists

    def close(self):
        if self._it:
            lib().sptag_b200_iterator_close(self._it)
            self._it = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200ShardGroup:
    """Vector-partition shards of one process (sptag_b200_group_*): `shards` are B200Index objects, one per partition."""

    def __init__(self, shards):
        self.shards = list(shards)   # keep the handles alive
        arr = (C.c_void_p * len(self.shards))(*[s._h for s in self.shards])
        g = C.c_void_p()
        _check(lib().sptag_b200_group_create(arr, len(self.shards), C.byref(g)))
        self._g = g

    def search(self, queries, k):
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        _check(lib().sptag_b200_group_search(self._g, queries.ctypes.data, nq, k, ids.ctypes.data, dists.ctypes.data))
        return ids, dists

    def close(self):
        if self._g:
            lib().sptag_b200_group_destroy(self._g)
            self._g = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def merge_topk(device, d_ids_ptr, d_dists_ptr, num_lists, nq, k, d_out_ids_ptr, d_out_dists_ptr, stream=0):
    _check(lib().sptag_b200_merge_topk(device, d_ids_ptr, d_dists_ptr, num_lists, nq, k, d_out_ids_ptr,
                                       d_out_dists_ptr, stream or None))


def launch_count():
    return int(lib().sptag_b200_launch_count())
