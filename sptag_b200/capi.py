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
# multi_scan stats per query: rounds, ids seen, consecutive drops at the end, why it ended (MS_END_EXHAUSTED + i: index i)
MS_ROUNDS, MS_SEEN, MS_DROPS, MS_END = range(4)
MS_END_DROPS, MS_END_LIMIT, MS_END_EXHAUSTED = 0, 1, 2
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
    "sptag_b200_num_deleted", "sptag_b200_spann_load", "sptag_b200_spann_destroy", "sptag_b200_spann_search",
    "sptag_b200_spann_set_param", "sptag_b200_spann_get_param", "sptag_b200_spann_iterator_open",
    "sptag_b200_spann_iterator_next", "sptag_b200_spann_iterator_close", "sptag_b200_multi_scan",
    "sptag_b200_spann_build", "sptag_b200_debug_kernel_for", "sptag_b200_spann_load_ex", "sptag_b200_spann_cache_warm",
    "sptag_b200_spann_cache_lists", "sptag_b200_spann_build_ex", "sptag_b200_spann_group_load",
    "sptag_b200_spann_group_member", "sptag_b200_spann_group_set_param", "sptag_b200_spann_group_search",
    "sptag_b200_spann_group_cache_warm", "sptag_b200_spann_group_cache_lists", "sptag_b200_spann_group_destroy",
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


class SpannLoadOptions(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("posting_placement", C.c_int32)]


class SpannBuildOptions(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("device_budget_bytes", C.c_int64)]


# sptag_b200_spann_load_ex's posting_placement (SPTAG_B200_POSTINGS_*)
POSTING_PLACEMENTS = {"auto": 0, "device": 1, "host": 2, "file": 3}


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
        L.sptag_b200_debug_kernel_for.argtypes = [C.c_int32] * 11 + [C.c_char_p, C.c_int32]
        L.sptag_b200_spann_load.argtypes = [C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_spann_load_ex.argtypes = [C.c_char_p, C.c_int32, C.POINTER(SpannLoadOptions), C.POINTER(C.c_void_p)]
        L.sptag_b200_spann_destroy.argtypes = [C.c_void_p]
        L.sptag_b200_spann_destroy.restype = None
        L.sptag_b200_spann_build.argtypes = [C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_void_p]
        L.sptag_b200_spann_build_ex.argtypes = [C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                C.POINTER(SpannBuildOptions), C.c_void_p]
        L.sptag_b200_spann_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.sptag_b200_spann_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.sptag_b200_spann_get_param.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int32]
        L.sptag_b200_spann_cache_warm.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                                  C.POINTER(C.c_int32)]
        L.sptag_b200_spann_cache_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.sptag_b200_spann_iterator_open.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_spann_iterator_next.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p]
        L.sptag_b200_spann_iterator_close.argtypes = [C.c_void_p]
        L.sptag_b200_spann_iterator_close.restype = None
        L.sptag_b200_spann_group_load.argtypes = [C.c_char_p, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_spann_group_member.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.sptag_b200_spann_group_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        L.sptag_b200_spann_group_search.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]
        L.sptag_b200_spann_group_cache_warm.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                                        C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        L.sptag_b200_spann_group_cache_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.sptag_b200_spann_group_destroy.argtypes = [C.c_void_p]
        L.sptag_b200_spann_group_destroy.restype = None
        L.sptag_b200_multi_scan.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(C.c_void_p), C.c_void_p, C.c_int32,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
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
        buf = C.create_string_buffer(256)
        _check(lib().sptag_b200_get_param(self._h, name.encode(), buf, 256))
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


FAMILY_SEARCH, FAMILY_ITERATE, FAMILY_NEAREST_FIRST = 0, 1, 2


def debug_kernel_for(*, value_type, metric, algo, dim, simd_width=16, enable_bfs=0, row_sketch=0, quantized=False,
                     mres_cap, slots=0, family=FAMILY_SEARCH):
    """The kernel instantiation the selectors pick for these launch inputs (sptag_b200_debug_kernel_for), as the name
    B200.LastSearchKernel reports; None when no kernel serves that m_Results capacity.  Needs no GPU."""
    buf = C.create_string_buffer(256)
    rc = lib().sptag_b200_debug_kernel_for(value_type, metric, algo, dim, simd_width, enable_bfs, row_sketch,
                                           1 if quantized else 0, mres_cap, slots, family, buf, 256)
    if rc == 0x13:  # LackOfInputs
        return None
    _check(rc)
    return buf.value.decode()


class B200SpannIndex:
    """Handle to a SPANN index whose head lives in HBM and whose posting lists live in HBM, in pinned host memory
    (posting_placement="host") or in their posting files (posting_placement="file") (SPANN::Index<T>: LoadIndex,
    SearchIndex)."""

    STATS_PER_QUERY = 3  # postings scanned, list elements read, distances computed

    def __init__(self, handle, group=None):
        self._h = C.c_void_p(handle)
        self._group = group  # a group member's owner (B200SpannGroup): kept alive, and close() does not destroy

    @classmethod
    def load(cls, folder, device=-1, posting_placement=None):
        """VectorIndex::LoadIndex(folder) for a SPANN folder.  posting_placement: None (the posting lists in HBM, as
        sptag_b200_spann_load), or "auto", "device", "host" or "file" (sptag_b200_spann_load_ex: "host" keeps them in
        pinned host memory and gathers each batch's lists into HBM; "file" leaves them in the posting files and reads
        each batch's lists from there into HBM, with the same stages, rounds and results as "host" (B200.LastReadBytes:
        the file bytes the last call read); "auto" picks HBM when they fit)."""
        h = C.c_void_p()
        if posting_placement is None:
            _check(lib().sptag_b200_spann_load(os.fsencode(folder), device, C.byref(h)))
        else:
            if posting_placement not in POSTING_PLACEMENTS:
                raise ValueError("posting_placement %r: one of %s" % (posting_placement, sorted(POSTING_PLACEMENTS)))
            o = SpannLoadOptions(C.sizeof(SpannLoadOptions), POSTING_PLACEMENTS[posting_placement])
            _check(lib().sptag_b200_spann_load_ex(os.fsencode(folder), device, C.byref(o), C.byref(h)))
        return cls(h.value)

    BUILD_STATS = ("searched", "rng_rejected", "edges_before_cut", "edges_after_cut", "search_us", "rng_us", "sort_us",
                   "write_us")
    # sptag_b200_spann_build_ex's: BUILD_STATS, the path (0 resident, 1 streamed), the row batches, the edge groups and
    # the bytes copied host to device
    BUILD_STATS_EX = BUILD_STATS + ("streamed", "row_batches", "edge_groups", "h2d_bytes")

    @classmethod
    def build(cls, folder, vectors, normalized=False, device=-1, stats=None, budget_bytes=None):
        """The SSD stage of SPANN::Index::BuildIndex (SelectHead and BuildHead off) on the device: writes the posting
        files of `folder`, whose head is already built, from HOST vectors (row i is vector id i), and returns
        load(folder, device).  budget_bytes: None (sptag_b200_spann_build: rows and edges in HBM), or the device bytes
        the build may use (sptag_b200_spann_build_ex, -1: free HBM less 1 GB), which streams rows and edges from host
        memory when they do not fit.  If `stats` is a dict it receives BUILD_STATS, or BUILD_STATS_EX with a budget."""
        vectors = np.ascontiguousarray(vectors)
        args = (os.fsencode(folder), vectors.ctypes.data, vectors.shape[0], vectors.shape[1] if vectors.ndim == 2 else 0,
                int(bool(normalized)), device)
        if budget_bytes is None:
            names = cls.BUILD_STATS
            out = np.zeros(len(names), np.int64)
            _check(lib().sptag_b200_spann_build(*args, out.ctypes.data))
        else:
            names = cls.BUILD_STATS_EX
            out = np.zeros(len(names), np.int64)
            o = SpannBuildOptions(C.sizeof(SpannBuildOptions), int(budget_bytes))
            _check(lib().sptag_b200_spann_build_ex(*args, C.byref(o), out.ctypes.data))
        if stats is not None:
            stats.update(zip(names, out.tolist()))
        return cls.load(folder, device)

    def close(self):
        if self._h:
            if self._group is None:
                lib().sptag_b200_spann_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_param(self, name, value):
        """SearchInternalResultNum, MaxDistRatio, SearchPostingPageLimit, MaxCheck and EnableADC (the head's)."""
        _check(lib().sptag_b200_spann_set_param(self._h, name.encode(), str(value).encode()))

    def get_param(self, name):
        buf = C.create_string_buffer(256)  # room for B200.LastPostingKernel's kernel names
        _check(lib().sptag_b200_spann_get_param(self._h, name.encode(), buf, 256))
        return buf.value.decode()

    def search(self, queries, k, want_stats=False):
        """SPANN::Index::SearchIndex for a batch of HOST queries: ids [nq, k], dists [nq, k] (and stats [nq, 3]).
        On a quantized index the queries are raw vectors of the quantizer's reconstruct type and dimension."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        stats = np.zeros((nq, self.STATS_PER_QUERY), np.int32) if want_stats else None
        _check(lib().sptag_b200_spann_search(self._h, queries.ctypes.data, nq, k, ids.ctypes.data, dists.ctypes.data,
                                             stats.ctypes.data if want_stats else None))
        return (ids, dists, stats) if want_stats else (ids, dists)

    def iterators(self, queries):
        """SPANN::Index::GetIterator for a batch of HOST queries, one iterator per query."""
        return B200SpannIterators(self, queries)

    def cache_warm(self, queries, budget_bytes=-1):
        """On a posting_placement="host" or "file" handle: caches in HBM the lists the sample HOST queries choose most
        often, as many as fit budget_bytes (-1: free HBM less 1 GB), and returns them as int32 list ids in rank order
        (sptag_b200_spann_cache_warm; a "file" handle reads the taken lists from the posting files here, once).
        cache_lists(ids) installs the same set again later."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        # a query chooses at most SearchInternalResultNum lists, so that many per query bound the taken set
        cap = max(nq * max(int(self.get_param("SearchInternalResultNum")), 1), 1)
        out = np.empty(cap, np.int32)
        n = C.c_int32()
        _check(lib().sptag_b200_spann_cache_warm(self._h, queries.ctypes.data, nq, int(budget_bytes), out.ctypes.data,
                                                 cap, C.byref(n)))
        if n.value > cap:  # SearchInternalResultNum was raised during the call
            raise RuntimeError("cache_warm installed a cache of %d lists, but only the first %d ids were returned; read "
                               "them again with a second cache_warm at the same budget" % (n.value, cap))
        return out[:n.value].copy()

    def cache_lists(self, lists):
        """On a posting_placement="host" or "file" handle: caches exactly these list ids in HBM (empty: releases the cache;
        sptag_b200_spann_cache_lists)."""
        lists = np.ascontiguousarray(lists, np.int32)
        _check(lib().sptag_b200_spann_cache_lists(self._h, lists.ctypes.data, len(lists)))


class B200SpannIterators:
    """A batch of SPANN ResultIterators (SPANNResultIterator.h): one resumable, deduplicated stream of posting elements per
    query, state resident in HBM."""

    def __init__(self, index, queries):
        queries = np.ascontiguousarray(queries)
        self.index = index           # the handle must outlive the iterators
        self.nq = queries.shape[0]
        h = C.c_void_p()
        _check(lib().sptag_b200_spann_iterator_open(index._h, queries.ctypes.data, self.nq, C.byref(h)))
        self._it = h

    def next(self, batch):
        """Next(batch) for every query -> (counts [nq], ids [nq, batch], dists [nq, batch], relaxed [nq] bool)."""
        ids = np.empty((self.nq, batch), np.int32)
        dists = np.empty((self.nq, batch), np.float32)
        counts = np.empty(self.nq, np.int32)
        relaxed = np.empty(self.nq, np.uint8)
        _check(lib().sptag_b200_spann_iterator_next(self._it, batch, ids.ctypes.data, dists.ctypes.data,
                                                    counts.ctypes.data, relaxed.ctypes.data))
        return counts, ids, dists, relaxed.astype(bool)

    def close(self):
        if self._it:
            lib().sptag_b200_spann_iterator_close(self._it)
            self._it = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class B200SpannGroup:
    """A SPANN index on several GPUs of one host (sptag_b200_spann_group_*): one pinned host copy of the posting lists
    that every member maps, one member handle per device, and an HBM cache spread over the members so that each list is
    cached at most once; a member gathers a list another member caches from that member's HBM."""

    def __init__(self, handle, n):
        self._h = C.c_void_p(handle)
        self.members = []
        for i in range(n):
            m = C.c_void_p()
            _check(lib().sptag_b200_spann_group_member(self._h, i, C.byref(m)))
            self.members.append(B200SpannIndex(m.value, group=self))

    @classmethod
    def load(cls, folder, devices):
        """Loads `folder` once into pinned host memory and opens one member per entry of `devices` (CUDA ordinals; one
        may repeat)."""
        devs = np.ascontiguousarray(devices, np.int32)
        h = C.c_void_p()
        _check(lib().sptag_b200_spann_group_load(os.fsencode(folder), devs.ctypes.data if len(devs) else None, len(devs),
                                                 C.byref(h)))
        return cls(h.value, len(devs))

    def close(self):
        if self._h:
            for m in self.members:
                m._h = C.c_void_p()
            lib().sptag_b200_spann_group_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_param(self, name, value):
        """set_param on every member"""
        _check(lib().sptag_b200_spann_group_set_param(self._h, name.encode(), str(value).encode()))

    def search(self, queries, k, want_stats=False):
        """B200SpannIndex.search with the batch split into one contiguous slice per member: ids [nq, k], dists [nq, k]
        (and stats [nq, 3] int64)."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        ids = np.empty((nq, k), np.int32)
        dists = np.empty((nq, k), np.float32)
        stats = np.zeros((nq, B200SpannIndex.STATS_PER_QUERY), np.int64) if want_stats else None
        _check(lib().sptag_b200_spann_group_search(self._h, queries.ctypes.data, nq, k, ids.ctypes.data,
                                                   dists.ctypes.data, stats.ctypes.data if want_stats else None))
        return (ids, dists, stats) if want_stats else (ids, dists)

    def cache_warm(self, queries, budget_bytes=-1):
        """Ranks the lists as B200SpannIndex.cache_warm does and gives each, in rank order, to the member with the most
        budget left that holds it whole (budget_bytes per member; -1: each member's free HBM less 1 GB); installs them and
        returns (lists, owners), int32, in rank order."""
        queries = np.ascontiguousarray(queries)
        nq = queries.shape[0]
        cap = max(nq * max(int(self.members[0].get_param("SearchInternalResultNum")), 1), 1)
        lists = np.empty(cap, np.int32)
        owners = np.empty(cap, np.int32)
        n = C.c_int32()
        _check(lib().sptag_b200_spann_group_cache_warm(self._h, queries.ctypes.data, nq, int(budget_bytes),
                                                       lists.ctypes.data, owners.ctypes.data, cap, C.byref(n)))
        if n.value > cap:  # SearchInternalResultNum was raised during the call
            raise RuntimeError("cache_warm installed %d lists, but only the first %d were returned" % (n.value, cap))
        return lists[:n.value].copy(), owners[:n.value].copy()

    def cache_lists(self, lists, owners):
        """Caches list lists[i] on member owners[i] (empty: releases every member's cache)."""
        lists = np.ascontiguousarray(lists, np.int32)
        owners = np.ascontiguousarray(owners, np.int32)
        if lists.shape != owners.shape:
            raise ValueError("one owner per list")
        _check(lib().sptag_b200_spann_group_cache_lists(self._h, lists.ctypes.data, owners.ctypes.data, len(lists)))


def multi_scan(indexes, queries, k, *, term_cond, search_limit, weights=None, want_stats=False):
    """MultiIndexScan (Init + Next until false) for a batch: the k ids with the smallest weighted sum of per-index
    distances over B200Index handles that hold the same ids.  queries[i]: [nq x dim_i] of index i's value type;
    weights: one float per index or None for the plain sum.  term_cond / search_limit as the reference's termCondVal /
    searchLimit, required as the reference has no defaults (negative: never ends that way; with both negative every
    query runs until an iterator is exhausted).  -> (ids [nq x k], scores [nq x k], counts [nq][, stats [nq x 4]])"""
    n = len(indexes)
    qs = [np.ascontiguousarray(q) for q in queries]
    if len(qs) != n or n == 0:
        raise ValueError("one query array per index")
    nq = qs[0].shape[0]
    if any(q.shape[0] != nq for q in qs):
        raise ValueError("every query array needs the same number of rows")
    hs = (C.c_void_p * n)(*[ix._h.value for ix in indexes])
    qp = (C.c_void_p * n)(*[q.ctypes.data for q in qs])
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    if w is not None and w.shape != (n,):
        raise ValueError("one weight per index")
    ids = np.empty((nq, k), np.int32)
    scores = np.empty((nq, k), np.float32)
    counts = np.empty(nq, np.int32)
    stats = np.empty((nq, 4), np.int32) if want_stats else None
    _check(lib().sptag_b200_multi_scan(hs, n, qp, None if w is None else w.ctypes.data, nq, k, term_cond, search_limit,
                                       ids.ctypes.data, scores.ctypes.data, counts.ctypes.data,
                                       None if stats is None else stats.ctypes.data))
    return (ids, scores, counts, stats) if want_stats else (ids, scores, counts)
