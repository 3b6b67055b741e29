/* sptag_b200.h -- C ABI of libsptag_b200: the H100-native drop-in for SPTAG's batched in-memory
 * search path (BKT/KDT seed lookup -> RNG best-first expansion -> DistanceUtils inner loop).
 *
 * Every entry point names the reference interface it replaces (paths relative to
 * /root/reference/AnnService).  Plain pointers and sizes only; no C++ or torch types cross this
 * boundary.  Return values are the reference's ErrorCode numerics
 * (inc/Core/DefinitionList.h:54-68): 0 Success, 1 Fail, 0x12 MemoryOverFlow, 0x13 LackOfInputs,
 * 0x15 EmptyIndex, 0x17 DimensionSizeMismatch, 0x02 FailedOpenFile, 0x10 ParamNotFound,
 * 0x11 FailedParseValue.
 *
 * There is NO CPU fallback: every search call runs the sm_90a kernels or fails.
 */
#ifndef SPTAG_B200_H_
#define SPTAG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ErrorCode numerics (inc/Core/DefinitionList.h:54-68) */
#define SPTAG_B200_SUCCESS 0x0000
#define SPTAG_B200_FAIL 0x0001
#define SPTAG_B200_FAILED_OPEN_FILE 0x0002
#define SPTAG_B200_PARAM_NOT_FOUND 0x0010
#define SPTAG_B200_FAILED_PARSE_VALUE 0x0011
#define SPTAG_B200_MEMORY_OVERFLOW 0x0012
#define SPTAG_B200_LACK_OF_INPUTS 0x0013
#define SPTAG_B200_VECTOR_NOT_FOUND 0x0014
#define SPTAG_B200_EMPTY_INDEX 0x0015
#define SPTAG_B200_EMPTY_DATA 0x0016
#define SPTAG_B200_DIMENSION_MISMATCH 0x0017

/* enum orders follow inc/Core/DefinitionList.h:6-9 (VectorValueType), :36-38 (DistCalcMethod),
 * :92-93 (IndexAlgoType) */
#define SPTAG_B200_VT_INT8 0
#define SPTAG_B200_VT_UINT8 1
#define SPTAG_B200_VT_INT16 2
#define SPTAG_B200_VT_FLOAT 3
#define SPTAG_B200_METRIC_L2 0
#define SPTAG_B200_METRIC_COSINE 1
#define SPTAG_B200_METRIC_INNERPRODUCT 2
#define SPTAG_B200_ALGO_BKT 0
#define SPTAG_B200_ALGO_KDT 1

typedef struct sptag_b200_index* sptag_b200_handle;

/* Host-side description of an already-built index: exactly the arrays the reference keeps in
 * BKT::Index<T> / KDT::Index<T> (m_pSamples, m_pGraph, m_pTrees, m_deletedID) and persists as
 * vectors.bin / graph.bin / tree.bin / deletes.bin (Dataset.h:146-180, NeighborhoodGraph.h:606-615,
 * BKTree.h:635-645, KDTree.h:123-133, Labelset.h:78-83).  The library copies everything to HBM;
 * the host arrays may be freed after sptag_b200_create returns. */
typedef struct {
    int32_t struct_size;   /* sizeof(sptag_b200_index_desc), for ABI growth */
    int32_t device;        /* CUDA device ordinal; -1 = current device */
    int32_t algo;          /* SPTAG_B200_ALGO_* */
    int32_t value_type;    /* SPTAG_B200_VT_* (element type T of the index) */
    int32_t metric;        /* SPTAG_B200_METRIC_* */
    int32_t num_vectors;   /* N (Dataset::R()) */
    int32_t dim;           /* Dataset::C() */
    int32_t graph_degree;  /* NeighborhoodSize = graph.bin cols */
    const void* vectors;   /* N x dim, row-major, unpadded (vectors.bin body) */
    const int32_t* graph;  /* N x graph_degree, -1 padded; last slot < -1 = duplicate back-pointer */
    int32_t tree_num;      /* BKTNumber / KDTNumber */
    int32_t node_count;    /* tree node count */
    const int32_t* tree_starts; /* tree_num root indices */
    const void* tree_nodes;     /* BKT: node_count x {centerid, childStart, childEnd} int32 (BKTree.h:25-32);
                                   KDT: node_count x {left, right, split_dim, split_value} (KDTree.h:22-28) */
    const int8_t* deleted; /* N tombstone bytes (1 = deleted) or NULL (Labelset.h:43-57) */
    int32_t num_deleted;   /* Labelset::Count(); 0 disables the tombstone test (BKTIndex.cpp:473) */
    int32_t id_offset;     /* added to every returned id >= 0 (vector-partition shards; 0 otherwise) */
} sptag_b200_index_desc;

/* Per-query work counters; they equal the reference's WorkSpace counters (WorkSpace.h:303-308) and
 * feed the algorithmic-bytes roofline figure (SURVEY.md 8d).  8 x int32 per query. */
#define SPTAG_B200_STATS_PER_QUERY 8
#define SPTAG_B200_ST_CHECKED 0      /* m_iNumberOfCheckedLeaves at exit */
#define SPTAG_B200_ST_TREE_CHECKED 1 /* m_iNumberOfTreeCheckedLeaves (KDT) */
#define SPTAG_B200_ST_NG_LEFT 2      /* m_NGQueue.size() at exit */
#define SPTAG_B200_ST_SPT_LEFT 3     /* m_SPTQueue.size() at exit */
#define SPTAG_B200_ST_NDIST 4        /* distance evaluations D_q */
#define SPTAG_B200_ST_NEXPAND 5      /* graph rows read E_q */
#define SPTAG_B200_ST_NTREE 6        /* tree nodes read Tn_q */
#define SPTAG_B200_ST_FLAGS 7        /* 0 = ok; nonzero = internal error for this query */

/* Replaces: VectorIndex::CreateInstance + LoadIndexData for an index already in host memory
 * (VectorIndex.cpp:566-614, BKTIndex.cpp:85-106). */
int sptag_b200_create(const sptag_b200_index_desc* desc, sptag_b200_handle* out);

/* Replaces: VectorIndex::LoadIndex(folder, index) (VectorIndex.cpp:617-681): parses
 * indexloader.ini and the four binary files of a reference index folder and uploads them. */
int sptag_b200_load(const char* folder, int32_t device, int32_t id_offset, sptag_b200_handle* out);

/* Replaces: VectorIndex::LoadQuantizer / SetQuantizer (VectorIndex.cpp:548-563, BKTIndex.cpp:34-50) for an
 * index whose value type is UInt8 PQ codes.  `blob` is the content of a quantizer file exactly as
 * PQQuantizer::SaveQuantizer / OPQQuantizer::SaveQuantizer write it (PQQuantizer.h:226-239,
 * OPQQuantizer.h:133-147): uint8 quantizer type (1 PQ, 2 OPQ), uint8 reconstruct type, int32 M, int32 Ks,
 * int32 DimPerSubvector, codebooks[M*Ks*Dsub], OPQ only: rotation[(M*Dsub)^2].  Supported: PQQuantizer<float>
 * and OPQQuantizer<T> for every T (its codebooks/rotation are float).  After this call the search entry
 * points take RAW query vectors (M*Dsub elements of the reconstruct type), quantize them on the device
 * exactly like QueryResultSet::SetTarget -> IQuantizer::QuantizeVector (QueryResultSet.h:46-60) and compute
 * distances by SDC table look-ups (PQQuantizer::L2Distance, ADC off = the reference's default).
 * sptag_b200_load calls it automatically when indexloader.ini has a [Quantizer] section. */
int sptag_b200_set_quantizer(sptag_b200_handle h, const void* blob, int64_t blob_bytes);

/* Replaces: VectorIndex::QuantizeVector (VectorIndex.h:146-153): num raw vectors -> num x M code bytes.
 * Host buffers; blocking. */
int sptag_b200_quantize(sptag_b200_handle h, const void* raw_vectors, int32_t num, uint8_t* codes_out);

/* Replaces: VectorIndex destructor. */
void sptag_b200_destroy(sptag_b200_handle h);

/* Replaces: VectorIndex::SetParameter / GetParameter (BKTIndex.cpp:980-1025) for the search-time
 * parameters, same names as the ini file: MaxCheck, MaxCheckForRefineGraph,
 * NumberOfInitialDynamicPivots, NumberOfOtherDynamicPivots,
 * ThresholdOfNumberOfContinuousNoBetterPropagation; EnableBfs (BKT only, any int, default 0: BKTree::m_bfs, the number
 * of breadth-first seeding levels of every search, BKTree.h:703-758; negative values seed breadth-first with no level;
 * read when a search call is made, and by an iterator at its first Next / SearchIndexIterativeFromNeareast call; on a
 * KDT handle it is ParamNotFound, and sptag_b200_load ignores it there); the update parameters AddCEF (500), CEF (1000) and RNGFactor (1.0,
 * a float) used by sptag_b200_add / sptag_b200_delete_vectors; "EnableADC" = VectorIndex::SetQuantizerADC
 * (VectorIndex.h:136-138) for quantized indexes; "SearchDeleted" (0/1) = the handle-wide DEFAULT of the
 * p_searchDeleted argument (the per-call value is sptag_b200_search_options.search_deleted /
 * sptag_b200_iterator_open_ex); the refine pass always runs with 0 like NeighborhoodGraph::RefineNode.  Additional B200 tuning knobs (not in the
 * reference) are prefixed "B200.": B200.QueriesPerSM (query slots per SM, 0 = auto: what registers and shared memory allow;
 * for 512-byte float rows the slot count in [14, 20] that fills the batch's last round best), B200.StageRows, B200.Stages
 * (depth of the row ring; 512-byte float rows run one stage unless 2 is set explicitly at <= 16 slots),
 * B200.NGCacheEntries, B200.SPTCacheEntries (queue entries kept in shared memory, 0 = the slot's spare), B200.SimdWidth (which DistanceUtils summation tree to
 * reproduce bit-exactly -- the reference picks by cpuid, DistanceUtils.h:118-163: 16 = AVX-512 (default; all specialised
 * kernels), 8 = AVX / AVX2, 4 = SSE; 8 and 4 are built for float, int8 and uint8 rows and run the generic-dimension
 * kernels; int16 rows and quantized indexes exist in the AVX-512 form only and return LackOfInputs otherwise), B200.VisitedLog (-1 auto, 0 clear the
 * visited bitmap per query, 1 log the touched words and clear only those: for indexes of tens of millions
 * of vectors), B200.VisitedLogEntries, B200.VisitedSet (-1 auto: the per-slot visited bitmap unless its allocation fails
 * for lack of device memory, then the hashed set; a bitmap size that failed is not tried again until a launch needs a
 * smaller one or B200.VisitedSet is set; 0 bitmap; 1 hashed set: one table of 2^(bits(max(MaxCheck,
 * MaxCheckForRefineGraph)) + 2) entries per query slot, at least 64, independent of the number of vectors; a query that fills half of
 * it is searched again on a bitmap by a second launch on the same stream; results are identical in every mode),
 * B200.VisitedHashEntries (table entries per slot: 0 = the default above, otherwise a power of two in [64, 2^30]).
 * B200.RowSketch (-1 auto, 0 off, 1 on: a 1-byte-per-dimension copy of the rows of a float BKT index, dim + 16 bytes per
 * vector of device memory, built on the device from the rows before the next search; BKT search reads it to prove that
 * m_Results rejects a graph neighbour and then does not fetch that neighbour's row; results and per-query counters are
 * identical in every mode; auto = on for rows of 2 KB or more unless the array does not fit; off with EnableBfs; 1 returns
 * LackOfInputs on KDT, integer and quantized indexes).
 * B200.VisitedSet governs search only.  Iterators: B200.IteratorVisitedSet (-1 auto: a bitmap over the index per open
 * iterator query unless the iterator's bitmaps fail to allocate for lack of device memory, then hashed; 0 bitmap;
 * 1 hashed: per query a hash table that grows as the scan proceeds and becomes a bitmap when it would outgrow one;
 * results are identical in every mode; an open iterator keeps the mode it was opened with),
 * B200.IteratorVisitedHashEntries (initial table entries per query: 0 = the default above, otherwise a power of two in
 * [64, 2^30]; raised to what one search step needs).
 * Read-only: B200.RowsSkipped (graph neighbours whose row the finished searches of this handle did not fetch, summed
 * since the handle was made), B200.LastVisitedOverflows (queries the hashed set handed to the bitmap re-run in the last blocking search
 * call of this handle; 0 on the bitmap), B200.ScratchBytes (device bytes held by the handle's search scratch sets),
 * B200.LastIteratorSuspensions ("step,trees": how often the last iterator call suspended a query at the top of a step /
 * before a tree pop to grow its table), B200.LastIteratorGrowths (tables grown or restarted by that call),
 * B200.LastIteratorVisitedBytes (device bytes of that iterator's visited sets after the call), B200.LastRefineSearchUs
 * and B200.LastRefineRebuildUs (device microseconds of the last sptag_b200_refine_graph call's search and rebuild),
 * B200.LastSearchKernel (the demangled name of the last search, refine or iterator kernel instantiation this handle
 * launched, e.g. "sptag_b200::search_kernel<128, false, 16, false, false, 0, 20>"; empty before the first; the value can
 * be longer than 64 bytes).
 * Names are matched case-insensitively, as the reference's StrEqualIgnoreCase does.  Unknown names are ParamNotFound;
 * writing a read-only name is LackOfInputs. */
int sptag_b200_set_param(sptag_b200_handle h, const char* name, const char* value);
int sptag_b200_get_param(sptag_b200_handle h, const char* name, char* value_out, int32_t capacity);

/* Replaces: VectorIndex::SearchIndex(const void* p_vector, int p_vectorCount, int p_neighborCount,
 * bool p_withMeta, BasicResult* p_results) (VectorIndex.h:103, VectorIndex.cpp:454-463).
 * queries: HOST buffer, num_queries x dim elements of the index value type, row-major, borrowed.
 * out_ids / out_dists: HOST buffers [num_queries x k]; ascending by (dist, id); unfilled slots are
 * id -1 / dist MaxDist (FLT_MAX/10) exactly like a default BasicResult (SearchResult.h:72).
 * out_stats: HOST buffer [num_queries x 8] int32 or NULL.  Blocking.  H2D/D2H copies included. */
int sptag_b200_search(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                      int32_t* out_ids, float* out_dists, int32_t* out_stats);

/* Per-call arguments of the reference's search entry points that are not part of the index state:
 *   search_deleted = p_searchDeleted of SearchIndex(QueryResult&, bool) / SearchIndexWithFilter / GetIterator
 *                    (VectorIndex.h:41-57; dispatch flag BKTIndex.cpp:473, KDTIndex.cpp:260): 1 makes tombstoned
 *                    vectors eligible results;
 *   max_check      = maxCheck of SearchIndexWithFilter (BKTIndex.cpp:622-647): 0 = the index's MaxCheck;
 *   allowed        = filterFunc evaluated once per vector by the caller: HOST buffer, one byte per vector,
 *                    0 = never added to the results (filtered vectors are still traversed); NULL = no filter.
 * They travel with the call, never through the handle, so concurrent callers with different values do not interact. */
typedef struct {
    int32_t struct_size;    /* sizeof(sptag_b200_search_options) */
    int32_t search_deleted;
    int32_t max_check;
    const uint8_t* allowed;
} sptag_b200_search_options;

/* sptag_b200_search with per-call options (NULL = defaults: the handle's "SearchDeleted", the index's MaxCheck, no
 * filter).  Thread-safe: concurrent callers are served from two internal staging sets, so one caller's H2D / D2H copies
 * overlap another caller's kernel; kernels of one handle run one after the other (they share the per-slot scratch). */
int sptag_b200_search_ex(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                         const sptag_b200_search_options* options, int32_t* out_ids, float* out_dists,
                         int32_t* out_stats);

/* Replaces: VectorIndex::SearchIndexWithFilter(QueryResult&, std::function<bool(const ByteArray&)> filterFunc,
 * int maxCheck, bool) (VectorIndex.h:57, BKTIndex.cpp:622-647) for a batch.  The reference evaluates `filterFunc` on
 * the metadata of every vector it is about to add to the results; a device cannot call back into host code, so the
 * caller (or the C++ adapter) evaluates its predicate once per vector into `allowed` (HOST buffer, one byte per
 * vector, 0 = filtered out).  Filtered vectors are still traversed, exactly as in the reference.  max_check: 0 = the
 * index's MaxCheck, otherwise this call's budget.  BKT only ("Not Support Filter on KDT Index!", KDTIndex.cpp:361-365
 * -> Fail). */
int sptag_b200_search_filtered(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                               const uint8_t* allowed, int32_t max_check, int32_t* out_ids, float* out_dists,
                               int32_t* out_stats);

/* Same call with every buffer already resident in HBM on the index's device (device pointers) and
 * stream-ordered on `cuda_stream` (a cudaStream_t; NULL = default stream).  Does not synchronise.  Calls on different
 * streams are safe: all kernels of a handle share its per-slot scratch, so the library orders each launch after the
 * handle's previous one with an event (they do not overlap each other; copies and other work on the streams do). */
int sptag_b200_search_device(sptag_b200_handle h, const void* d_queries, int32_t num_queries, int32_t k,
                             int32_t* d_out_ids, float* d_out_dists, int32_t* d_out_stats,
                             void* cuda_stream);

/* Replaces: the reference's DistanceCalcSelector<T>(method)(query, m_pSamples[id], dim) call
 * (DistanceUtils.h:118-163; call site BKTIndex.cpp:339) for a ragged list of ids per query:
 * out[q*ids_per_query + j] = dist(query_q, vector[ids[q*ids_per_query + j]]) (ids < 0 -> MaxDist).
 * Host buffers; blocking.  Exists so the inner loop can be parity-tested on its own. */
int sptag_b200_distance_batch(sptag_b200_handle h, const void* queries, int32_t num_queries,
                              const int32_t* ids, int32_t ids_per_query, float* out);

/* Replaces: one pass of NeighborhoodGraph::RefineNode(index, node, updateNeighbors=false, searchDeleted=false, CEF)
 * (NeighborhoodGraph.h:534-545, looped by RefineGraph :459-488) over nodes [first_node, first_node+num_nodes):
 *   RefineSearchIndex (BKTIndex.cpp:698-711 / KDTIndex.cpp:367-390): the search kernel with the node's own row as the
 *   query, K = cef+1, MaxCheckForRefineGraph as the budget, searchDuplicated = false;
 *   RelativeNeighborhoodGraph::RebuildNeighbors (RelativeNeighborhoodGraph.h:20-38) with m_iNeighborhoodSize =
 *   neighborhood_size and m_fRNGFactor = rng_factor.
 * Every node is refined against the graph as it is when the call starts (the reference updates rows in place under
 * OpenMP, so its pass depends on thread timing; this is the deterministic double-buffered form).
 * out_graph (host, nullable): [num_nodes x neighborhood_size] new rows, -1 padded, local ids.
 * out_res_ids / out_res_dists (host, nullable): [num_nodes x (cef+1)] the refine-search result lists.
 * install != 0 (needs a full pass): the new rows replace the index's graph on the device -- the index's degree becomes
 * neighborhood_size, which may differ from the current one (RefineGraph's passes run on rows NeighborhoodScale times
 * wider); duplicate-group back-pointers in the last slot are carried over (NeighborhoodGraph.h:395-401).
 * cef <= 2047.  Quantized indexes: as RefineNode does (NeighborhoodGraph.h:538-543), the node's code row is reconstructed,
 * quantized again and searched with that; RebuildNeighbors uses the quantizer's SDC distance; K = cef + 1 <= 1024 there,
 * and ADC must be off (with ADC on the reference's RebuildNeighbors reads a code row as a distance table). */
int sptag_b200_refine_graph(sptag_b200_handle h, int32_t first_node, int32_t num_nodes, int32_t cef,
                            int32_t neighborhood_size, float rng_factor, int32_t* out_graph, int32_t* out_res_ids,
                            float* out_res_dists, int32_t install);

/* Replaces: NeighborhoodGraph::RefineGraph(index) (NeighborhoodGraph.h:460-492), the schedule BuildGraph runs after
 * the initial graph: RefineIterations - 1 full passes with CEF x CEFScale candidates on rows of
 * NeighborhoodSize x NeighborhoodScale entries, then one pass with CEF on rows of NeighborhoodSize entries; every pass
 * is sptag_b200_refine_graph(install = 1) (deterministic double-buffered form, see there).  The index's graph ends with
 * (int)((int)(neighborhood_size * neighborhood_scale) / neighborhood_scale) columns.  The reference's defaults
 * (BKT/ParameterDefinitionList.h): RefineIterations 2, CEF 1000, GraphCEFScale 2, NeighborhoodSize 32,
 * GraphNeighborhoodScale 2, RNGFactor 1.  With EnableRebuild the reference runs the schedule on rows twice as wide
 * (NeighborhoodGraph.h:369) and calls RebuildGraph afterwards: pass 2 x NeighborhoodSize here, then
 * sptag_b200_rebuild_graph. */
int sptag_b200_refine_schedule(sptag_b200_handle h, int32_t refine_iterations, int32_t cef, float cef_scale,
                               int32_t neighborhood_size, float neighborhood_scale, float rng_factor);

/* Replaces: NeighborhoodGraph::RebuildGraph(index) (NeighborhoodGraph.h:404-456), the in-degree repair BuildGraph runs
 * after its refine passes when EnableRebuild is set (:388-391).  The index's graph rows must hold 2 x N candidates
 * (current degree even, N = degree / 2): the first N / 2 stay, the other slots are refilled from entries [N / 2, 2 N) --
 * first those whose target has an in-degree below N / 2, then the earliest others -- in index order, the in-degree array
 * following every change.  The reference's node loop updates that array from all OpenMP threads without synchronisation,
 * so its result depends on thread timing; this call computes its single-thread order (node 0, 1, 2, ...), which is
 * sequential by construction (one warp walks the nodes).
 * out_graph (host, nullable): [n x N] new rows.  install != 0: the rows replace the index's graph (degree becomes N;
 * duplicate-group back-pointers are re-attached to the last slot, NeighborhoodGraph.h:395-401). */
int sptag_b200_rebuild_graph(sptag_b200_handle h, int32_t* out_graph, int32_t install);

/* Replaces: VectorIndex::RefineSearchIndex(QueryResult&, bool p_searchDeleted) (VectorIndex.h:53, BKTIndex.cpp:698-711,
 * KDTIndex.cpp:367-390) for a batch of arbitrary query vectors in HOST memory (element type of the index): the search
 * with MaxCheckForRefineGraph as the budget and searchDuplicated = false; ids are local (no shard offset).  This is the
 * call NeighborhoodGraph::RefineNode makes with a base vector as the target; sptag_b200_refine_graph is the batched
 * form that never leaves the device. */
int sptag_b200_refine_search(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                             int32_t search_deleted, int32_t* out_ids, float* out_dists);

/* The index's current graph rows (NeighborhoodGraph::SaveGraph payload, NeighborhoodGraph.h:606-615):
 * [num_vectors x graph_degree] int32 to a host buffer. */
int sptag_b200_get_graph(sptag_b200_handle h, int32_t* out_graph);
int32_t sptag_b200_graph_degree(sptag_b200_handle h);

/* Replaces: VectorIndex::GetIterator + ResultIterator::Next / Close (VectorIndex.h:43-49, ResultIterator.cpp,
 * BKTIndex.cpp:354-427 SearchIterative, :650-696) for a BATCH of queries -- one resumable search per query.
 *   open:  rents one WorkSpace per query in HBM (visited set, NGQueue, SPTQueue; about N/8 + 8*min(30*MaxCheck, N)
 *          + 8*min(10*MaxCheck, nodes) bytes each) and copies the queries (they need not outlive the call).
 *          MaxCheck / MaxCheckForRefineGraph are sampled here, like the reference's RentWorkSpace.
 *   next:  ResultIterator::Next(batch) for every query: up to `batch` further results per query in pop order, sorted
 *          ascending within the call; out_ids / out_dists are [num_queries x batch] with unfilled slots (-1, MaxDist),
 *          out_counts[q] = resultCount (nullable), out_relaxed_mono[q] = RelaxedMono (nullable).  As in the reference,
 *          the effective batch of a query is capped by the result count of its previous call (ResultIterator.cpp:36-41,
 *          :52), so a batch never grows and an exhausted iterator stays exhausted.  batch <= 1024.
 *   close: returns the work spaces.  The handle must outlive its iterators.
 * BKT without quantizer only; KDT returns Fail like the reference ("ITERATIVE NOT SUPPORT FOR KDT"). */
typedef struct sptag_b200_iterator* sptag_b200_iter;
int sptag_b200_iterator_open(sptag_b200_handle h, const void* queries, int32_t num_queries, sptag_b200_iter* out);
/* GetIterator(p_target, p_searchDeleted): search_deleted 0 / 1, or -1 for the handle's "SearchDeleted" default */
int sptag_b200_iterator_open_ex(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t search_deleted,
                                sptag_b200_iter* out);
int sptag_b200_iterator_next(sptag_b200_iter it, int32_t batch, int32_t* out_ids, float* out_dists,
                             int32_t* out_counts, uint8_t* out_relaxed_mono);
/* Replaces: VectorIndex::SearchIndexIterativeFromNeareast(QueryResult&, WorkSpace*, p_isFirst) (VectorIndex.h:49,
 * BKTIndex.cpp:543-595) for every query of an iterator -- the head-index call of SPANN's iterative search
 * (SPANNIndex.cpp:259-285).  The first call on a freshly opened iterator returns the k nearest by a full search and
 * re-seeds the scan from their graph neighbours; every later call (same k) returns the next k in pop order, sorted.
 * out_ids / out_dists: [num_queries x k], unfilled slots (-1, MaxDist); out_found[q] (nullable) = the reference's bool
 * (first slot holds a vector).  k <= 1024.  Do not mix with sptag_b200_iterator_next on the same iterator before the
 * first call. */
int sptag_b200_iterator_next_from_nearest(sptag_b200_iter it, int32_t k, int32_t* out_ids, float* out_dists,
                                          uint8_t* out_found);
void sptag_b200_iterator_close(sptag_b200_iter it);

/* Vector-partition sharding (SURVEY.md 8e): merges `num_lists` per-shard result lists of a query
 * batch, each [num_queries x k] ascending by (dist,id), into the global top-k with the comparator
 * of QueryResultSet.h:17-26.  All pointers are DEVICE pointers on `device`; lists are laid out
 * [num_lists][num_queries][k] (the layout an all-gather produces).  Stream-ordered. */
int sptag_b200_merge_topk(int32_t device, const int32_t* d_ids, const float* d_dists, int32_t num_lists,
                          int32_t num_queries, int32_t k, int32_t* d_out_ids, float* d_out_dists,
                          void* cuda_stream);

/* Vector-partition shards inside ONE process (the reference's Aggregator deployment, AggregatorService.cpp:215-412,
 * fans each query out to its index servers and merges their lists): every shard is an ordinary handle, normally on
 * its own GPU (sptag_b200_index_desc.device / sptag_b200_load's device) and with its own id_offset.  A group search
 * copies the HOST query batch to every shard's GPU, runs all shard searches concurrently and merges on the first
 * shard's GPU with the comparator of QueryResultSet.h:17-26 -- the merge kernel reads the other GPUs' result lists
 * directly over NVLink peer access, so gather + merge is one kernel and there is no collective library call.
 * (One process per GPU: exchange the lists with NCCL and call sptag_b200_merge_topk -- bench.py's shard leg.)
 * The group borrows the handles; destroy it before them.  num_shards <= 16. */
typedef struct sptag_b200_shard_group* sptag_b200_group;
int sptag_b200_group_create(const sptag_b200_handle* shards, int32_t num_shards, sptag_b200_group* out);
int sptag_b200_group_search(sptag_b200_group g, const void* queries, int32_t num_queries, int32_t k, int32_t* out_ids,
                            float* out_dists);
void sptag_b200_group_destroy(sptag_b200_group g);

/* ---- Index mutation ----
 * Every call below takes the handle's lock and runs after every kernel already launched on the handle, so a concurrent
 * search sees all of a mutation or none of it.  add / delete / delete_vectors return Fail while an iterator of the handle
 * is open (its per-query visited sets are sized to the vector count).  A handle in a shard group may be mutated between
 * group searches: the group reads each shard's current size on every search.  Quantized indexes: add, delete_vectors
 * and save return LackOfInputs; delete by id works on them (it only sets tombstone bytes).
 *
 * Replaces: VectorIndex::DeleteIndex(const SizeType& id) per id, in array order (BKTIndex.cpp:893-899, KDTIndex.cpp:619-625,
 * Labelset::Insert, Labelset.h:59-76).  ids are the ids search returns (id_offset is subtracted).  out_codes (HOST, nullable)
 * [num]: Success, or VectorNotFound for an id that is already deleted or repeated earlier in the array.  An id outside
 * the index gets VectorNotFound; the reference tombstones nothing for it either, but answers Success for ids >= R
 * (InvalidIDBehavior::AlwaysContains, Labelset.h:43-57) and is undefined for negative ids.  The tombstone map is created on the
 * first deletion and the searches test it from then on (Labelset::Count() > 0, BKTIndex.cpp:473). */
int sptag_b200_delete(sptag_b200_handle h, const int32_t* ids, int32_t num, int32_t* out_codes);

/* Replaces: VectorIndex::DeleteIndex(const void* p_vectors, SizeType num) (BKTIndex.cpp:876-890, KDTIndex.cpp:602-616):
 * for every vector SearchIndex (the index's MaxCheck, searchDeleted = false, K = CEF), then DeleteIndex of every result
 * with Dist < 1e-6.  The reference runs the vectors under OpenMP, where one deletion can change a later search; this
 * call computes its single-thread order (vector 0, 1, ...).  vectors: HOST, num x dim of the index value type. */
int sptag_b200_delete_vectors(sptag_b200_handle h, const void* vectors, int32_t num);

/* Replaces: VectorIndex::AddIndex(p_data, p_vectorNum, p_dimension, nullptr, false, p_normalized) (BKTIndex.cpp:902-970,
 * KDTIndex.cpp:628-696): appends the rows (graph rows -1, tombstone bytes 0; Dataset.h:127-144), normalises them for
 * Cosine unless `normalized` (Utils::Normalize, CommonUtils.h:62-76), then for node = first .. last in order runs
 * RefineNode(node, updateNeighbors = true, searchDeleted = true, AddCEF) (NeighborhoodGraph.h:535-561): the refine search
 * with the node's row (MaxCheckForRefineGraph, K = AddCEF + 1), RebuildNeighbors into the node's row with the graph's
 * degree as NeighborhoodSize and RNGFactor, and InsertNeighbors (RelativeNeighborhoodGraph.h:40-82) of the node into the
 * row of every other result.  The reference's loop is sequential too, so the graph equals its graph bit for bit.
 * The tree is not changed.  Once AddCountForRebuild vectors (default 1000) were added since the tree was built, the
 * reference starts an asynchronous tree rebuild (RebuildJob) whose result and timing are not reproducible: results equal
 * the reference's as long as that job has not replaced its tree.
 * vectors: HOST, num x dim.  out_first_id (nullable): the first new id, id_offset included.
 * EmptyData for null / num <= 0 / dim <= 0, DimensionSizeMismatch for a wrong dim.  Buffers grow geometrically.
 * If a step of the chain fails, the call returns its error and the index keeps the rows that were linked in before the
 * failing one (sptag_b200_num_vectors tells how many); the later rows are dropped. */
int sptag_b200_add(sptag_b200_handle h, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                   int32_t* out_first_id);

/* Replaces: VectorIndex::SaveIndex(folder) (VectorIndex.cpp:197-222 SaveIndexConfig): writes indexloader.ini (algorithm,
 * value type, metric, NeighborhoodSize, the search and update parameters) and vectors.bin / graph.bin / tree.bin /
 * deletes.bin in the formats sptag_b200_load parses (Dataset.h:146-180, NeighborhoodGraph.h:606-615, BKTree.h:635-645 /
 * KDTree.h:123-133, Labelset.h:78-83).  The reference's VectorIndex::LoadIndex reads the folder too.  Live rows' tombstone
 * bytes are 0 (the reference's own save has 0xff for rows added since load, Dataset.h:127-144; both mean "live").  Creates the folder
 * if needed.  Quantized handles: LackOfInputs (the quantizer blob is not kept). */
int sptag_b200_save(sptag_b200_handle h, const char* folder);

/* ---- SPANN with its posting lists in HBM ----
 * Replaces: VectorIndex::LoadIndex(folder) for a SPANN folder (VectorIndex.cpp:617-681, SPANN::Index<T>::LoadConfig /
 * LoadIndexData, SPANNIndex.cpp:59-140, ExtraFullGraphSearcher::LoadIndex / LoadingHeadInfo, ExtraFullGraphSearcher.h:
 * 163-220, :1030-1120).  Reads indexloader.ini ([Base] ValueType, HeadIndexFolder, HeadVectorIDs; [BuildSSDIndex]
 * SSDIndex, SearchInternalResultNum, MaxDistRatio, SearchPostingPageLimit, PostingVectorLimit,
 * EnablePostingListRearrange), loads the head folder with sptag_b200_load and applies to it the [BuildHead] keys that
 * sptag_b200_load reads from [Index], as SPANN::Index::SetParameter does (:1033-1038), reads the translate map and every posting file (SSDIndex,
 * SSDIndex_1, ...) in the plain or the rearranged layout, and packs the lists into HBM.  Each list keeps its full element
 * count; SearchPostingPageLimit truncates at search time.  Section and parameter names are read case-insensitively, as
 * Helper::IniReader reads them.  LackOfInputs for EnableDataCompression and EnableDeltaEncoding.
 * Quantized SPANN ([Base] QuantizerFilePath set, as the reference builds it from PQ/OPQ code rows): the head must be a
 * quantized BKT index (UInt8 code rows and a quantizer), the folder's quantizer (the file its [Quantizer] section names)
 * is installed on the head as SPANN::Index::SetQuantizer does (SPANNIndex.cpp:39-56), [BuildSSDIndex] EnableADC sets the
 * head's EnableADC, ValueType must be UInt8 (what the reference writes) or the quantizer's reconstruct type, and the
 * lists hold M-byte code rows (M + 4 bytes per element).  LackOfInputs when the head holds no quantizer (tested before
 * the quantizer file is opened) and for Cosine with a quantizer (quantized search is L2 only, PQQuantizer.h:130-136).
 * Device memory: the packed lists (rows at the head's row stride, one int32 id each), plus during the load a staging
 * buffer of at most 64 MB (or the largest list, if larger); MemoryOverFlow when that does not fit. */
typedef struct sptag_b200_spann* sptag_b200_spann_handle;
int sptag_b200_spann_load(const char* folder, int32_t device, sptag_b200_spann_handle* out);
void sptag_b200_spann_destroy(sptag_b200_spann_handle s);

/* Where sptag_b200_spann_load_ex keeps the packed posting lists (rows and ids).
 *   AUTO:   HBM when cudaMemGetInfo's free bytes, after the head and the translate map are loaded, exceed the lists' bytes
 *           plus a reserve of 1 GB for the searches' buffers; pinned host memory otherwise.
 *   DEVICE: HBM, as sptag_b200_spann_load (MemoryOverFlow when they do not fit).
 *   HOST:   one pinned, mapped host allocation (cudaHostAlloc), in the layout they have in HBM.  The translate map and each
 *           list's offset, count and page count stay in HBM.  Every search and iterator step copies the lists its queries
 *           read (their searched prefix, at the page limit in force) into an HBM stage of B200.PostingStageBytes per
 *           staging set and scans them there; results equal the device placement's bit for bit.  When a batch's union of
 *           lists does not fit the stage, the batch runs in rounds: a round takes the next n items (queries of a search,
 *           queries of a posting-step launch of an iterator), n starting at the whole batch and halved (rounded up) until
 *           their union fits; the next round starts from the same n.  The stage is never smaller than one query's worst
 *           case, SearchInternalResultNum x the longest searched list x (row stride + 4) bytes.  MemoryOverFlow when the
 *           pinned allocation fails.  sptag_b200_spann_cache_warm / sptag_b200_spann_cache_lists keep some lists, whole,
 *           in HBM as well: those are read in place and never copied, and a batch's union and its rounds count the
 *           other lists only.
 *   FILE:   the lists stay in their posting files, as the reference keeps them on SSD (ExtraFullGraphSearcher::
 *           SearchIndex reads each chosen list's pages at search time).  The load reads the ini, the head, the translate
 *           map and each posting file's header, and none of the lists' bodies; it keeps one descriptor per posting file
 *           open for the handle's life, and each list's offset, count and page count in HBM.  It returns Fail when a
 *           list's full extent runs past the end of its file.  Searches, iterator steps and cache installs run as on a
 *           HOST handle, with the same stages, rounds and results, but read each round's union from the files: a pool
 *           of min(16, hardware threads) threads preads it, a piece of at most 64 MB (or the largest list) at a time,
 *           into one of two pinned, mapped windows per staging set, and a kernel cuts each piece's records into the
 *           stage while the next piece is read.  A round reads each list's searched prefix (plain layout) or the whole
 *           list (rearranged layout): element count x (dim x sizeof(T) + 4) bytes; lists cached in HBM are never read.
 *           Each call first checks that every posting file is still the file loaded at its path (same device and
 *           inode).  A posting file moved away or replaced, or a read that fails or ends early (a file truncated after
 *           the load), fails the call with Fail, whose message names the file (and the list and offset of a read); the
 *           handle keeps working, and the next call reads again.  Pinned host memory: 2 x 2 x (64 MB, or the largest
 *           list's bytes, + 64 KB) windows, allocated on a staging set's first read; HBM: the lists' offsets, counts and
 *           pages, the stages and the cache.  Compressed and delta-encoded lists are refused as on every placement, and
 *           SPANN groups (sptag_b200_spann_group_load) keep the HOST layout. */
enum {
    SPTAG_B200_POSTINGS_AUTO = 0,
    SPTAG_B200_POSTINGS_DEVICE = 1,
    SPTAG_B200_POSTINGS_HOST = 2,
    SPTAG_B200_POSTINGS_FILE = 3
};
typedef struct {
    int32_t struct_size;        /* sizeof(sptag_b200_spann_load_options) */
    int32_t posting_placement;  /* SPTAG_B200_POSTINGS_* */
} sptag_b200_spann_load_options;

/* sptag_b200_spann_load with a choice of where the posting lists live (options NULL: AUTO).  LackOfInputs for an unknown
 * placement, Fail for a struct_size other than sizeof(sptag_b200_spann_load_options).  The handle's B200.PostingPlacement
 * reads "device", "host" or "file". */
int sptag_b200_spann_load_ex(const char* folder, int32_t device, const sptag_b200_spann_load_options* options,
                             sptag_b200_spann_handle* out);

/* Replaces: the SSD stage of SPANN::Index<T>::BuildIndex with SelectHead and BuildHead off (SPANNIndex.cpp:889-951):
 * ExtraFullGraphSearcher::BuildIndex (ExtraFullGraphSearcher.h:587-922) with VectorIndex::ApproximateRNG
 * (VectorIndex.cpp:884-986, its CPU form), SortSelections (EdgeCompare, SearchResult.h:29-63), the posting cut (:722-760),
 * SelectPostingOffset (:1206-1290) and OutputSSDIndexFile (:1292-1568), for a folder that already holds its head.
 * folder: indexloader.ini (names read case-insensitively), the head index folder and the head-id file.  Keys read, with
 * the reference's defaults (SPANN/ParameterDefinitionList.h): [Base] ValueType, DistCalcMethod, Dim, HeadIndexFolder,
 * HeadVectorIDs, SSDIndex, SSDIndexFileNum, QuantizerFilePath; [BuildSSDIndex] ReplicaCount (<= 64), InternalResultNum
 * (<= 2048), RNGFactor, PostingPageLimit, PostingVectorLimit, ExcludeHead, EnablePostingListRearrange, MaxCheck (the
 * head's, as SPANNIndex.cpp:901 sets it), EnableDataCompression, EnableDeltaEncoding, OutputEmptyReplicaID.
 * vectors: HOST, num x dim of ValueType, row i is vector id i.  Cosine rows are normalised first unless `normalized`.
 * Every vector that is not a head (the head-id file's uint64s cast to SizeType) is searched on the head at K =
 * InternalResultNum; the RNG test (RNGFactor * ComputeDistance(head_i, head_j) < dist_i rejects candidate i) keeps at
 * most ReplicaCount heads; the lists are sorted by (distance, vector id), cut to PostingPageLimit pages, split over
 * SSDIndexFileNum files (SSDIndex, SSDIndex_1, ...) and written byte for byte as the reference writes them, in the plain
 * or the rearranged layout.  With ExcludeHead false the head-id file is first rewritten with MaxSize for every head, so
 * every vector is searched.  indexloader.ini is not rewritten.  device: CUDA ordinal of the head.
 * out_stats: HOST int64[8] or NULL: vectors searched, RNG rejections, edges before the cut, edges after it, then device
 * microseconds of the head searches, the RNG selection and the sort, and host microseconds of writing the files.
 * Device memory: the head index, the rows (num x dim, tightly packed), 24 bytes per edge (num x ReplicaCount edges, the
 * radix sort's two key / vector-id buffers) plus the sort's scratch, one search batch of 65536 rows x InternalResultNum
 * results, and a 64 MB window of the file being written.
 * Codes: EmptyData (null input, num <= 0), DimensionSizeMismatch (dim differs from [Base] Dim or the head's),
 * MemoryOverFlow (the rows and edges do not fit, or more than 2^31 - 1 edges), LackOfInputs (QuantizerFilePath,
 * EnableDataCompression, EnableDeltaEncoding, OutputEmptyReplicaID, a head whose type or distance differs from the
 * folder's, a NaN or infinity in a float row or a distance, parameters outside the ranges above). */
int sptag_b200_spann_build(const char* folder, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                           int32_t device, int64_t* out_stats);

/* sptag_b200_spann_build for vector sets whose rows or edges do not fit the device.  device_budget_bytes: the device bytes
 * the call may allocate beyond the head index (and beyond what the head search allocates, as in every search); -1:
 * cudaMemGetInfo's free bytes after the head is loaded, less 1 GB (AUTO's reserve, sptag_b200_spann_load_ex). */
typedef struct {
    int32_t struct_size;          /* sizeof(sptag_b200_spann_build_options) */
    int64_t device_budget_bytes;  /* >= -1 */
} sptag_b200_spann_build_options;

/* sptag_b200_spann_build with a device budget (options NULL: budget -1).  The same arguments, ini keys and refusals; the
 * files are the same byte for byte, whichever path runs.  Fail for a struct_size other than
 * sizeof(sptag_b200_spann_build_options), LackOfInputs for a budget below -1.
 * Path: the resident path (sptag_b200_spann_build's) runs when num x ReplicaCount <= 2^31 - 1 and its working set fits
 * the budget: num x dim x sizeof(T) (the rows) + 24 x num x ReplicaCount (the edges) + the radix sort's scratch for them
 * + min(num, 65536) x InternalResultNum x 8 (one search batch of results) + 64 MB (the window).  Otherwise the streamed
 * path runs:
 *   The caller's rows stay where they are: the buffer is registered (cudaHostRegisterMapped; one registered before is
 *   used as it is) for the call and never written.  Pass 1 copies batches of B rows into two HBM batch buffers (batch
 *   i + 1's copy overlaps batch i's search), checks and normalises them as the resident path does, searches the head,
 *   runs the RNG selection and appends the filled edges, in vector-id order, to a pinned host edge store of 12 B per
 *   edge (keys and vector ids, room for every non-head vector x min(ReplicaCount, InternalResultNum, head count)).  B is
 *   65536 (at most num), halved while pass 1's device bytes exceed the budget:
 *     P1(B) = B x (2 x row + 5 + 8 x InternalResultNum + 25 x ReplicaCount) + the selection's scratch for B x
 *             ReplicaCount edges + 4 x heads + 40,  row = dim x sizeof(T).
 *   Pass 2 cuts each file's lists, in placement order, into groups (never across files, at least one list each) and
 *   per group streams the whole edge store through HBM in chunks of C edges, keeps the group's edges, sorts them,
 *   gathers the rows of the kept elements from the caller's buffer and writes the group's part of the file.  Its
 *   device bytes are F(C) + the largest group's G:
 *     F(C) = 25 x C + the selection's scratch for C edges + 32 + 4 x heads + 28 x (lists of the largest file) + the
 *            window, min(64 MB, the largest file's list area);
 *     G    = a(8E) x 2 + a(4E) x 2 + a(the radix sort's scratch for E edges) + a(kept elements x row), for a group of
 *            E edges before the cut, a(x) = x rounded up to 256.
 *   C is min(edges, 2^22), halved while F(C) + G(the longest list) exceeds the budget, never below min(edges, 4096);
 *   a group then takes lists while its G fits budget - F(C).  Every group costs one pass over the store:
 *   groups x 12 B x edges host to device.
 * MemoryOverFlow, before any posting file is created: a budget below the streamed path's minimum, the larger of P1(1)
 * and F(min(edges, 4096)) + G(the longest list) (the two passes never hold their buffers at once; the message names
 * the minimum), or a pinned edge store that cannot be allocated.
 * out_stats: HOST int64[12] or NULL: sptag_b200_spann_build's 8 (on the streamed path the sort is every group's, and the
 * write's host microseconds are pass 2's other work: edge passes, gathers, images and fwrite), then the path (0
 * resident, 1 streamed), the row batches, the edge groups (1 on the resident path) and the bytes copied host to device
 * (rows, edge passes and gathered rows). */
int sptag_b200_spann_build_ex(const char* folder, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                              int32_t device, const sptag_b200_spann_build_options* options, int64_t* out_stats);

/* Replaces: SPANN::Index<T>::SearchIndex(QueryResult&) (SPANNIndex.cpp:193-250) with ExtraFullGraphSearcher::SearchIndex
 * (ExtraFullGraphSearcher.h:226-375) for a batch.  The head search runs at W = max(K, SearchInternalResultNum); the
 * postings are chosen from its results, the result array is reversed, every chosen list is scanned in order with the
 * deduper, the head's distance function and QueryResultSet::AddPoint, and SortResult orders the array
 * (QueryResultSet.h:77-112); the first K entries are returned.  Results equal the reference's bit for bit.
 * queries: HOST, num_queries x dim of the value type; on a quantized index raw vectors of the quantizer's reconstruct type
 * and dimension, which the head search and the posting scan both score with the quantizer's SDC or (EnableADC) ADC
 * distance, ExtraFullGraphSearcher<std::uint8_t> (ExtraFullGraphSearcher.h:120-130).
 * out_ids / out_dists: HOST [num_queries x k].  out_stats: HOST
 * [num_queries x 3] int32 or NULL: postings scanned (m_diskIOCount), list elements read (m_totalListElementsCount),
 * distances computed.  k <= 2048.  Thread-safe; two callers overlap.  LackOfInputs when the page limit truncates lists
 * of the rearranged layout (the reference then reads ids from an offset computed with the truncated count,
 * ExtraFullGraphSearcher.h:1186-1190, which is not reproduced). */
int sptag_b200_spann_search(sptag_b200_spann_handle s, const void* queries, int32_t num_queries, int32_t k, int32_t* out_ids,
                            float* out_dists, int32_t* out_stats);

/* Replaces: SPANN::Index<T>::SetParameter / GetParameter (SPANNIndex.cpp:1033-1073) for SearchInternalResultNum,
 * MaxDistRatio (a float), SearchPostingPageLimit (raised at search time to the pages of PostingVectorLimit vectors, as
 * ExtraFullGraphSearcher::LoadIndex does, :167), MaxCheck and EnableADC (the head's; on a quantized index EnableADC
 * switches the head search and the posting scan together, as the shared quantizer does, VectorIndex.h:136-138) and
 * IterativeSearchHeadBatch ([BuildSSDIndex],
 * default 32, in [1, 1024]; sampled when an iterator opens).  B200.IteratorVisitedSet and B200.IteratorVisitedHashEntries
 * are the head handle's (sptag_b200_set_param): they choose the visited sets of the head iterators SPANN iterators open.
 * B200.SpannDedupEntries: the first dedup table size of an iterator's queries, 0 (default: room for one head batch of
 * the longest list, at most 2^14) or a power of two >= 64; tables double as they fill.  B200.PostingStageBytes (host
 * or file placement, sptag_b200_spann_load_ex): the HBM stage of each of the two staging sets, default 268435456 (256 MB), in
 * [0, 2^31 - 1]; 0 leaves one query's worst case.  The stage grows when a call needs more and never shrinks.
 * Read-only: PostingBytes (device bytes of the posting lists and the translate map; with host or file placement the
 * lists' offsets, counts and page counts only), B200.PostingPlacement ("device", "host" or "file"),
 * B200.PostingHostBytes (pinned host bytes of the lists' rows and ids, 0 with device or file placement),
 * B200.LastGatherBytes and B200.LastGatherRounds (host or file placement: the staged elements x (row stride + 4) bytes
 * and the rounds of the last search or iterator step on this handle; a FILE handle's equal a HOST handle's for the same
 * calls), B200.LastReadBytes (file placement: the posting-file bytes the last search, iterator step or cache install on
 * this handle read, the sum of element count x (dim x sizeof(T) + 4) over the lists read; 0 otherwise),
 * B200.LastIteratorRounds (head refill rounds of the last sptag_b200_spann_iterator_next on this handle) and
 * B200.LastIteratorDedupBytes (that iterator's dedup table bytes), and B200.LastPostingKernel (the demangled name of the
 * last posting-scan or posting-step kernel instantiation a search or iterator step on this handle launched, e.g.
 * "sptag_b200::(anonymous namespace)::spann_scan_kernel<true, 2>"; empty before the first).
 * Names are matched case-insensitively, and codes are those of sptag_b200_set_param. */
int sptag_b200_spann_set_param(sptag_b200_spann_handle s, const char* name, const char* value);
int sptag_b200_spann_get_param(sptag_b200_spann_handle s, const char* name, char* value_out, int32_t capacity);

/* An HBM cache of posting lists on a handle loaded with the HOST or FILE placement (on FILE, the cached lists are read
 * from their files once, by the install, and never again).  Ranks the posting lists by how many of
 * num_queries sample queries choose them, and caches the top of that order in HBM.  Each query runs the head search and
 * the posting choice of a search with K <= SearchInternalResultNum (W = SearchInternalResultNum), with the search
 * parameters in force; the lists are counted on the device, ranked by count, descending, then list id, ascending, and
 * walked in that order: a list is taken when its full size, element count x (row stride + 4) bytes, fits what is left
 * of budget_bytes, and skipped otherwise.  Lists no query chose are never taken.  budget_bytes -1: cudaMemGetInfo's
 * free bytes, after the previous cache is released, less the 1 GB reserve of the AUTO placement.  The taken lists are
 * installed as sptag_b200_spann_cache_lists installs them, and written to out_lists (HOST, NULL when capacity is 0) in
 * rank order, at most capacity of them; *out_num_lists receives how many were taken.
 * queries: HOST, as sptag_b200_spann_search's.  Codes as sptag_b200_spann_cache_lists', and LackOfInputs for a null
 * buffer, a budget below -1 and a page limit that truncates lists of the rearranged layout. */
int sptag_b200_spann_cache_warm(sptag_b200_spann_handle s, const void* queries, int32_t num_queries,
                                int64_t budget_bytes, int32_t* out_lists, int32_t capacity, int32_t* out_num_lists);
/* Caches exactly the given lists in HBM (num_lists = 0 releases the cache), e.g. a set an earlier
 * sptag_b200_spann_cache_warm returned.  lists: HOST, distinct ids in [0, number of lists).  The call waits until no
 * search or iterator step runs on the handle (it takes both staging sets), releases the old cache and copies every
 * element of each list, whatever SearchPostingPageLimit is, from the pinned host allocation (FILE: from the posting
 * files, through staging set 0's windows) into one HBM allocation that
 * also holds the stage of each staging set.  Searches and iterator steps that start after it returns read the cached
 * lists in place; iterators opened earlier keep working, with unchanged results.  Results equal the device placement's
 * bit for bit with any cache.  B200.LastGatherBytes and B200.LastGatherRounds count only what is still copied from host
 * memory.  A stage that a later call needs to grow (B200.PostingStageBytes, SearchInternalResultNum or the page limit
 * raised) re-installs the same lists.  Read-only parameters: B200.PostingCacheLists (lists cached) and
 * B200.PostingCacheBytes (the HBM their rows and ids take).  Device memory: those bytes plus both stages.
 * Codes: LackOfInputs for a DEVICE-placed handle, an id outside the range, an id given twice and a null buffer;
 * MemoryOverFlow when the allocation fails, and on a FILE handle Fail when a read fails, after either of which the
 * handle works uncached. */
int sptag_b200_spann_cache_lists(sptag_b200_spann_handle s, const int32_t* lists, int32_t num_lists);

/* ---- SPANN on several GPUs of one host ----
 * Replaces: N processes of SPANN::Index<T> on one folder, one per GPU (VectorIndex::LoadIndex, SPANNIndex.cpp:59-140,
 * SearchIndex, :193-250); the reference has no single call for it.  A group holds one pinned copy of the posting lists
 * for all its members, and an HBM cache of lists spread over them.
 *   load:   devices: 1 to 16 CUDA ordinals, one member each (a device may repeat).  The folder's posting files are read
 *           once, as sptag_b200_spann_load_ex reads them, into one pinned allocation that every device maps
 *           (cudaHostAlloc, mapped and portable; the HOST placement's layout).  Each member is a HOST-placed handle with
 *           its own head (sptag_b200_load on its device), translate map, list offsets, counts and page counts, and
 *           staging sets.  Peer access is enabled both ways between the members' devices where the hardware allows it.
 *           Codes: sptag_b200_spann_load_ex's refusals with the same codes, LackOfInputs for a null or empty device
 *           list or more than 16 entries, Fail for a device that does not exist.
 *   member: member i's handle, borrowed: sptag_b200_spann_search, the iterators, get_param and set_param work on it as
 *           on any HOST-placed handle; sptag_b200_spann_destroy on it does nothing; sptag_b200_spann_cache_warm and
 *           sptag_b200_spann_cache_lists on it return LackOfInputs (its peers read its cache).  LackOfInputs for i
 *           outside [0, members).
 *   set_param:  sptag_b200_spann_set_param on every member in turn, under the group's lock; the first failure's code.
 *   search: sptag_b200_spann_search's arguments.  Member i searches queries [i * ceil(Q / n), (i + 1) * ceil(Q / n)) on a
 *           thread of its own; outputs are written in place, out_stats (HOST [num_queries x 3] int64 or NULL) as
 *           sptag_b200_spann_search's.  A query's result does not depend on which member runs it, and equals the
 *           reference's bit for bit.  LackOfInputs when the members differ in SearchInternalResultNum, MaxDistRatio,
 *           SearchPostingPageLimit or MaxCheck (one was set on its own); otherwise the first failing member's code.
 *   cache_warm: ranks the lists as sptag_b200_spann_cache_warm does, on member 0's head, then walks the ranking: each
 *           list goes to the member with the most budget left (the lower index of equals) if its full size, element
 *           count x (row stride + 4) bytes, fits there, and is skipped otherwise.  budget_bytes_per_member -1: each
 *           member's free HBM after its cache is released, less 1 GB (members sharing a device each count all of its
 *           free HBM).  The lists are installed, and written in rank order to out_lists with their members to
 *           out_owners (HOST, at most capacity; *out_n receives how many were taken).  Codes as
 *           sptag_b200_spann_cache_warm's.
 *   cache_lists: caches list lists[i] on member owners[i] (HOST); n = 0 releases every member's cache.  LackOfInputs
 *           for a list outside the range or given twice, an owner outside [0, members) and a null buffer.
 * Every list is cached on at most one member.  A member copies a list it does not cache from the pool of the member
 * that caches it when both are on one device or peer access reaches it (HBM or NVLink), and from the pinned allocation
 * otherwise; B200.LastGatherBytes and B200.LastGatherRounds count both, over the lists the member does not cache
 * itself, exactly as on a single handle.  Read-only member parameters: B200.PostingPeerLists (lists the member reads from
 * a peer's cache) and B200.LastPeerGatherBytes (the part of B200.LastGatherBytes copied from peers; the rest crossed the
 * host link).  A cache install on any member (these calls, or a stage that grows with B200.PostingStageBytes,
 * SearchInternalResultNum or the page limit) waits until no search or iterator step runs on any member.
 *   destroy: destroys every member and frees the pinned allocation. */
typedef struct sptag_b200_spann_group* sptag_b200_spann_group_handle;
int sptag_b200_spann_group_load(const char* folder, const int32_t* devices, int32_t num_members,
                                sptag_b200_spann_group_handle* out);
int sptag_b200_spann_group_member(sptag_b200_spann_group_handle g, int32_t i, sptag_b200_spann_handle* out);
int sptag_b200_spann_group_set_param(sptag_b200_spann_group_handle g, const char* name, const char* value);
int sptag_b200_spann_group_search(sptag_b200_spann_group_handle g, const void* queries, int32_t num_queries, int32_t k,
                                  int32_t* out_ids, float* out_dists, int64_t* out_stats);
int sptag_b200_spann_group_cache_warm(sptag_b200_spann_group_handle g, const void* queries, int32_t num_queries,
                                      int64_t budget_bytes_per_member, int32_t* out_lists, int32_t* out_owners,
                                      int32_t capacity, int32_t* out_n);
int sptag_b200_spann_group_cache_lists(sptag_b200_spann_group_handle g, const int32_t* lists, const int32_t* owners,
                                       int32_t n);
void sptag_b200_spann_group_destroy(sptag_b200_spann_group_handle g);

/* Replaces: SPANN::Index<T>::GetIterator(p_target) (SPANNIndex.cpp:299-314) and SPANNResultIterator::Next(batch)
 * (SPANNResultIterator.h:37-63, SPANNIndex.cpp:261-296, :416-446, ExtraFullGraphSearcher.h:131-147, :492-525) for every
 * query of a HOST batch, one iterator per query.
 *   open:  opens a head iterator per query (p_searchDeleted = false) and an empty ExtraWorkSpace; the head batch is
 *          IterativeSearchHeadBatch as set now.  The SPANN handle must outlive its iterators.
 *   next:  up to `batch` further results per query, a resumable, deduplicated stream of posting elements.  The first call
 *          runs the head's SearchIndexIterativeFromNeareast(first); then each query reads its chosen lists from where it
 *          stopped, and when they run out asks the head for its next batch, until the call has `batch` results or the
 *          head finds nothing.  As in the reference, a call's batch is capped by the previous call's result count, the
 *          deduper spans every head batch and call, an element found as the last element of the last list is added to
 *          the result but not counted, and RelaxedMono turns on once SearchInternalResultNum lists were loaded before a
 *          load.  out_ids / out_dists: HOST [num_queries x batch], sorted, unfilled slots (-1, MaxDist); out_counts[q] =
 *          resultCount; out_relaxed_mono[q] = GetRelaxedMono().  Results equal the reference's bit for bit.
 *          sptag_b200_spann_search on the same handle may run between calls; it does not change their results.
 *   close: frees the iterators.
 * LackOfInputs: null arguments, batch outside [1, 1024], IterativeSearchHeadBatch outside [1, 1024] (open) or above
 * SearchInternalResultNum (next: the reference has only that many page buffers, IExtraSearcher.h:114-122), a page
 * limit that truncates lists of the rearranged layout (as sptag_b200_spann_search), and quantized SPANN handles (open:
 * head iterators are not built for quantized indexes). */
typedef struct sptag_b200_spann_iterator* sptag_b200_spann_iter;
int sptag_b200_spann_iterator_open(sptag_b200_spann_handle s, const void* queries, int32_t num_queries,
                                   sptag_b200_spann_iter* out);
int sptag_b200_spann_iterator_next(sptag_b200_spann_iter it, int32_t batch, int32_t* out_ids, float* out_dists,
                                   int32_t* out_counts, uint8_t* out_relaxed_mono);
void sptag_b200_spann_iterator_close(sptag_b200_spann_iter it);

/* ---- Multi-index scan ----
 * Replaces: MultiIndexScan::Init(indexes, targets, weight, k, useTimer = false, termCondVal, searchLimit), Next until it
 * returns false, and Close (inc/Core/MultiIndexScan.h, src/Core/MultiIndexScan.cpp:51-183) for every query of a HOST
 * batch: the k ids with the smallest weighted sum of per-index distances, over indexes that hold the same ids (for example
 * an image and a text embedding of each item).  Per query, an iterator with p_searchDeleted = true is opened on every
 * index; each round asks every index in order for Next(1) and scores an id not seen before as
 * sum_i weight[i] * dist_i(target_i, id), with GetDistance for the indexes that did not return it; the score enters the
 * top-k unless the queue is full and its largest score is <= it, which counts a consecutive drop.  The round that finds an
 * iterator empty ends the query at that index.  After a round the query ends when the consecutive drops reach term_cond
 * (compared unsigned: a negative value never ends by drops), or else when the ids seen reach search_limit (compared as
 * size_t: a negative value never ends by size).  Results equal the reference's bit for bit, including which of equal
 * scores is kept and their output order (libstdc++'s heap), and the score's rounding as GCC compiles WeightedRankFunc
 * for x86-64-v3 (rounded products added one after another in blocks of 8 and 4, the last num_indexes % 4 terms fused).
 *   queries[i]: HOST, num_queries rows of index i's dimension and value type; the indexes may differ in dimension, value
 *               type and metric.
 *   weights:    num_indexes floats, or NULL for the plain sum (rankFunc, MultiIndexScan.cpp:37-39), which equals unit
 *               weights bit for bit.
 *   out_ids / out_scores: HOST [num_queries x k] in the order Next returns them (smallest score first, Dist = score);
 *               unfilled slots (-1, MaxDist).  out_counts[q]: the number of results.
 *   out_stats:  HOST [num_queries x 4] int32 or NULL: rounds run, seenSet.size(), consecutive_drops at the end, and why the
 *               query ended (SPTAG_B200_MS_END_*; SPTAG_B200_MS_END_EXHAUSTED + i: iterator i returned nothing).
 * The timer form (useTimer = true) is not offered: a wall-clock limit does not give reproducible results.  A user rank
 * function cannot run on the device either.  The handles are not changed: their iterators are opened and closed inside
 * the call, so they can be mutated again when it returns.
 * LackOfInputs: null arguments, num_indexes outside [1, 16], k outside [1, 1024], handles that differ in device, vector
 * count or id offset, and quantized handles.  Fail: a KDT handle (GetIterator on KDT).  Blocking. */
#define SPTAG_B200_MS_STATS_PER_QUERY 4
#define SPTAG_B200_MS_END_DROPS 0
#define SPTAG_B200_MS_END_LIMIT 1
#define SPTAG_B200_MS_END_EXHAUSTED 2
int sptag_b200_multi_scan(const sptag_b200_handle* indexes, int32_t num_indexes, const void* const* queries,
                          const float* weights, int32_t num_queries, int32_t k, int32_t term_cond, int32_t search_limit,
                          int32_t* out_ids, float* out_scores, int32_t* out_counts, int32_t* out_stats);

/* Labelset::Count(): tombstones set so far. */
int32_t sptag_b200_num_deleted(sptag_b200_handle h);

/* Device time in milliseconds of the search kernel(s) of the most recent sptag_b200_search*
 * call on this handle, measured with CUDA events on the launching stream (synchronises). */
int sptag_b200_last_kernel_ms(sptag_b200_handle h, float* ms_out);

/* Number of kernels this library launched so far in this process (for bench.py's gpu_launches). */
int64_t sptag_b200_launch_count(void);

/* For tests: the kernel instantiation a launch would take, by the same selectors, as the name B200.LastSearchKernel
 * reports after it.  Host-only: no CUDA call, no device needed.  value_type / metric / algo as sptag_b200_index_desc;
 * simd_width, enable_bfs, row_sketch as B200.SimdWidth, EnableBfs, B200.RowSketch (non-zero: the sketches are in use,
 * which only float BKT rows without breadth-first seeding take); quantized: PQ / OPQ codes (value_type UInt8, dim = M);
 * mres_cap: max(MaxCheck / 16, K); slots: the query slots per SM the launch aims at (128-d float rows: B200.QueriesPerSM,
 * or the automatic 14 to 20; otherwise 0); family: 0 search, 1 ResultIterator::Next, 2 the first
 * SearchIndexIterativeFromNeareast call.  LackOfInputs: no kernel for that m_Results capacity. */
int sptag_b200_debug_kernel_for(int32_t value_type, int32_t metric, int32_t algo, int32_t dim, int32_t simd_width,
                                int32_t enable_bfs, int32_t row_sketch, int32_t quantized, int32_t mres_cap, int32_t slots,
                                int32_t family, char* name_out, int32_t capacity);

/* Index facts (VectorIndex::GetNumSamples / GetFeatureDim / ...). */
int32_t sptag_b200_num_vectors(sptag_b200_handle h);
int32_t sptag_b200_dim(sptag_b200_handle h);
int32_t sptag_b200_value_type(sptag_b200_handle h);
int32_t sptag_b200_metric(sptag_b200_handle h);
int32_t sptag_b200_algo(sptag_b200_handle h);

/* Human-readable text for the last failure on this thread. */
const char* sptag_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* SPTAG_B200_H_ */
