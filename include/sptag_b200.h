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
 * ThresholdOfNumberOfContinuousNoBetterPropagation; the update parameters AddCEF (500), CEF (1000) and RNGFactor (1.0,
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
 * of vectors), B200.VisitedLogEntries. */
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

/* Labelset::Count(): tombstones set so far. */
int32_t sptag_b200_num_deleted(sptag_b200_handle h);

/* Device time in milliseconds of the search kernel(s) of the most recent sptag_b200_search*
 * call on this handle, measured with CUDA events on the launching stream (synchronises). */
int sptag_b200_last_kernel_ms(sptag_b200_handle h, float* ms_out);

/* Number of kernels this library launched so far in this process (for bench.py's gpu_launches). */
int64_t sptag_b200_launch_count(void);

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
