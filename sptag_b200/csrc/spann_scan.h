// spann_scan.h -- the SPANN posting kernels as sptag_b200.cu launches them: the posting scan (SPANNIndex.cpp:193-250
// after the head search, ExtraFullGraphSearcher.h:226-375; kern_spann.cu on raw rows, kern_spann_pq.cu on PQ code rows)
// and the posting step of SPANN iterators (kern_spann_iter.cu), with the posting-list view both read.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace sptag_b200 {

struct IterState;  // search_kernels.cuh

// The posting lists in HBM: list l has cnt[l] elements (its full count) and pages[l] pages, its ids at ids[off[l]...] and
// its rows at rows + (off[l] + i) * row_stride
struct PostingLists {
    const long long* off;
    const int* cnt;
    const int* pages;
    const int* ids;
    const unsigned char* rows;
    size_t row_stride;     // also the stride of the query rows
    int vector_info_size;  // dim * sizeof(T) + sizeof(int)
    int page_limit;        // SearchPostingPageLimit in force (already max'ed with PostingVectorLimit's pages)
};

// Elements of a list of cnt elements on `pages` pages that a search reads at page limit `limit` (LoadingHeadInfo's
// truncation, ExtraFullGraphSearcher.h:1093-1097)
__host__ __device__ inline int posting_searched(int cnt, int pages, int limit, int vector_info_size) {
    const long long lim = (long long)(pages < limit ? pages : limit) << 12;
    const long long fit = lim / vector_info_size;
    return (int)(cnt < fit ? cnt : fit);
}

struct SpannScanParams {
    // head search results of every query, W per query, ascending, head-local ids (the head's m_results after SortResult)
    const int* head_ids;
    const float* head_dists;
    int nq, w, k;
    // the query rows, lists.row_stride bytes apart (16-byte aligned, zero padded)
    const unsigned char* queries;
    int dim, simd_width;
    // m_vectorTranslateMap, each uint64 cast to SizeType (int32) as the reference does; INT_MAX = MaxSize = "no vector"
    const int* translate;
    PostingLists lists;
    // search parameters
    int internal;     // SearchInternalResultNum
    float max_dist_ratio;
    // per-block dedup table of table_entries int keys (vid + 1, 0 = empty)
    int* tables;
    int table_entries;
    // outputs: [nq x k] ids / dists, [nq x 3] stats (postings, list elements, distances) or nullptr
    int* out_ids;
    float* out_dists;
    int* out_stats;
};

// Launches the scan for the index's metric and element type (0 float, 1 int8, 2 uint8, 3 int16) on `stream`.
// grid: blocks of one warp, each serving queries blockIdx.x, blockIdx.x + grid, ...  Returns the launch error; *kernel
// receives the host stub of the instantiation it launched (B200.LastPostingKernel names it), as do the launchers below.
cudaError_t launch_spann_scan(const SpannScanParams& p, bool cosine, int elem, int grid, cudaStream_t stream,
                              const void** kernel);
// Single-warp blocks of the scan kernel that fit on one SM with W results per query.
int spann_scan_blocks_per_sm(bool cosine, int elem, int w);
// Its dynamic shared memory: W result dists, vids and posting ids, three 32-entry chunk arrays and two counters
__host__ __device__ inline size_t spann_scan_smem(int w) { return (size_t)w * 12 + 3 * 32 * 4 + 16; }

// The posting scan of a PQ/OPQ-quantized SPANN index (ExtraFullGraphSearcher<std::uint8_t>, SPANNIndex.cpp:93-99): the
// rows are M code bytes and the distance is the quantizer's L2Distance to the quantized query (PQQuantizer.h:110-128).
// Everything else is the scan above; of `s`, queries, dim and simd_width are not read.
struct SpannPqScanParams {
    SpannScanParams s;
    int m, ks, dsub;
    int adc;                      // 0: SDC, the query is M codes; 1: ADC, the query is the rotated float vector
    const unsigned char* qcodes;  // SDC: [nq x m] the quantized queries
    const float* sdc;             // SDC: [m x ks x ks] InitializeDistanceTables
    const float* qrot;            // ADC: [nq x m*dsub] the (OPQ-rotated) float queries
    const float* codebooks;       // ADC: [m x ks x dsub]
    float* adc_tables;            // ADC: per block, the current query's m x ks table
};
cudaError_t launch_spann_pq_scan(const SpannPqScanParams& p, int grid, cudaStream_t stream, const void** kernel);
int spann_pq_scan_blocks_per_sm(int w, int m);
size_t spann_pq_scan_smem(int w, int m);

// What a SPANN iterator keeps per query between launches (SPANNResultIterator's ExtraWorkSpace and the call in progress)
struct SpannIterState {
    int np, pi, offset;  // m_postingIDs.size(), m_pi, m_offset
    int loaded;          // m_loadedPostingNum
    int relaxed;         // m_relaxedMono
    int load;            // m_loadPosting
    int count, batch;    // the call in progress: resultCount and its batch (capped by slots)
    int slots;           // the QueryResult's result count after the last call (SetResultNum); -1 before the first
    int await_head;      // on the refill list: the head iterator was asked for its next batch since the last launch
    int pad[2];
};
static_assert(sizeof(SpannIterState) == 48, "SpannIterState is 12 ints");

// One launch of the posting step of SPANN iterators (SPANNIndex.cpp:261-296, :416-446; ExtraFullGraphSearcher.h:131-147,
// :492-525).  A query runs until its call has `batch` results, its postings run out (it joins `refill`: the host asks the
// head iterator for its next batch and launches again over that list), its head iterator found nothing (the call ends),
// or its dedup table would pass half its capacity within the next chunk (it joins `susp`: the host doubles the table and
// launches again over that list).  A query whose call ends writes its outputs.
struct SpannIterParams {
    const int* head_ids;  // [nq x hb] the head iterator's latest results, head-local ids
    int nq, hb;
    const unsigned int* list;  // the queries of this launch (kIterListHeader layout), or nullptr: all nq
    int batch;                 // Next(batch) as the caller asked
    int fresh;                 // the first launch of a Next: cap the batch by slots and Reset() the QueryResult
    const unsigned char* queries;  // lists.row_stride bytes apart
    int dim, simd_width;
    PostingLists lists;
    int internal;  // SearchInternalResultNum
    SpannIterState* st;
    int* posts;                // [nq x hb] m_postingIDs
    float* heap_d;             // [nq x cap] the call's QueryResult between launches
    int* heap_v;
    int cap;
    unsigned int* const* tables;  // per query: its dedup table (the hashed visited-set format, vhash_home)
    IterState* dedup;             // per query: vbits = log2 of its table's entries, vfill = ids in it
    unsigned int* refill;         // kIterListHeader layout
    unsigned int* susp;
    int* out_ids;                 // [nq x batch]
    float* out_dists;
    int* out_counts;
    unsigned char* out_relaxed;
};
cudaError_t launch_spann_iter_step(const SpannIterParams& p, bool cosine, int elem, int grid, cudaStream_t stream,
                                   const void** kernel);
int spann_iter_step_blocks_per_sm(bool cosine, int elem, int cap);

// Posting lists in pinned host memory (kern_spann_gather.cu).  The packed lists stay where they were loaded (`host`: ids
// and rows in mapped host memory, off, cnt and pages in HBM); before the scan or a posting step runs, the union of the
// lists its queries read is copied into an HBM stage, and the kernels read a PostingLists view of the stage:
// off = stage_off, ids = stage_ids, rows = stage_rows, cnt and pages unchanged.  A union list keeps its searched prefix
// (posting_searched at host.page_limit) in the stage.
// With an HBM cache of lists (sptag_b200_spann_cache_lists), the cached lists, whole, and the stage of each staging set
// share one allocation and one element space: `resident` holds a cached list's first element there (-1: not cached),
// the union takes the other lists only, the stage starts at element stage_base (stage_rows / stage_ids point there), and
// the kernels read a view of the whole allocation with off = view_off.
// A member of a SPANN group (sptag_b200_spann_group_load) also has `peers`: a union list that another member caches
// (same device, or one peer access reaches) is copied from that member's pool instead of from host memory.
constexpr int kMaxSpannPeers = 16;
struct PostingPeers {
    const long long* first;  // [num_lists] the list's first element in its owner's pool, -1: read from host memory
                             // (nullptr: no list is, and the host-only gather runs)
    const int* owner;        // [num_lists] the member that caches it
    const unsigned char* rows[kMaxSpannPeers];  // per member, its pool's rows and ids (element space of its cache)
    const int* ids[kMaxSpannPeers];
    unsigned long long* elems;  // += the elements copied from peers
};
struct PostingGather {
    PostingLists host;
    int num_lists;
    unsigned char* flags;   // [num_lists] the union's lists
    long long* len;         // [num_lists + 1] searched elements of a union list, 0 for the others
    long long* stage_off;   // [num_lists + 1] exclusive sum of len: a union list's first element in the stage; the last
                            // entry is the union's element count
    int* lists;             // [num_lists] the union, compacted in list order
    int* nlists;            // its size
    void* temp;             // CUB scratch of spann_union_temp_bytes(num_lists) bytes
    size_t temp_bytes;
    int* stage_ids;
    unsigned char* stage_rows;
    const long long* resident;  // [num_lists], or nullptr without a cache
    long long stage_base;
    long long* view_off;        // [num_lists] with a cache: resident[l], or stage_base + stage_off[l]
    PostingPeers peers;
};
size_t spann_union_temp_bytes(int num_lists);
// chosen[q * stride ...] / nchosen[q]: the lists query q of a search reads (choose_postings), for every query of p
cudaError_t launch_spann_choose(const SpannScanParams& p, int* chosen, int* nchosen, int stride, cudaStream_t stream);
// chosen[(li - b) * p.hb ...] / nchosen[li - b]: the lists the queries li in [b, e) of an iterator launch read (p.list, or
// every query when it is null): the head's latest batch if the query loads it (load_postings), else posts[pi .. np).
// sub (kIterListHeader layout) receives those queries, for a launch over them.
cudaError_t launch_spann_iter_chosen(const SpannIterParams& p, int b, int e, int* chosen, int* nchosen, unsigned int* sub,
                                     cudaStream_t stream);
// The union of the lists of n items (chosen / nchosen as above, stride apart): g.flags, g.len, g.stage_off, g.lists and
// g.nlists (and with a cache g.view_off).  g.stage_off[g.num_lists] is the union's element count.
cudaError_t launch_spann_union(const PostingGather& g, const int* chosen, const int* nchosen, int stride, int n,
                               cudaStream_t stream);
// Copies g.len[l] elements of every list l of g.lists (the union: its searched prefix) from host memory, or with
// g.peers.first from the peer that caches it, to element g.stage_off[l] of the stage
cudaError_t launch_spann_gather(const PostingGather& g, int grid, cudaStream_t stream);
// Posting lists left in their files (the FILE placement): a union's raw records are read from the posting files into a
// mapped host window, a piece of lists at a time, each list at a 16-byte-aligned window_off.  The unpack cuts each
// list's records into the stage as the gather does: g.len[l] rows at g.host.row_stride, padding bytes zero, and ids,
// from element g.stage_off[l].  Plain layout: element i is [int32 id | row] at i * vis; rearranged: row i at i * (vis -
// 4), id i at (vis - 4) * cnt + 4 * i (the whole list is in the window).  table: [n] in device memory.
struct FilePieceList {
    long long window_off;
    int list;
    int pad;
};
cudaError_t launch_spann_file_unpack(const PostingGather& g, const FilePieceList* table, int n, const unsigned char* window,
                                     bool rearranged, cudaStream_t stream);
// counts[l] += the items (chosen / nchosen as above) that read list l
cudaError_t launch_spann_count(const int* chosen, const int* nchosen, int stride, int n, int* counts, cudaStream_t stream);

}  // namespace sptag_b200
