// spann_scan.h -- the SPANN posting scan (SPANNIndex.cpp:193-250 after the head search, ExtraFullGraphSearcher.h:226-375)
// as sptag_b200.cu launches it; the kernel lives in kern_spann.cu.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace sptag_b200 {

struct SpannScanParams {
    // head search results of every query, W per query, ascending, head-local ids (the head's m_results after SortResult)
    const int* head_ids;
    const float* head_dists;
    int nq, w, k;
    // the query rows, row_stride bytes apart (16-byte aligned, zero padded)
    const unsigned char* queries;
    size_t row_stride;
    int dim, simd_width;
    // m_vectorTranslateMap, each uint64 cast to SizeType (int32) as the reference does; INT_MAX = MaxSize = "no vector"
    const int* translate;
    // posting lists: list l has cnt[l] elements (its full count) and pages[l] pages, its ids at ids[off[l]...] and its
    // rows at rows + (off[l] + i) * row_stride
    const long long* off;
    const int* cnt;
    const int* pages;
    const int* ids;
    const unsigned char* rows;
    int vector_info_size;  // dim * sizeof(T) + sizeof(int)
    // search parameters
    int internal;     // SearchInternalResultNum
    float max_dist_ratio;
    int page_limit;   // SearchPostingPageLimit in force (already max'ed with PostingVectorLimit's pages)
    // per-block dedup table of table_entries int keys (vid + 1, 0 = empty)
    int* tables;
    int table_entries;
    // outputs: [nq x k] ids / dists, [nq x 3] stats (postings, list elements, distances) or nullptr
    int* out_ids;
    float* out_dists;
    int* out_stats;
};

// Launches the scan for the index's metric and element type (0 float, 1 int8, 2 uint8, 3 int16) on `stream`.
// grid: blocks of one warp, each serving queries blockIdx.x, blockIdx.x + grid, ...  Returns the launch error.
cudaError_t launch_spann_scan(const SpannScanParams& p, bool cosine, int elem, int grid, cudaStream_t stream);
// Single-warp blocks of the scan kernel that fit on one SM with W results per query.
int spann_scan_blocks_per_sm(bool cosine, int elem, int w);
size_t spann_scan_smem(int w);

}  // namespace sptag_b200
