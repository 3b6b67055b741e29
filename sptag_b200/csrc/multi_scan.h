// multi_scan.h -- MultiIndexScan's fusion of several BKT iterators over one id space (MultiIndexScan.cpp:87-160) as
// sptag_b200.cu launches it; the kernels live in kern_multi_scan.cu.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace sptag_b200 {

struct IterState;  // search_kernels.cuh

constexpr int kMultiScanMaxIndexes = 16;

// What a scan keeps per query between rounds
struct MultiScanState {
    int rounds;  // rounds of the while loop run so far
    int drops;   // consecutive_drops (compared unsigned)
    int end;     // -1 running; 0 ended by drops, 1 by the search limit, 2 + i: iterator i returned nothing
    int size;    // pq.size()
};
static_assert(sizeof(MultiScanState) == 16, "MultiScanState is 4 ints");

// The round's Next(1) results of every index, as its iterator left them: for query q, counts[i][q] results (0 or 1),
// ids[i][q] (the handle's id offset included) and dists[i][q]
struct MultiScanRound {
    const int* ids[kMultiScanMaxIndexes];
    const float* dists[kMultiScanMaxIndexes];
    const int* counts[kMultiScanMaxIndexes];
};

// GetDistance(target_j, vid) of index j = target for the round's candidates of every other index
struct MultiScanDistParams {
    const unsigned int* list;  // the queries still running (kIterListHeader layout)
    int n, target, id_offset;
    MultiScanRound c;
    const unsigned char* queries;  // index j's query rows, row_stride bytes apart, zero padded
    const unsigned char* rows;     // index j's vectors
    size_t row_stride;
    int dim, simd_width;
    float* cross;  // [nq x n x n]: cross[(q * n + i) * n + j] = distance of index i's candidate in index j
};
cudaError_t launch_multi_scan_distance(const MultiScanDistParams& p, bool cosine, int elem, int grid, cudaStream_t stream);

// One round's merge: the candidates in index order, then the termination test.  Queries that keep running are appended
// to `next` (kIterListHeader layout).
struct MultiScanMergeParams {
    const unsigned int* list;
    unsigned int* next;
    int n, k, id_offset;
    unsigned int term_cond;              // termCondVal as MultiIndexScan stores it
    unsigned long long search_limit;     // searchLimit as seenSet.size() >= searchLimit converts it
    float weight[kMultiScanMaxIndexes];  // WeightedRankFunc's weights
    MultiScanRound c;
    const float* cross;
    MultiScanState* st;
    float* heap_s;  // [nq x k] pq's vector: scores and local ids
    int* heap_v;
    unsigned int* const* tables;  // per query: seenSet (the hashed visited-set format, vhash_home)
    IterState* seen;              // per query: vbits = log2 of its table's entries, vfill = seenSet.size()
};
cudaError_t launch_multi_scan_merge(const MultiScanMergeParams& p, int grid, cudaStream_t stream);

// The end of the scan: pq drained onto outputStk and popped, i.e. Next until it returns false, for every query
struct MultiScanDrainParams {
    int nq, k, id_offset;
    MultiScanState* st;
    const IterState* seen;
    float* heap_s;
    int* heap_v;
    int* out_ids;     // [nq x k]
    float* out_scores;
    int* out_counts;  // [nq]
    int* out_stats;   // [nq x 4] or nullptr
};
cudaError_t launch_multi_scan_drain(const MultiScanDrainParams& p, int grid, cudaStream_t stream);

}  // namespace sptag_b200
