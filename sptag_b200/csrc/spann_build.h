// spann_build.h -- the device half of SPANN's posting-list build (ExtraFullGraphSearcher::BuildIndex,
// ExtraFullGraphSearcher.h:587-922, with VectorIndex::ApproximateRNG, VectorIndex.cpp:884-986) as sptag_b200.cu
// launches it; the kernels live in kern_spann_build.cu.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>

namespace sptag_b200 {

constexpr int kSpannBuildMaxReplicas = 64;

// ApproximateRNG for the vectors [first, first + num): one warp per vector.  A vector marked in `head` keeps Edge()'s
// unfilled slots; every other one walks its head results (res_ids / res_dists, row v - first, k per vector, ascending,
// -1 ends them) and accepts candidate i unless an already accepted head j has rng_factor * ComputeDistance(i, j) < dist_i,
// until `replicas` are accepted.  Edge slot s of vector v is keys[v * replicas + s] = (node << 32) | order bits of the
// distance, tonode[v * replicas + s] = v; an unfilled slot has node = num_heads (after every list).
struct SpannRngParams {
    const int* res_ids;
    const float* res_dists;
    int k, first, num;
    const unsigned char* head;     // per vector id: 1 = a head id (not searched)
    const unsigned char* rows;     // the head index's rows, row_stride bytes apart (16-byte aligned, zero padded)
    size_t row_stride;
    int dim, simd_width;
    int replicas, num_heads;
    float rng_factor;
    unsigned long long* keys;
    int* tonode;
    int* list_size;                 // [num_heads] accepted edges per head (postingListSize)
    unsigned long long* rejected;   // RNG rejections (rngFailedCount)
    int* bad;                       // set when a distance is not finite
};
cudaError_t launch_spann_rng_select(const SpannRngParams& p, bool cosine, int elem, cudaStream_t stream);

// Sets *bad when one of n float values is not finite
cudaError_t launch_spann_nonfinite_check(const float* v, size_t n, int* bad, cudaStream_t stream);

// SortSelections with EdgeCompare (SearchResult.h:29-63) on edges in ascending tonode order: a stable LSD radix sort of
// the keys over their low end_bit bits, tonode carried along.  temp == nullptr: *temp_bytes receives the scratch size.
cudaError_t spann_sort_edges(void* temp, size_t* temp_bytes, const unsigned long long* keys_in, unsigned long long* keys_out,
                             const int* tonode_in, int* tonode_out, int n, int end_bit, cudaStream_t stream);

// One window [win_begin, win_end) of a posting file's list area (OutputSSDIndexFile, ExtraFullGraphSearcher.h:1421-1550,
// with GetPostingListFullData, :527-585): list i of the file (in placement order) starts at byte start[i] of the area and
// holds count[i] elements, the sorted edges edge_off[i], ...; an element is its int32 vector id and its row of row_bytes
// bytes, laid out [id][row] per element or, rearranged, every row and then every id.  `out` holds the window, zeroed.
struct SpannImageParams {
    const long long* start;
    const long long* edge_off;
    const int* count;
    int first_list, num_lists;  // the lists that overlap the window
    const int* tonode;
    const unsigned char* rows;  // the full rows, row_bytes apart
    int row_bytes, rearranged;
    long long win_begin, win_end;
    unsigned char* out;
    const long long* row_off;   // nullptr: element e of list l is row tonode[edge_off[l] + e] of `rows`; otherwise row
                                // row_off[l] + e (the rows a group gathered, sptag_b200_spann_build_ex's streamed path)
};
cudaError_t launch_spann_posting_image(const SpannImageParams& p, cudaStream_t stream);

// The order-preserving selection of n edges (keys, tonode) into keys_out / tonode_out, *num_selected (device) their
// count: group_of == nullptr keeps the filled edges (node < num_heads) and first adds tonode_add to every tonode in
// place; otherwise it keeps the edges whose list l has group_of[l] == group.  flags: n bytes of scratch.
// temp == nullptr: *temp_bytes receives the scratch size.
cudaError_t spann_select_edges(void* temp, size_t* temp_bytes, const unsigned long long* keys, int* tonode, int n,
                               int tonode_add, int num_heads, const int* group_of, int group, unsigned char* flags,
                               unsigned long long* keys_out, int* tonode_out, int* num_selected, cudaStream_t stream);

// The rows of lists [first_list, first_list + num_lists) of a group: list l's first count[l] sorted edges
// tonode[edge_off[l]], ... name rows of src (row_bytes apart, unpadded; mapped host memory), copied to dst rows
// row_off[l], ... with the widest word that the row size and both bases' alignment allow
struct SpannGatherParams {
    const long long* edge_off;
    const long long* row_off;
    const int* count;
    int first_list, num_lists;
    const int* tonode;
    const unsigned char* src;
    int row_bytes;
    unsigned char* dst;
};
cudaError_t launch_spann_row_gather(const SpannGatherParams& p, cudaStream_t stream);

}  // namespace sptag_b200
