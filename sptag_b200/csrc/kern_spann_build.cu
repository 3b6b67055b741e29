// SPANN posting-list build on the device (ExtraFullGraphSearcher::BuildIndex, ExtraFullGraphSearcher.h:587-922): the
// RNG replica selection of VectorIndex::ApproximateRNG (VectorIndex.cpp:884-986), SortSelections' order (EdgeCompare,
// SearchResult.h:29-63) and the list bytes OutputSSDIndexFile writes (:1421-1550).  sptag_b200.cu runs the head
// searches, the posting cut, SelectPostingOffset and the file headers.
#include "spann_build.h"
#include "spann_device.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

namespace sptag_b200 {
namespace {

constexpr int kRngWarps = 4;

// A float's bits mapped so that unsigned order is float order; -0.0 first becomes +0.0, which EdgeCompare's == treats
// as equal
__device__ __forceinline__ unsigned int order_bits(float d) {
    unsigned int u = __float_as_uint(d == 0.0f ? 0.0f : d);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32 * kRngWarps) spann_rng_select_kernel(const SpannRngParams p) {
    __shared__ int accepted[kRngWarps][kSpannBuildMaxReplicas];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, j = lane & 15, half = lane >> 4;
    const int r = blockIdx.x * kRngWarps + warp;
    if (r >= p.num) return;
    const int v = p.first + r;
    const size_t slot0 = (size_t)v * p.replicas;
    int* acc = accepted[warp];
    int n_acc = 0;
    unsigned long long rejected = 0;
    if (!p.head[v]) {
        const int* ids = p.res_ids + (size_t)r * p.k;
        const float* ds = p.res_dists + (size_t)r * p.k;
        for (int i = 0; i < p.k && n_acc < p.replicas; ++i) {
            const int vid = ids[i];
            if (vid == -1) break;
            const float d = ds[i];
            if (lane == 0 && !isfinite(d)) atomicExch(p.bad, 1);
            const unsigned char* row_i = p.rows + (size_t)vid * p.row_stride;
            // ComputeDistance(head_i, head_j) for the accepted heads, two at a time (one per half-warp)
            bool reject = false;
            for (int a0 = 0; a0 < n_acc && !reject; a0 += 2) {
                const int a = min(a0 + half, n_acc - 1);
                const float nd = spann_distance<COSINE, ELEM>(p.rows + (size_t)acc[a] * p.row_stride, row_i, p.dim, j,
                                                              p.simd_width);
                const bool mine = j == 0 && a0 + half < n_acc;
                if (mine && !isfinite(nd)) atomicExch(p.bad, 1);
                reject = __any_sync(kFull, mine && __fmul_rn(p.rng_factor, nd) < d);
            }
            if (reject) {
                ++rejected;
                continue;
            }
            if (lane == 0) {
                acc[n_acc] = vid;
                p.keys[slot0 + n_acc] = ((unsigned long long)vid << 32) | order_bits(d);
                p.tonode[slot0 + n_acc] = v;
                atomicAdd(p.list_size + vid, 1);
            }
            __syncwarp();
            ++n_acc;
        }
    }
    for (int s = n_acc + lane; s < p.replicas; s += 32) {  // Edge(): after every list
        p.keys[slot0 + s] = (unsigned long long)p.num_heads << 32;
        p.tonode[slot0 + s] = v;
    }
    if (lane == 0 && rejected) atomicAdd(p.rejected, rejected);
}

__global__ void spann_nonfinite_kernel(const float* __restrict__ v, size_t n, int* bad) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (!isfinite(v[i])) *bad = 1;
}

// One block per list that overlaps the window, one byte per thread and step.  GATHERED: element e of list l reads its row
// from row row_off[l] + e of the gathered rows, not from the vector's own row
template <bool GATHERED>
__device__ __forceinline__ void posting_image(const SpannImageParams& p) {
    const long long rb = p.row_bytes, vis = rb + 4;
    for (int li = blockIdx.x; li < p.num_lists; li += gridDim.x) {
        const int l = p.first_list + li;
        const long long s = p.start[l], cnt = p.count[l];
        const long long lo = max(s, p.win_begin), hi = min(s + cnt * vis, p.win_end);
        const int* ton = p.tonode + p.edge_off[l];
        for (long long b = lo + threadIdx.x; b < hi; b += blockDim.x) {
            const long long o = b - s;
            long long e, at;
            bool id;
            if (p.rearranged) {
                id = o >= cnt * rb;
                e = id ? (o - cnt * rb) >> 2 : o / rb;
                at = id ? (o - cnt * rb) & 3 : o - e * rb;
            } else {
                e = o / vis;
                at = o - e * vis;
                id = at < 4;
                if (!id) at -= 4;
            }
            const int vec = ton[e];
            const size_t row = GATHERED ? (size_t)(p.row_off[l] + e) : (size_t)vec;
            p.out[b - p.win_begin] = id ? (unsigned char)((unsigned int)vec >> (8 * at)) : p.rows[row * rb + at];
        }
    }
}

__global__ void __launch_bounds__(256) spann_posting_image_kernel(const SpannImageParams p) { posting_image<false>(p); }
__global__ void __launch_bounds__(256) spann_posting_image_gathered_kernel(const SpannImageParams p) { posting_image<true>(p); }

// One thread per edge: flags[i] = the edge is kept.  group_of == nullptr: the edge is filled (node < num_heads), and
// tonode[i] += tonode_add; otherwise: its list belongs to `group`
__global__ void spann_edge_flag_kernel(const unsigned long long* __restrict__ keys, int* __restrict__ tonode, int n,
                                       int tonode_add, int num_heads, const int* __restrict__ group_of, int group,
                                       unsigned char* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int node = (int)(keys[i] >> 32);
    if (group_of) {
        flags[i] = group_of[node] == group;
    } else {
        flags[i] = node < num_heads;
        tonode[i] += tonode_add;
    }
}

// One block per list, one word of W per thread and step: the list's first count[l] sorted edges' rows, from src (row
// tonode[e], row_bytes apart) to dst (row row_off[l] + e)
template <typename W>
__global__ void __launch_bounds__(256) spann_row_gather_kernel(const SpannGatherParams p) {
    const int wpr = p.row_bytes / (int)sizeof(W);
    const W* src = reinterpret_cast<const W*>(p.src);
    W* dst = reinterpret_cast<W*>(p.dst);
    for (int li = blockIdx.x; li < p.num_lists; li += gridDim.x) {
        const int l = p.first_list + li;
        const int* ton = p.tonode + p.edge_off[l];
        W* out = dst + (size_t)p.row_off[l] * wpr;
        const long long words = (long long)p.count[l] * wpr;
        for (long long t = threadIdx.x; t < words; t += blockDim.x) {
            const long long e = t / wpr;
            out[t] = src[(size_t)ton[e] * wpr + (t - e * wpr)];
        }
    }
}

}  // namespace

cudaError_t launch_spann_rng_select(const SpannRngParams& p, bool cosine, int elem, cudaStream_t stream) {
    if (p.num <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)((p.num + kRngWarps - 1) / kRngWarps);
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        spann_rng_select_kernel<cos, el><<<grid, 32 * kRngWarps, 0, stream>>>(p);
        return cudaGetLastError();
    });
}

cudaError_t launch_spann_nonfinite_check(const float* v, size_t n, int* bad, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, 4096);
    spann_nonfinite_kernel<<<grid, 256, 0, stream>>>(v, n, bad);
    return cudaGetLastError();
}

cudaError_t spann_sort_edges(void* temp, size_t* temp_bytes, const unsigned long long* keys_in, unsigned long long* keys_out,
                             const int* tonode_in, int* tonode_out, int n, int end_bit, cudaStream_t stream) {
    return cub::DeviceRadixSort::SortPairs(temp, *temp_bytes, keys_in, keys_out, tonode_in, tonode_out, n, 0, end_bit,
                                           stream);
}

cudaError_t launch_spann_posting_image(const SpannImageParams& p, cudaStream_t stream) {
    if (p.num_lists <= 0) return cudaSuccess;
    if (p.row_off)
        spann_posting_image_gathered_kernel<<<(unsigned)std::min(p.num_lists, 65535), 256, 0, stream>>>(p);
    else
        spann_posting_image_kernel<<<(unsigned)std::min(p.num_lists, 65535), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t spann_select_edges(void* temp, size_t* temp_bytes, const unsigned long long* keys, int* tonode, int n,
                               int tonode_add, int num_heads, const int* group_of, int group, unsigned char* flags,
                               unsigned long long* keys_out, int* tonode_out, int* num_selected, cudaStream_t stream) {
    if (!temp) {
        size_t a = 0, b = 0;
        cudaError_t e = cub::DeviceSelect::Flagged(nullptr, a, keys, flags, keys_out, num_selected, n, stream);
        if (e == cudaSuccess) e = cub::DeviceSelect::Flagged(nullptr, b, tonode, flags, tonode_out, num_selected, n, stream);
        *temp_bytes = std::max(a, b);
        return e;
    }
    if (n <= 0) return cudaMemsetAsync(num_selected, 0, 4, stream);
    spann_edge_flag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(keys, tonode, n, tonode_add, num_heads, group_of,
                                                                           group, flags);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceSelect::Flagged(temp, *temp_bytes, keys, flags, keys_out, num_selected, n, stream);
    if (e == cudaSuccess)
        e = cub::DeviceSelect::Flagged(temp, *temp_bytes, (const int*)tonode, flags, tonode_out, num_selected, n, stream);
    return e;
}

cudaError_t launch_spann_row_gather(const SpannGatherParams& p, cudaStream_t stream) {
    if (p.num_lists <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)std::min(p.num_lists, 65535);
    // the widest word that divides the row size and both bases' alignment
    const size_t align = (size_t)p.row_bytes | (size_t)(uintptr_t)p.src | (size_t)(uintptr_t)p.dst;
    if (align % 16 == 0)
        spann_row_gather_kernel<uint4><<<grid, 256, 0, stream>>>(p);
    else if (align % 8 == 0)
        spann_row_gather_kernel<uint2><<<grid, 256, 0, stream>>>(p);
    else if (align % 4 == 0)
        spann_row_gather_kernel<unsigned int><<<grid, 256, 0, stream>>>(p);
    else if (align % 2 == 0)
        spann_row_gather_kernel<unsigned short><<<grid, 256, 0, stream>>>(p);
    else
        spann_row_gather_kernel<unsigned char><<<grid, 256, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace sptag_b200
