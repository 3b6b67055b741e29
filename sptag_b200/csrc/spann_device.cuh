// spann_device.cuh -- pieces shared by the posting-side kernels: the SPANN posting scan (kern_spann.cu), the posting
// step of SPANN iterators (kern_spann_iter.cu) and the multi-index scan's cross distances (kern_multi_scan.cu).
// QueryResultSet's comparator and Heapify, the distance, LoadingHeadInfo's truncation, and the launchers' dispatch.
#pragma once
#include "search_kernels.cuh"

#include <type_traits>

namespace sptag_b200 {
namespace {

// Calls f(cos, el) with the runtime metric flag and element code (0 float, 1 int8, 2 uint8, 3 int16) as compile-time
// constants (std::bool_constant, std::integral_constant<int, ELEM>), so that f can name its kernel's <COSINE, ELEM>
// instantiation
template <typename F>
auto with_cosine_elem(bool cosine, int elem, F&& f) {
    using T = std::true_type;
    using N = std::false_type;
    switch (elem) {
    case 1: return cosine ? f(T(), std::integral_constant<int, 1>()) : f(N(), std::integral_constant<int, 1>());
    case 2: return cosine ? f(T(), std::integral_constant<int, 2>()) : f(N(), std::integral_constant<int, 2>());
    case 3: return cosine ? f(T(), std::integral_constant<int, 3>()) : f(N(), std::integral_constant<int, 3>());
    default: return cosine ? f(T(), std::integral_constant<int, 0>()) : f(N(), std::integral_constant<int, 0>());
    }
}

// Blocks of one warp of kernel k with smem bytes of dynamic shared memory that fit on one SM (0: none, or the query
// failed)
inline int warp_blocks_per_sm(const void* k, size_t smem) {
    int fit = 0;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, k, 32, smem) != cudaSuccess) return 0;
    return fit;
}

// BasicResult operator< (QueryResultSet.h:17-20)
__device__ __forceinline__ bool res_less(float da, int va, float db, int vb) {
    return da < db || (da == db && va < vb);
}

// QueryResultSet::Heapify(count) on (dist, vid) arrays, exactly as written (QueryResultSet.h:99-112)
__device__ void heapify(float* d, int* v, int count) {
    int parent = 0, next = 1;
    const int maxidx = count - 1;
    while (next < maxidx) {
        if (res_less(d[next], v[next], d[next + 1], v[next + 1])) next++;
        if (res_less(d[parent], v[parent], d[next], v[next])) {
            const float td = d[next];
            const int tv = v[next];
            d[next] = d[parent];
            v[next] = v[parent];
            d[parent] = td;
            v[parent] = tv;
            parent = next;
            next = (parent << 1) + 1;
        } else {
            break;
        }
    }
    if (next == maxidx && res_less(d[parent], v[parent], d[next], v[next])) {
        const float td = d[next];
        const int tv = v[next];
        d[next] = d[parent];
        v[next] = v[parent];
        d[parent] = td;
        v[parent] = tv;
    }
}

// ComputeDistance(query, row) by one half-warp with the trees of the search kernels (both are symmetric bit for bit)
template <bool COSINE, int ELEM>
__device__ __forceinline__ float spann_distance(const unsigned char* row, const unsigned char* q, int dim, int j,
                                                int simd_width) {
    if (ELEM == 0) {
        QueryRegs<0> qr;
        if (simd_width != 16)
            return half_warp_distance_w<COSINE>(reinterpret_cast<const float*>(row), reinterpret_cast<const float*>(q), dim, j,
                                                simd_width);
        return half_warp_distance<0, COSINE>(reinterpret_cast<const float*>(row), qr, reinterpret_cast<const float*>(q), dim, j);
    }
    return half_warp_distance_elem_w<COSINE, ELEM>(row, q, dim, j, simd_width);
}

// LoadingHeadInfo's truncation (ExtraFullGraphSearcher.h:1093-1097)
template <typename Params>
__device__ __forceinline__ int searched_count(const Params& p, int l) {
    const long long lim = (long long)min(p.pages[l], p.page_limit) << 12;
    return (int)min((long long)p.cnt[l], lim / p.vector_info_size);
}

}  // namespace
}  // namespace sptag_b200
