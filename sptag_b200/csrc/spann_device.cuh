// spann_device.cuh -- device pieces shared by the SPANN posting scan (kern_spann.cu) and the posting step of SPANN
// iterators (kern_spann_iter.cu): QueryResultSet's comparator and Heapify, the distance, LoadingHeadInfo's truncation.
#pragma once
#include "search_kernels.cuh"

namespace sptag_b200 {
namespace {

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
