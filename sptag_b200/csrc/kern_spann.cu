// SPANN posting scan on raw rows (SPANN::Index<T>::SearchIndex after its head search, ExtraFullGraphSearcher<T>): the
// body of spann_scan_body (spann_device.cuh) with the head index's DistanceUtils tree, a half-warp per row.
#include "spann_device.cuh"
#include "spann_scan.h"

namespace sptag_b200 {
namespace {

template <bool COSINE, int ELEM>
struct RowDistance {
    const unsigned char* qrow;
    int j, half;  // the lane's place in its half-warp, and which half-warp

    __device__ __forceinline__ void begin_query(const SpannScanParams& p, int q) { qrow = p.queries + (size_t)q * p.row_stride; }

    __device__ __forceinline__ void chunk(const SpannScanParams& p, int l, const int* cl, int cnt, float* cd) {
        for (int r0 = 0; r0 < cnt; r0 += 2) {
            const int r = min(r0 + half, cnt - 1);
            const unsigned char* row = p.rows + (size_t)(p.off[l] + cl[r]) * p.row_stride;
            const float d = spann_distance<COSINE, ELEM>(row, qrow, p.dim, j, p.simd_width);
            if (j == 0 && r0 + half < cnt) cd[r] = d;
        }
    }
};

template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32) spann_scan_kernel(const SpannScanParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    RowDistance<COSINE, ELEM> dist{nullptr, (int)threadIdx.x & 15, (int)threadIdx.x >> 4};
    spann_scan_body(p, smem, dist);
}

}  // namespace

int spann_scan_blocks_per_sm(bool cosine, int elem, int w) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        return warp_blocks_per_sm((const void*)spann_scan_kernel<cos, el>, spann_scan_smem(w));
    });
}

cudaError_t launch_spann_scan(const SpannScanParams& p, bool cosine, int elem, int grid, cudaStream_t stream) {
    const size_t smem = spann_scan_smem(p.w);
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        void (*k)(const SpannScanParams) = spann_scan_kernel<cos, el>;
        if (smem > 48 * 1024) {
            cudaError_t e = cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        k<<<grid, 32, smem, stream>>>(p);
        return cudaGetLastError();
    });
}


}  // namespace sptag_b200
