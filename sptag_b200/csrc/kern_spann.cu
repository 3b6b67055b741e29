// SPANN posting scan on raw rows (SPANN::Index<T>::SearchIndex after its head search, ExtraFullGraphSearcher<T>): the
// body of spann_scan_body (spann_device.cuh) with RowDistance, the head index's DistanceUtils tree, a half-warp per row.
#include "spann_device.cuh"
#include "spann_scan.h"

namespace sptag_b200 {
namespace {

template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32) spann_scan_kernel(const SpannScanParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    RowDistance<COSINE, ELEM> dist{nullptr, p.dim, p.simd_width, (int)threadIdx.x & 15, (int)threadIdx.x >> 4};
    spann_scan_body(p, smem, dist);
}

}  // namespace

int spann_scan_blocks_per_sm(bool cosine, int elem, int w) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        return warp_blocks_per_sm((const void*)spann_scan_kernel<cos, el>, spann_scan_smem(w));
    });
}

cudaError_t launch_spann_scan(const SpannScanParams& p, bool cosine, int elem, int grid, cudaStream_t stream,
                              const void** kernel) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        *kernel = (const void*)spann_scan_kernel<cos, el>;
        return launch_warp_blocks(spann_scan_kernel<cos, el>, p, grid, spann_scan_smem(p.w), stream);
    });
}

}  // namespace sptag_b200
