// EnableBfs != 0: SearchIndexIterativeFromNeareast's first call with breadth-first tree seeding (see kern_bfs_float.cu
// for why a unit of its own)
#include "kernel_select.h"
#include "search_kernels.cuh"
#include "../../include/sptag_b200.h"
namespace sptag_b200 {
template <bool COSINE, int ELEM>
static NearestFirstKernelFn pick_nearest_rpl(int mres_cap) {
    if (mres_cap <= 32 * 16) return bfs::nearest_first_kernel<COSINE, 16, ELEM>;
    if (mres_cap <= 32 * 32) return bfs::nearest_first_kernel<COSINE, 32, ELEM>;
    return nullptr;
}
NearestFirstKernelFn pick_nearest_first_bfs_kernel_for(int value_type, bool cosine, int mres_cap) {
    switch (value_type) {
    case SPTAG_B200_VT_FLOAT: return cosine ? pick_nearest_rpl<true, 0>(mres_cap) : pick_nearest_rpl<false, 0>(mres_cap);
    case SPTAG_B200_VT_INT8: return cosine ? pick_nearest_rpl<true, 1>(mres_cap) : pick_nearest_rpl<false, 1>(mres_cap);
    case SPTAG_B200_VT_UINT8: return cosine ? pick_nearest_rpl<true, 2>(mres_cap) : pick_nearest_rpl<false, 2>(mres_cap);
    case SPTAG_B200_VT_INT16: return cosine ? pick_nearest_rpl<true, 3>(mres_cap) : pick_nearest_rpl<false, 3>(mres_cap);
    default: return nullptr;
    }
}
}  // namespace sptag_b200
