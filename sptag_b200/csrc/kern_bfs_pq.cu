// EnableBfs != 0: PQ / OPQ code rows with breadth-first tree seeding, at pick_pq_kernel's register caps (see
// kern_bfs_float.cu for why a unit of its own)
#include "kernel_select.h"
#include "search_kernels.cuh"
namespace sptag_b200 {
SearchKernelFn pick_pq_bfs_kernel(int mres_cap) {
    if (mres_cap <= 32 * 16) return bfs::search_kernel<0, false, 16, false, true, 0, 24>;
    if (mres_cap <= 32 * 32) return bfs::search_kernel<0, false, 32, false, true, 0, 16>;
    return nullptr;
}
}  // namespace sptag_b200
