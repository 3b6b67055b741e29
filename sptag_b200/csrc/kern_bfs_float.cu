// EnableBfs != 0: float rows of every dimension with breadth-first tree seeding (BKTree.h:703-758), on the
// generic-dimension kernels at pick_rpl's register caps.  The BFS instantiations live in units of their own
// (kern_bfs_*.cu): kernels of one unit share the compiled form of the out-of-line helpers (heap_full_slot, vhash_*), so
// a BFS kernel next to the others can change their code.
#include "kernel_select.h"
#include "search_kernels.cuh"
namespace sptag_b200 {
template <bool COSINE>
static SearchKernelFn pick_bfs_rpl(int mres_cap) {
    if (mres_cap <= 32 * 16) return bfs::search_kernel<0, COSINE, 16, false, false, 0, 12>;
    if (mres_cap <= 32 * 32) return bfs::search_kernel<0, COSINE, 32, false, false, 0, 14>;
    if (mres_cap <= 32 * 64) return bfs::search_kernel<0, COSINE, 64, false, false, 0, 8>;
    return nullptr;
}
SearchKernelFn pick_float_bfs_kernel_l2(int mres_cap) { return pick_bfs_rpl<false>(mres_cap); }
SearchKernelFn pick_float_bfs_kernel_cosine(int mres_cap) { return pick_bfs_rpl<true>(mres_cap); }
}  // namespace sptag_b200
