// EnableBfs != 0: int16 rows with breadth-first tree seeding (see kern_bfs_float.cu for why a unit of its own)
#include "kern_bfs_int_impl.cuh"
namespace sptag_b200 {
SearchKernelFn pick_int16_bfs_kernel(bool cosine, int mres_cap) {
    return cosine ? pick_int_bfs<true, 3>(mres_cap) : pick_int_bfs<false, 3>(mres_cap);
}
}  // namespace sptag_b200
