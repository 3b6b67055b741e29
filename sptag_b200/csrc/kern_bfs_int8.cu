// EnableBfs != 0: int8 / uint8 rows with breadth-first tree seeding (see kern_bfs_float.cu for why a unit of its own)
#include "kern_bfs_int_impl.cuh"
namespace sptag_b200 {
SearchKernelFn pick_int8_bfs_kernel(bool is_unsigned, bool cosine, int mres_cap) {
    if (is_unsigned) return cosine ? pick_int_bfs<true, 2>(mres_cap) : pick_int_bfs<false, 2>(mres_cap);
    return cosine ? pick_int_bfs<true, 1>(mres_cap) : pick_int_bfs<false, 1>(mres_cap);
}
}  // namespace sptag_b200
