// EnableBfs != 0: PQ / OPQ code rows with breadth-first tree seeding (see kern_bfs_float.cu for why a unit of its
// own)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_pq_kernel<true>(int);
}  // namespace sptag_b200
