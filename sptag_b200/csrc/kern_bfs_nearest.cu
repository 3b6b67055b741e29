// EnableBfs != 0: SearchIndexIterativeFromNeareast's first call with breadth-first tree seeding (see kern_bfs_float.cu
// for why a unit of its own)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template NearestFirstKernelFn pick_iter_kernel<NearestFirstKernelFn, true>(int, bool, int);
}  // namespace sptag_b200
