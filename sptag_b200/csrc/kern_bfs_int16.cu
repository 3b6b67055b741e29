// EnableBfs != 0: int16 rows with breadth-first tree seeding (see kern_bfs_float.cu for why a unit of its own)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_int_kernel<true, 3>(bool, int, bool);
}  // namespace sptag_b200
