// EnableBfs != 0: ResultIterator::Next with breadth-first tree seeding at the first call (see kern_bfs_float.cu for why a
// unit of its own)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template IterateKernelFn pick_iter_kernel<IterateKernelFn, true>(int, bool, int);
}  // namespace sptag_b200
