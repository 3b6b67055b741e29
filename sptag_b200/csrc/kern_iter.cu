// ResultIterator::Next for a batch of open iterators (BKTIndex.cpp:354-427)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template IterateKernelFn pick_iter_kernel<IterateKernelFn, false>(int, bool, int);
}  // namespace sptag_b200
