// SearchIndexIterativeFromNeareast, first call (BKTIndex.cpp:543-573)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template NearestFirstKernelFn pick_iter_kernel<NearestFirstKernelFn, false>(int, bool, int);
}  // namespace sptag_b200
