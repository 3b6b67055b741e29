// float rows, cosine / inner product as 1 - dot (DistanceUtils.cpp:1016-1046)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_float_kernel<false, true>(int, int, bool, int);
}  // namespace sptag_b200
