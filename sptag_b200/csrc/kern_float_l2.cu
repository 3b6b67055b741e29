// float rows, squared L2 (DistanceUtils.cpp:650-682)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_float_kernel<false, false>(int, int, bool, int);
}  // namespace sptag_b200
