// int16 rows (DistanceUtils.cpp:559-596, :930-967)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_int_kernel<false, 3>(bool, int, bool);
}  // namespace sptag_b200
