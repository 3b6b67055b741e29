// int8 / uint8 rows (DistanceUtils.cpp:363-400, :460-496, :744-780, :838-874)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_int_kernel<false, 1>(bool, int, bool);
template SearchKernelFn pick_int_kernel<false, 2>(bool, int, bool);
}  // namespace sptag_b200
