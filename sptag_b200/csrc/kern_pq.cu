// PQ / OPQ code rows: SDC / ADC table look-ups (PQQuantizer.h:110-128)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_pq_kernel<false>(int);
}  // namespace sptag_b200
