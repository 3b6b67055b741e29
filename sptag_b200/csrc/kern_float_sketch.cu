// float rows, BKT, with the row-sketch test in the graph step (search_kernels.cuh compute_dists_gated)
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_sketch_kernel<true>(int, int);
template SearchKernelFn pick_sketch_kernel<false>(int, int);
}  // namespace sptag_b200
