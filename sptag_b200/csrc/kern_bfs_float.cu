// EnableBfs != 0: float rows of every dimension with breadth-first tree seeding (BKTree.h:703-758), on the
// generic-dimension kernels.  The BFS instantiations live in units of their own (kern_bfs_*.cu): kernels of one unit
// share the compiled form of the out-of-line helpers (heap_full_slot, vhash_*), so a BFS kernel next to the others can
// change their code.
#include "kernel_select_impl.cuh"
namespace sptag_b200 {
template SearchKernelFn pick_float_kernel<true, false>(int, int, bool, int);
template SearchKernelFn pick_float_kernel<true, true>(int, int, bool, int);
}  // namespace sptag_b200
