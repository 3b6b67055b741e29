// kern_bfs_int_impl.cuh -- integer-row instantiations of bfs::search_kernel (included by kern_bfs_int8.cu /
// kern_bfs_int16.cu): pick_int's BKT kernels with breadth-first tree seeding
#pragma once
#include "kernel_select.h"
#include "search_kernels.cuh"

namespace sptag_b200 {

// ELEM 1 int8, 2 uint8, 3 int16
template <bool COSINE, int ELEM>
static SearchKernelFn pick_int_bfs(int mres_cap) {
    if (mres_cap <= 32 * 16) return bfs::search_kernel<0, COSINE, 16, false, false, ELEM>;
    if (mres_cap <= 32 * 32) return bfs::search_kernel<0, COSINE, 32, false, false, ELEM, 12>;
    if (mres_cap <= 32 * 64) return bfs::search_kernel<0, COSINE, 64, false, false, ELEM, 8>;
    return nullptr;
}

}  // namespace sptag_b200
