// kernel_select.h -- which instantiation of the search kernels serves an index / parameter set.
//
// The kernel templates (search_kernels.cuh) are instantiated in several translation units (kern_*.cu) so that nvcc can
// compile them in parallel; each unit exports one selector that returns the host-side launch stub of the instantiation
// (nullptr: this m_Results capacity / combination is not built).  sptag_b200.cu launches through these pointers.
#pragma once

namespace sptag_b200 {

struct SearchParams;
struct IterVisited;
typedef void (*SearchKernelFn)(const SearchParams);
typedef void (*IterateKernelFn)(const SearchParams, int*, int*, unsigned char*, const IterVisited);
typedef void (*NearestFirstKernelFn)(const SearchParams, int*, const IterVisited);

// float rows; dim 128 / 768 select the register-resident query variants
// slots: query slots per SM the host aims at (512-byte rows: register-capped variants above 16)
SearchKernelFn pick_float_kernel_l2(int dim, int mres_cap, bool kdt, int slots);
SearchKernelFn pick_float_kernel_cosine(int dim, int mres_cap, bool kdt, int slots);
// value_type: SPTAG_B200_VT_INT8 / UINT8 / INT16
SearchKernelFn pick_int8_kernel(bool is_unsigned, bool cosine, int mres_cap, bool kdt);
SearchKernelFn pick_int16_kernel(bool cosine, int mres_cap, bool kdt);
// PQ / OPQ codes (BKT + L2 only, PQQuantizer.h:130-136)
SearchKernelFn pick_pq_kernel(int mres_cap);
// ResultIterator::Next and SearchIndexIterativeFromNeareast's first call; value_type as in include/sptag_b200.h
IterateKernelFn pick_iterate_kernel_for(int value_type, bool cosine, int mres_cap);
NearestFirstKernelFn pick_nearest_first_kernel_for(int value_type, bool cosine, int mres_cap);
// EnableBfs != 0 (BKT only): the same families with breadth-first tree seeding.  Float rows of every dimension take the
// generic-dimension instantiations (no 128- / 768-d specialisation).
SearchKernelFn pick_float_bfs_kernel_l2(int mres_cap);
SearchKernelFn pick_float_bfs_kernel_cosine(int mres_cap);
SearchKernelFn pick_int8_bfs_kernel(bool is_unsigned, bool cosine, int mres_cap);
SearchKernelFn pick_int16_bfs_kernel(bool cosine, int mres_cap);
SearchKernelFn pick_pq_bfs_kernel(int mres_cap);
IterateKernelFn pick_iterate_bfs_kernel_for(int value_type, bool cosine, int mres_cap);
NearestFirstKernelFn pick_nearest_first_bfs_kernel_for(int value_type, bool cosine, int mres_cap);

}  // namespace sptag_b200
