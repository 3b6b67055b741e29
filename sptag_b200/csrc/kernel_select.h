// kernel_select.h -- which instantiation of the search kernels serves an index / parameter set.
//
// The kernel templates (search_kernels.cuh) are instantiated in several translation units (kern_*.cu) so that nvcc can
// compile them in parallel; each unit explicitly instantiates the selectors below (kernel_select_impl.cuh) for the
// kernels it owns.  A selector returns the host-side launch stub of the instantiation (nullptr: this m_Results capacity /
// combination is not built).  sptag_b200.cu launches through these pointers.
//
// BFS: EnableBfs != 0 (BKT only), the same families with breadth-first tree seeding, in kern_bfs_*.cu.  Float rows of
// every dimension take the generic-dimension instantiations (no 128- / 768-d specialisation), and kdt / slots are unused.
#pragma once

namespace sptag_b200 {

struct SearchParams;
struct IterVisited;
typedef void (*SearchKernelFn)(const SearchParams);
typedef void (*IterateKernelFn)(const SearchParams, int*, int*, unsigned char*, const IterVisited);
typedef void (*NearestFirstKernelFn)(const SearchParams, int*, const IterVisited);

// float rows; dim 128 / 768 select the register-resident query variants
// slots: query slots per SM the host aims at (512-byte rows: register-capped variants above 16)
template <bool BFS, bool COSINE>
SearchKernelFn pick_float_kernel(int dim, int mres_cap, bool kdt, int slots);
// float rows, BKT: the sketch:: kernels, which test a graph candidate's row sketch before they fetch its row
// (SearchParams::sketch must be bound); dim 768 selects the unrolled variant
template <bool COSINE>
SearchKernelFn pick_sketch_kernel(int dim, int mres_cap);
// ELEM 1 int8, 2 uint8, 3 int16
template <bool BFS, int ELEM>
SearchKernelFn pick_int_kernel(bool cosine, int mres_cap, bool kdt);
// PQ / OPQ codes (BKT + L2 only, PQQuantizer.h:130-136)
template <bool BFS>
SearchKernelFn pick_pq_kernel(int mres_cap);
// Fn = IterateKernelFn: ResultIterator::Next; Fn = NearestFirstKernelFn: SearchIndexIterativeFromNeareast's first call.
// value_type as in include/sptag_b200.h
template <typename Fn, bool BFS>
Fn pick_iter_kernel(int value_type, bool cosine, int mres_cap);

}  // namespace sptag_b200
