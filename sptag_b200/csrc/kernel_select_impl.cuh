// kernel_select_impl.cuh -- the selectors of kernel_select.h, each family's tiers written once for both seedings
// (included by kern_*.cu, each of which instantiates the selectors it owns).
//
// BFS = true names the bfs:: kernels (EnableBfs's breadth-first tree seeding, BKT only): float rows of every dimension
// take the generic-dimension instantiations, and there are no KDT or slot-capped variants.  Kernels of one unit share
// the compiled form of the out-of-line helpers (heap_full_slot, vhash_*), so a unit must instantiate exactly the kernels
// it owns: every choice between a plain and a bfs:: kernel is an `if constexpr`, which leaves the other one
// uninstantiated (a ternary or a plain `if` would instantiate both in every unit and change their code).
#pragma once
#include <type_traits>
#include "kernel_select.h"
#include "search_kernels.cuh"
#include "../../include/sptag_b200.h"

namespace sptag_b200 {

template <bool BFS, int DIM, bool COSINE, int RPL, bool KDT, bool PQ = false, int ELEM = 0, int MINB = 1>
static SearchKernelFn search_fn() {
    if constexpr (BFS) return bfs::search_kernel<DIM, COSINE, RPL, KDT, PQ, ELEM, MINB>;
    else return search_kernel<DIM, COSINE, RPL, KDT, PQ, ELEM, MINB>;
}

template <bool BFS, int DIM, bool COSINE>
static SearchKernelFn pick_rpl(int mres_cap, bool kdt, int slots) {
    if constexpr (!BFS) {
        if (kdt) {  // KDT has no m_Results gate
            if constexpr (DIM == 128) {
                if (slots > 16) return search_kernel<DIM, COSINE, 16, true, false, 0, 20>;
            }
            return search_kernel<DIM, COSINE, 16, true>;
        }
    }
    // register caps (MINB resident single-warp CTAs per SM): 12 -> 168 registers; the kernel is latency-bound per
    // warp, so residency beats a few spilled values (refine passes run the 32-register m_Results file, K = CEF+1)
    if (mres_cap <= 32 * 16) return search_fn<BFS, DIM, COSINE, 16, false, false, 0, 12>();
    if (mres_cap <= 32 * 32) return search_fn<BFS, DIM, COSINE, 32, false, false, 0, 14>();
    // 64 registers per lane: K / CEF+1 up to 2048 (the reference's default RefineGraph schedule searches with
    // CEF x CEFScale + 1 = 2001 results, NeighborhoodGraph.h:459-470)
    if (mres_cap <= 32 * 64) return search_fn<BFS, DIM, COSINE, 64, false, false, 0, 8>();
    return nullptr;
}

// slots: the residency (query slots per SM) the host is aiming at; 512-byte rows have a register-capped variant for up to
// 20 slots (96 registers, 4 bytes of spills; a 24-slot / 80-register variant was slower)
template <bool BFS, bool COSINE>
SearchKernelFn pick_float_kernel(int dim, int mres_cap, bool kdt, int slots) {
    if constexpr (!BFS) {
        switch (dim) {
        case 128:
            if (!kdt && mres_cap <= 32 * 16) {
                if (slots > 16) return search_kernel<128, COSINE, 16, false, false, 0, 20>;
                return search_kernel<128, COSINE, 16, false, false, 0, 16>;  // 128 regs, 16/SM
            }
            return pick_rpl<BFS, 128, COSINE>(mres_cap, kdt, slots);
        case 768:
            // 15 resident queries per SM (127 registers, no spills) when the m_Results file is the 16-register one
            if (!kdt && mres_cap <= 32 * 16) return search_kernel<768, COSINE, 16, false, false, 0, 15>;
            return pick_rpl<BFS, 768, COSINE>(mres_cap, kdt, slots);
        }
    }
    return pick_rpl<BFS, 0, COSINE>(mres_cap, kdt, slots);
}

// 12 slots per SM (168 registers, no spills with the 16- and 32-register m_Results files): what lay_out runs rows of
// 2 KB or more at.  (A 128-register form of the 768-d kernel spills 330 bytes and was 19 % slower at 13 to 16 slots.)
template <int DIM, bool COSINE>
static SearchKernelFn pick_sketch_rpl(int mres_cap) {
    if (mres_cap <= 32 * 16) return sketch::search_kernel<DIM, COSINE, 16, false, false, 0, 12>;
    if (mres_cap <= 32 * 32) return sketch::search_kernel<DIM, COSINE, 32, false, false, 0, 12>;
    if (mres_cap <= 32 * 64) return sketch::search_kernel<DIM, COSINE, 64, false, false, 0, 8>;
    return nullptr;
}
template <bool COSINE>
SearchKernelFn pick_sketch_kernel(int dim, int mres_cap) {
    return dim == 768 ? pick_sketch_rpl<768, COSINE>(mres_cap) : pick_sketch_rpl<0, COSINE>(mres_cap);
}

template <bool BFS, bool COSINE, int ELEM>
static SearchKernelFn pick_int_rpl(int mres_cap, bool kdt) {
    if constexpr (!BFS) {
        if (kdt) return search_kernel<0, COSINE, 16, true, false, ELEM>;
    }
    if (mres_cap <= 32 * 16) return search_fn<BFS, 0, COSINE, 16, false, false, ELEM>();
    if (mres_cap <= 32 * 32) return search_fn<BFS, 0, COSINE, 32, false, false, ELEM, 12>();
    if (mres_cap <= 32 * 64) return search_fn<BFS, 0, COSINE, 64, false, false, ELEM, 8>();
    return nullptr;
}

template <bool BFS, int ELEM>
SearchKernelFn pick_int_kernel(bool cosine, int mres_cap, bool kdt) {
    return cosine ? pick_int_rpl<BFS, true, ELEM>(mres_cap, kdt) : pick_int_rpl<BFS, false, ELEM>(mres_cap, kdt);
}

template <bool BFS>
SearchKernelFn pick_pq_kernel(int mres_cap) {
    if (mres_cap <= 32 * 16) return search_fn<BFS, 0, false, 16, false, true, 0, 24>();
    if (mres_cap <= 32 * 32) return search_fn<BFS, 0, false, 32, false, true, 0, 16>();
    return nullptr;
}

template <typename Fn, bool BFS, bool COSINE, int RPL, int ELEM>
static Fn iter_fn() {
    if constexpr (std::is_same<Fn, IterateKernelFn>::value) {
        if constexpr (BFS) return bfs::iterate_kernel<COSINE, RPL, ELEM>;
        else return iterate_kernel<COSINE, RPL, ELEM>;
    } else {
        if constexpr (BFS) return bfs::nearest_first_kernel<COSINE, RPL, ELEM>;
        else return nearest_first_kernel<COSINE, RPL, ELEM>;
    }
}

template <typename Fn, bool BFS, bool COSINE, int ELEM>
static Fn pick_iter_rpl(int mres_cap) {
    if (mres_cap <= 32 * 16) return iter_fn<Fn, BFS, COSINE, 16, ELEM>();
    if (mres_cap <= 32 * 32) return iter_fn<Fn, BFS, COSINE, 32, ELEM>();
    return nullptr;
}

template <typename Fn, bool BFS>
Fn pick_iter_kernel(int value_type, bool cosine, int mres_cap) {
    switch (value_type) {
    case SPTAG_B200_VT_FLOAT: return cosine ? pick_iter_rpl<Fn, BFS, true, 0>(mres_cap) : pick_iter_rpl<Fn, BFS, false, 0>(mres_cap);
    case SPTAG_B200_VT_INT8: return cosine ? pick_iter_rpl<Fn, BFS, true, 1>(mres_cap) : pick_iter_rpl<Fn, BFS, false, 1>(mres_cap);
    case SPTAG_B200_VT_UINT8: return cosine ? pick_iter_rpl<Fn, BFS, true, 2>(mres_cap) : pick_iter_rpl<Fn, BFS, false, 2>(mres_cap);
    case SPTAG_B200_VT_INT16: return cosine ? pick_iter_rpl<Fn, BFS, true, 3>(mres_cap) : pick_iter_rpl<Fn, BFS, false, 3>(mres_cap);
    default: return nullptr;
    }
}

}  // namespace sptag_b200
