// search_kernels.cuh -- sm_90a device code of the batched search hot path.
//
// One warp (one 32-thread CTA) owns one query at a time and runs the reference's whole
// per-query algorithm on the device:
//   BKT::Index<T>::Search            (AnnService/src/Core/BKT/BKTIndex.cpp:268-352, incl. the filter variant :622-647)
//   BKTree::InitSearchTrees/SearchTrees (inc/Core/Common/BKTree.h:696-799)
//   KDT::Index<T>::Search, KDTree::KDTSearch (src/Core/KDT/KDTIndex.cpp:182-241, inc/Core/Common/KDTree.h:213-271)
//   Heap<NodeDistPair>               (inc/Core/Common/Heap.h:13-106)      -> exact binary-heap emulation
//   DistPriorityQueue m_Results      (inc/Core/Common/WorkSpace.h:167-225) -> multiset in registers
//   OptHashPosVector visited set     (inc/Core/Common/WorkSpace.h:43-165) -> exact bitmap in HBM/L2
//   QueryResultSet top-K             (inc/Core/Common/QueryResultSet.h:17-120) -> sorted list, one entry per lane
//                                     (K <= 32) or the reference's own max-heap in HBM (K <= 1024)
//   DistanceUtils float / int8 / uint8, L2 / cosine (src/Core/Common/DistanceUtils.cpp:305-1046)
//                                     -> same 16-accumulator summation tree, no FMA, bit-exact
//   PQQuantizer / OPQQuantizer       (inc/Core/Common/PQQuantizer.h:110-180, OPQQuantizer.h:96-121)
//                                     -> SDC / ADC table look-ups summed in sub-vector order, device-side QuantizeVector
//
// Candidate vectors (graph neighbours / tree-centre rows) are gathered with 1-D TMA bulk copies
// (cp.async.bulk global->shared, mbarrier complete_tx) into a per-warp shared-memory ring and
// reduced from there; the two priority queues keep their first entries in shared memory and spill
// the tail of the array to a per-slot arena in HBM so the emulation stays exact at any size.
//
// search_kernel<DIM, COSINE, RPL, KDT, PQ, ELEM, MINB>:
//   DIM    768 / 128: query slice in registers, fully unrolled; 0: any dimension (query in shared memory)
//   RPL    registers per lane of the m_Results multiset (16: cap <= 512, 32: cap <= 1024)
//   KDT    KD-tree flavour of the search loop;  PQ: rows are PQ codes;  ELEM 0 float, 1 int8, 2 uint8, 3 int16
//   MINB   __launch_bounds__ minimum resident CTAs per SM (register cap)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace sptag_b200 {

// Common.h:122  MaxDist = numeric_limits<float>::max() / 10 (float arithmetic)
#define SPTAG_B200_MAXDIST (3.402823466e+38F / 10)

constexpr unsigned kFull = 0xffffffffu;
constexpr int kStatsPerQuery = 8;

// Where an iterator call starts or resumes (IterState::resume of a suspended query; 0: none)
constexpr int kIterDone = 0, kIterStep = 1, kIterInitTrees = 2, kIterStepTrees = 3, kIterFirst = 4;
// What an open iterator keeps per query between calls (the kernels take it as `int* state`, 8 ints per query)
struct IterState {
    int ng_count, spt_count;  // NGQueue / SPTQueue sizes (the entries are in the query's HBM arenas)
    int first;                // 1: the next call is the first (InitSearchTrees + SearchTrees)
    int relaxed;              // relaxedMono
    int slots;                // result slots of the caller's QueryResult, which cap the next batch; -1: none yet
    int vbits;                // log2 of the visited table's entries; 0: the visited set is a bitmap
    int vfill;                // ids in the visited set
    int resume;               // where a suspended call resumes (kIterStep, ...); 0: not suspended
};
static_assert(sizeof(IterState) == 32, "IterState is 8 ints");
// Per-query HBM area of a suspended iterator call: the m_Results multiset (32 x RPL <= 1024 floats), then resultCount,
// the checked count and the pending SearchTrees limit
constexpr int kIterResumeWords = 32 * 32 + 4;
// Suspension list header: {queries listed, step suspensions, tree suspensions, pad}, then the query indices
constexpr int kIterListHeader = 4;

// The iterator kernels' visited sets (the per-launch part; the per-query part is in the iterator state)
struct IterVisited {
    unsigned int* const* tables;  // per query: its hash table, or its bitmap (IterState::vbits = 0); nullptr: p.visited bitmaps
    float* resume;                // per query kIterResumeWords
    unsigned int* suspended;      // the queries that stopped at their table's limit (kIterListHeader + nq words)
    const unsigned int* list;     // resume launch: run only the queries listed here (same layout); nullptr = all nq
    int margin;                   // degree + largest duplicate group + 1: more than one NGQueue step can insert
};

struct SearchParams {
    // index (device resident)
    const unsigned char* vectors;          // rows padded to a 16-byte multiple
    unsigned long long row_stride_bytes;   // bytes between rows (multiple of 16)
    int row_bytes;                         // bytes copied per row (multiple of 16)
    int n, dim;
    int off_sketch;                        // sketch:: kernels: the query's int8 sketch in shared memory (fills the padding)
    const int* graph;
    int degree;
    // EnableBfs (BKTree::m_bfs, the bfs:: kernels only): != 0 seeds each tree breadth-first.  (Here it fills the padding
    // before `nodes`: a longer struct would move the iterator kernels' later arguments and change their code.)
    int bfs;
    const int* nodes;                      // BKT: 3 x int32 per node; KDT: 4 x 32 bit per node
    const int* tree_starts;
    int tree_num, node_count;
    const signed char* deleted;            // nullptr when there are no tombstones
    const unsigned char* filter;           // SearchIndexWithFilter: 0 = never added to the results; nullptr = no filter
    // queries / outputs (device)
    const unsigned char* queries;
    unsigned long long query_stride_bytes;
    int nq, k;
    int* out_ids;
    float* out_dists;
    int* out_stats;                        // nullable
    int id_offset;
    // search parameters
    int max_check, initial_pivots, other_pivots, no_better_threshold;
    int ng_length, ng_lastlevel, spt_length, spt_lastlevel;  // the reference's Heap::length/lastlevel
    int mres_cap;                          // max(MaxCheck/16, K)
    // per-slot scratch in HBM
    unsigned int* visited;
    unsigned long long visited_words;      // per slot, multiple of 4
    int2* ng_spill;
    unsigned long long ng_spill_entries;   // per slot
    int2* spt_spill;
    unsigned long long spt_spill_entries;  // per slot
    unsigned int* work_counter;
    // large N: instead of clearing the whole bitmap per query, log the words that were set and clear only those
    unsigned int* vlog;                    // per slot, vlog_entries words; nullptr = clear the bitmap per query
    unsigned long long vlog_entries;
    // hashed visited set (search_kernel only): per slot an open-addressed table (format: vhash_home); `vlog` then logs the
    // table positions a query filled.  nullptr = the bitmap above.
    unsigned int* vhash;
    unsigned vhash_mask;                   // table entries per slot - 1 (a power of two)
    int vhash_shift;                       // 32 - log2(entries)
    int vhash_limit;                       // distinct ids a query may insert before it is abandoned; INT_MAX without a table
    unsigned int* overflow;                // {count, query indices}: the queries abandoned at the limit
    const unsigned int* rerun;             // re-run launch: the same list; the kernel searches only the queries listed there
    // shared-memory layout (bytes from the dynamic smem base)
    int stage_rows, stages, slot_stride;
    int slot_stagger;  // 1: odd ring slots start 64 B later (stride is a multiple of 128); 0: stride = 64 mod 128
    int h_ng, h_spt;
    int off_ng, off_spt, off_cand, off_bar, off_query;
    int sketch_batch;  // sketch:: kernels: sketch rows per TMA batch through the row ring (fills the padding)
    // PQ / OPQ quantized index (PQQuantizer.h:110-128, ADC off): rows are M code bytes, the query is M code
    // bytes too and distance = sum_i sdc[(i*Ks + x_i)*Ks + y_i]
    // (float rows are never PQ codes, so the row sketches of the sketch:: kernels share the PQ tables' slots: a longer
    //  struct would move the iterator kernels' later arguments and change their code)
    union {
        const float* sdc;
        const unsigned char* sketch;       // sketch:: kernels: per row round_up(dim, 16) int8 then a RowSketchTail
    };
    int pq_m, pq_ks;
    // ADC mode (IQuantizer::SetEnableADC, PQQuantizer.h:114-119, :141-157): the query is a rotated float vector,
    // each warp builds its M*Ks distance table in its slot of `adc_tables` and sums table[i*Ks + y_i]
    int pq_adc, pq_dsub;
    union {
        const float* codebooks;
        unsigned long long* rows_skipped;  // sketch:: kernels: candidates whose row was not fetched, summed over queries
    };
    float* adc_tables;                     // per slot, pq_m * pq_ks floats
    // which DistanceUtils summation tree to reproduce: 16 = AVX-512 (all specialised paths), 8 = AVX / AVX2, 4 = SSE
    // (DistanceUtils.h:118-163 picks one by cpuid; a reference host without AVX-512 rounds differently)
    int simd_width;
    // K > 32: the result set is the reference's own max-heap (QueryResultSet.h:77-120) in a per-slot HBM arena
    int2* topk;                            // per slot, topk_pad entries (id, distance bits); nullptr when k <= 32
    int topk_pad;                          // k rounded up to a power of two (the final sort is bitonic)
    // 1: RefineSearchIndex flavour (searchDuplicated = false -> StaticDispatch::NeverDup, BKTIndex.cpp:447-452, :698-711):
    // a duplicate group contributes its first live member only
    int never_dup;
};

// BKTree::InitSearchTrees with m_bfs != 0 (BKTree.h:703-758): MaxBFSNodes, and the entries of one BFS heap (1-based, so
// index 0 is never written).  The two heaps sit at the end of the query's SPTQueue arena, which is that much longer.
constexpr int kBfsMaxNodes = 100;
constexpr int kBfsHeapEntries = kBfsMaxNodes + 1;

// ------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + 1-D TMA bulk copy
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// global -> shared 1-D bulk copy executed by the TMA unit; completion is signalled on `bar`
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// L2 prefetch of a contiguous block by the TMA unit (no data returns to the SM)
__device__ __forceinline__ void tma_prefetch_l2(const void* gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// distance: the reference's AVX-512 float summation tree, one half-warp per row
// ------------------------------------------------------------------------------------------
template <bool COSINE>
__device__ __forceinline__ float dist_term(float x, float y) {
    if (COSINE) return __fmul_rn(x, y);
    float d = __fsub_rn(x, y);
    return __fmul_rn(d, d);
}
template <bool COSINE>
__device__ __forceinline__ float dist_tail(float x, float y, float acc) {
    // the reference's plain-C scalar tail is FMA-contracted by g++ (SURVEY.md 8a A1)
    if (COSINE) return __fmaf_rn(x, y, acc);
    float d = __fsub_rn(x, y);
    return __fmaf_rn(d, d, acc);
}

// The reference's float AVX-512 summation tree evaluated by ONE thread (any length d): used where the
// operands are tiny (sub-vectors of a codebook) or where one thread owns one output (rotation rows).
template <bool COSINE>
__device__ float exact_dist_thread(const float* __restrict__ x, const float* __restrict__ y, int d) {
    float a16[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) a16[j] = 0.0f;
    int i = 0;
    for (; i + 16 <= d; i += 16) {
#pragma unroll
        for (int j = 0; j < 16; ++j) a16[j] = __fadd_rn(a16[j], dist_term<COSINE>(x[i + j], y[i + j]));
    }
    float a8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a8[j] = __fadd_rn(a16[j], a16[j + 8]);
    if (d & 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) a8[j] = __fadd_rn(a8[j], dist_term<COSINE>(x[i + j], y[i + j]));
        i += 8;
    }
    float a4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) a4[j] = __fadd_rn(a8[j], a8[j + 4]);
    if (d & 4) {
#pragma unroll
        for (int j = 0; j < 4; ++j) a4[j] = __fadd_rn(a4[j], dist_term<COSINE>(x[i + j], y[i + j]));
        i += 4;
    }
    float s = __fadd_rn(__fadd_rn(__fadd_rn(a4[0], a4[1]), a4[2]), a4[3]);
    for (; i < d; ++i) s = dist_tail<COSINE>(x[i], y[i], s);
    return COSINE ? __fsub_rn(1.0f, s) : s;
}

// Registers holding this lane's slice of the query: element 16c + (lane & 15) for every full
// 16-chunk c.  DIM == 0 is the generic variant (query read from shared memory every time).
template <int DIM>
struct QueryRegs {
    float q[DIM / 16 > 0 ? DIM / 16 : 1];
};

// Distance of the query to NR rows staged in shared memory, computed by a half-warp (NR independent
// accumulator chains per lane for instruction-level parallelism; each chain is exactly the reference's).
// Lane j (0..15) owns accumulator j of ComputeL2Distance_AVX512 / ComputeCosineDistance_AVX512;
// the folds 16 -> 8 -> 4 -> 1 and the 8-/4-wide/scalar tails follow DistanceUtils.cpp:650-682.
// Results are valid in lane j == 0 of the half-warp.  Must be called by all 32 lanes.
template <int DIM, bool COSINE, int NR>
__device__ __forceinline__ void half_warp_distance_n(const float* const (&row)[NR], const QueryRegs<DIM>& qr,
                                                     const float* __restrict__ qs, int dim, int j, float (&out)[NR]) {
    float acc[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) acc[r] = 0.0f;
    if (DIM > 0) {
#pragma unroll
        for (int c = 0; c < DIM / 16; ++c) {
            const float q = qr.q[c];
#pragma unroll
            for (int r = 0; r < NR; ++r) acc[r] = __fadd_rn(acc[r], dist_term<COSINE>(q, row[r][16 * c + j]));
        }
    } else {
        const int nch = dim >> 4;
        for (int c = 0; c < nch; ++c) {
            const float q = qs[16 * c + j];
#pragma unroll
            for (int r = 0; r < NR; ++r) acc[r] = __fadd_rn(acc[r], dist_term<COSINE>(q, row[r][16 * c + j]));
        }
    }
    const int d = (DIM > 0) ? DIM : dim;
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        int off = (d >> 4) << 4;
        // diff256 = lo(diff512) + hi(diff512)
        float a8 = __fadd_rn(acc[r], __shfl_down_sync(kFull, acc[r], 8, 16));
        if (d & 8) {
            if (j < 8) a8 = __fadd_rn(a8, dist_term<COSINE>(qs[off + j], row[r][off + j]));
            off += 8;
        }
        // diff128 = lo(diff256) + hi(diff256)
        float a4 = __fadd_rn(a8, __shfl_down_sync(kFull, a8, 4, 16));
        if (d & 4) {
            if (j < 4) a4 = __fadd_rn(a4, dist_term<COSINE>(qs[off + j], row[r][off + j]));
            off += 4;
        }
        // DIFF128[0] + DIFF128[1] + DIFF128[2] + DIFF128[3], left to right
        const float a1 = __shfl_sync(kFull, a4, 1, 16);
        const float a2 = __shfl_sync(kFull, a4, 2, 16);
        const float a3 = __shfl_sync(kFull, a4, 3, 16);
        float sum = __fadd_rn(__fadd_rn(__fadd_rn(a4, a1), a2), a3);
        for (int i = off; i < d; ++i) sum = dist_tail<COSINE>(qs[i], row[r][i], sum);
        out[r] = COSINE ? __fsub_rn(1.0f, sum) : sum;
    }
}

// The AVX (8 accumulators, DistanceUtils.cpp ComputeL2Distance_AVX / ComputeCosineDistance_AVX: 16 elements per trip as
// two 8-wide adds, then the 8 -> 4 fold, 4-wide tail steps, scalar tail) and SSE (4 accumulators) float trees, for a
// reference host whose cpuid dispatch lands below AVX-512.  Lanes j < width of the half-warp own the accumulators;
// result valid in lane j == 0.  Must be called by all 32 lanes.
template <bool COSINE>
__device__ __forceinline__ float half_warp_distance_w(const float* __restrict__ row, const float* __restrict__ qs, int dim,
                                                      int j, int width) {
    float acc = 0.0f;
    int i = 0;
    if (width == 8) {
        for (; i + 16 <= dim; i += 16) {
            if (j < 8) {
                acc = __fadd_rn(acc, dist_term<COSINE>(qs[i + j], row[i + j]));
                acc = __fadd_rn(acc, dist_term<COSINE>(qs[i + 8 + j], row[i + 8 + j]));
            }
        }
        acc = __fadd_rn(acc, __shfl_down_sync(kFull, acc, 4, 16));  // a4[j] = a8[j] + a8[j + 4]
    }
    for (; i + 4 <= dim; i += 4)
        if (j < 4) acc = __fadd_rn(acc, dist_term<COSINE>(qs[i + j], row[i + j]));
    const float a1 = __shfl_sync(kFull, acc, 1, 16);
    const float a2 = __shfl_sync(kFull, acc, 2, 16);
    const float a3 = __shfl_sync(kFull, acc, 3, 16);
    float sum = __fadd_rn(__fadd_rn(__fadd_rn(acc, a1), a2), a3);
    for (; i < dim; ++i) sum = dist_tail<COSINE>(qs[i], row[i], sum);
    return COSINE ? __fsub_rn(1.0f, sum) : sum;
}

template <int DIM, bool COSINE>
__device__ __forceinline__ float half_warp_distance(const float* __restrict__ row, const QueryRegs<DIM>& qr,
                                                    const float* __restrict__ qs, int dim, int j) {
    const float* const rows[1] = {row};
    float out[1];
    half_warp_distance_n<DIM, COSINE, 1>(rows, qr, qs, dim, j, out);
    return out[0];
}

// ------------------------------------------------------------------------------------------
// int8 / uint8 rows (DistanceUtils.cpp:363-400, :460-496 L2; :744-780, :838-874 cosine; helpers :195-263).
// One AVX-512 step covers 64 bytes and yields 16 float lanes; lane t = (128-bit lane L = t/4, position p = t%4) is
// the EXACT int32 sum of the four terms at byte offsets 16L + 2p + {0,1,8,9} (unpacklo/hi_epi8 + madd_epi16 +
// add_epi32), converted by cvtepi32_ps and accumulated in fp32; 32- and 16-byte steps do the same on 8 / 4 lanes.
// ------------------------------------------------------------------------------------------
template <bool UNSIGNED>
__device__ __forceinline__ int byte_val(unsigned v) {
    return UNSIGNED ? (int)(v & 255u) : (int)(signed char)(v & 255u);
}
template <bool COSINE, bool UNSIGNED>
__device__ __forceinline__ float int_lane_term(const unsigned char* __restrict__ x, const unsigned char* __restrict__ y,
                                               int off) {
    const unsigned x0 = *reinterpret_cast<const unsigned short*>(x + off);
    const unsigned x1 = *reinterpret_cast<const unsigned short*>(x + off + 8);
    const unsigned y0 = *reinterpret_cast<const unsigned short*>(y + off);
    const unsigned y1 = *reinterpret_cast<const unsigned short*>(y + off + 8);
    const int a0 = byte_val<UNSIGNED>(x0), a1 = byte_val<UNSIGNED>(x0 >> 8), a2 = byte_val<UNSIGNED>(x1),
              a3 = byte_val<UNSIGNED>(x1 >> 8);
    const int b0 = byte_val<UNSIGNED>(y0), b1 = byte_val<UNSIGNED>(y0 >> 8), b2 = byte_val<UNSIGNED>(y1),
              b3 = byte_val<UNSIGNED>(y1 >> 8);
    int s;
    if (COSINE) {
        s = a0 * b0 + a1 * b1 + a2 * b2 + a3 * b3;
    } else {
        const int d0 = a0 - b0, d1 = a1 - b1, d2 = a2 - b2, d3 = a3 - b3;
        s = d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
    }
    return (float)s;
}

// x = query bytes, row = vector bytes (both 2-byte aligned); result valid in lane j == 0 of the half-warp
template <bool COSINE, bool UNSIGNED>
__device__ __forceinline__ float half_warp_distance_int(const unsigned char* __restrict__ row,
                                                        const unsigned char* __restrict__ x, int dim, int j) {
    float acc = 0.0f;
    int i = 0;
    const int lane_off = 16 * (j >> 2) + 2 * (j & 3);
    for (; i + 64 <= dim; i += 64) acc = __fadd_rn(acc, int_lane_term<COSINE, UNSIGNED>(x, row, i + lane_off));
    float a8 = __fadd_rn(acc, __shfl_down_sync(kFull, acc, 8, 16));
    if (dim & 32) {
        if (j < 8) a8 = __fadd_rn(a8, int_lane_term<COSINE, UNSIGNED>(x, row, i + lane_off));
        i += 32;
    }
    float a4 = __fadd_rn(a8, __shfl_down_sync(kFull, a8, 4, 16));
    if (dim & 16) {
        if (j < 4) a4 = __fadd_rn(a4, int_lane_term<COSINE, UNSIGNED>(x, row, i + lane_off));
        i += 16;
    }
    const float a1 = __shfl_sync(kFull, a4, 1, 16);
    const float a2 = __shfl_sync(kFull, a4, 2, 16);
    const float a3 = __shfl_sync(kFull, a4, 3, 16);
    float s = __fadd_rn(__fadd_rn(__fadd_rn(a4, a1), a2), a3);
    for (; i + 4 <= dim; i += 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            s = __fadd_rn(s, dist_term<COSINE>((float)byte_val<UNSIGNED>(x[i + k]), (float)byte_val<UNSIGNED>(row[i + k])));
    }
    for (; i < dim; ++i) s = dist_tail<COSINE>((float)byte_val<UNSIGNED>(x[i]), (float)byte_val<UNSIGNED>(row[i]), s);
    return COSINE ? __fsub_rn(UNSIGNED ? 65025.0f : 16129.0f, s) : s;
}

// AVX2 (32-byte steps, 8 lanes) and SSE (16-byte steps, 4 lanes) variants of the same int8 / uint8 kernels
template <bool COSINE, bool UNSIGNED>
__device__ __forceinline__ float half_warp_distance_int_w(const unsigned char* __restrict__ row,
                                                          const unsigned char* __restrict__ x, int dim, int j, int width) {
    float acc = 0.0f;
    int i = 0;
    const int lane_off = 16 * (j >> 2) + 2 * (j & 3);
    if (width == 8) {
        for (; i + 32 <= dim; i += 32)
            if (j < 8) acc = __fadd_rn(acc, int_lane_term<COSINE, UNSIGNED>(x, row, i + lane_off));
        acc = __fadd_rn(acc, __shfl_down_sync(kFull, acc, 4, 16));
    }
    for (; i + 16 <= dim; i += 16)
        if (j < 4) acc = __fadd_rn(acc, int_lane_term<COSINE, UNSIGNED>(x, row, i + lane_off));
    const float a1 = __shfl_sync(kFull, acc, 1, 16);
    const float a2 = __shfl_sync(kFull, acc, 2, 16);
    const float a3 = __shfl_sync(kFull, acc, 3, 16);
    float s = __fadd_rn(__fadd_rn(__fadd_rn(acc, a1), a2), a3);
    for (; i + 4 <= dim; i += 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            s = __fadd_rn(s, dist_term<COSINE>((float)byte_val<UNSIGNED>(x[i + k]), (float)byte_val<UNSIGNED>(row[i + k])));
    }
    for (; i < dim; ++i) s = dist_tail<COSINE>((float)byte_val<UNSIGNED>(x[i]), (float)byte_val<UNSIGNED>(row[i]), s);
    return COSINE ? __fsub_rn(UNSIGNED ? 65025.0f : 16129.0f, s) : s;
}

// ------------------------------------------------------------------------------------------
// int16 rows, AVX-512 variants (DistanceUtils.cpp:559-596 L2, :930-967 cosine; helpers :263-289).  One 512-bit step
// covers 32 elements and yields 16 float lanes, t = 4L + p (128-bit lane L, position p):
//   cosine: cvtepi32_ps(madd_epi16): lane t = (float)(int32)(x[2t]*y[2t] + x[2t+1]*y[2t+1]);
//   L2: unpacklo/hi_epi16 sign-extension: dlo = x[8L+p] - y[8L+p], dhi = x[8L+4+p] - y[8L+4+p]; the compiled reference
//       (g++ -O3) evaluates the lane as fma(dhi, dhi, dlo*dlo) and accumulates with a separate add.
// 256-/128-bit steps: same on 8 / 4 lanes.  Plain-C tails: the 4-unrolled statements are FMA-contracted, the
// single-element remainder loops are not (oracle/sptag_oracle.c dist_i16, pinned to the compiled reference).
// ------------------------------------------------------------------------------------------
template <bool COSINE>
__device__ __forceinline__ float i16_lane_term(const short* __restrict__ x, const short* __restrict__ y, int base, int t) {
    if (COSINE) {
        const int x2 = *reinterpret_cast<const int*>(x + base + 2 * t);  // rows and queries are 4-byte aligned
        const int y2 = *reinterpret_cast<const int*>(y + base + 2 * t);
        const unsigned lo = (unsigned)((int)(short)(x2 & 0xffff) * (int)(short)(y2 & 0xffff));
        const unsigned hi = (unsigned)((x2 >> 16) * (y2 >> 16));
        return __int2float_rn((int)(lo + hi));
    }
    const int off = base + 8 * (t >> 2) + (t & 3);
    const float dlo = __int2float_rn((int)x[off] - (int)y[off]);
    const float dhi = __int2float_rn((int)x[off + 4] - (int)y[off + 4]);
    return __fmaf_rn(dhi, dhi, __fmul_rn(dlo, dlo));
}

// x = query, row = vector (both 4-byte aligned int16 arrays); result valid in lane j == 0 of the half-warp
template <bool COSINE>
__device__ __forceinline__ float half_warp_distance_i16(const short* __restrict__ row, const short* __restrict__ x,
                                                        int dim, int j) {
    float acc = 0.0f;
    int i = 0;
    for (; i + 32 <= dim; i += 32) acc = __fadd_rn(acc, i16_lane_term<COSINE>(x, row, i, j));
    float a8 = __fadd_rn(acc, __shfl_down_sync(kFull, acc, 8, 16));
    if (dim & 16) {
        if (j < 8) a8 = __fadd_rn(a8, i16_lane_term<COSINE>(x, row, i, j));
        i += 16;
    }
    float a4 = __fadd_rn(a8, __shfl_down_sync(kFull, a8, 4, 16));
    if (dim & 8) {
        if (j < 4) a4 = __fadd_rn(a4, i16_lane_term<COSINE>(x, row, i, j));
        i += 8;
    }
    const float a1 = __shfl_sync(kFull, a4, 1, 16);
    const float a2 = __shfl_sync(kFull, a4, 2, 16);
    const float a3 = __shfl_sync(kFull, a4, 3, 16);
    float s = __fadd_rn(__fadd_rn(__fadd_rn(a4, a1), a2), a3);
    if (dim & 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) s = dist_tail<COSINE>((float)x[i + k], (float)row[i + k], s);
        i += 4;
    }
    for (; i < dim; ++i) {
        const float fx = (float)x[i], fy = (float)row[i];
        const float c = COSINE ? __fmul_rn(fx, fy) : __fmul_rn(__fsub_rn(fx, fy), __fsub_rn(fx, fy));
        s = __fadd_rn(s, c);
    }
    // base^2 - dot with the integer literal 1073676289 = 32767^2 converted to float (DistanceUtils.cpp:966)
    return COSINE ? __fsub_rn(1073676288.0f, s) : s;
}

// integer rows by element type: ELEM 1 int8, 2 uint8, 3 int16
template <bool COSINE, int ELEM>
__device__ __forceinline__ float half_warp_distance_elem(const unsigned char* __restrict__ row,
                                                         const unsigned char* __restrict__ x, int dim, int j) {
    if (ELEM == 3)
        return half_warp_distance_i16<COSINE>(reinterpret_cast<const short*>(row), reinterpret_cast<const short*>(x), dim, j);
    return half_warp_distance_int<COSINE, ELEM == 2>(row, x, dim, j);
}
// the same with the summation tree chosen at run time (16 / 8 / 4); int16 rows exist in the AVX-512 form only
template <bool COSINE, int ELEM>
__device__ __forceinline__ float half_warp_distance_elem_w(const unsigned char* __restrict__ row,
                                                           const unsigned char* __restrict__ x, int dim, int j, int width) {
    if (ELEM == 3 || width == 16) return half_warp_distance_elem<COSINE, ELEM>(row, x, dim, j);
    return half_warp_distance_int_w<COSINE, ELEM == 2>(row, x, dim, j, width);
}
// the query element the KD split test reads (KDTree.h:255)
template <int ELEM>
__device__ __forceinline__ float int_query_elem(const void* q, int i) {
    if (ELEM == 3) return (float)reinterpret_cast<const short*>(q)[i];
    return (float)byte_val<ELEM == 2>(reinterpret_cast<const unsigned char*>(q)[i]);
}

// ------------------------------------------------------------------------------------------
// Heap<NodeDistPair>: exact emulation of Heap.h:13-106.  entry = (node, distance bits) as int2.
// Index 0 holds the default pair (-1, MaxDist); indices 1..H live in shared memory, the rest of
// the array in the per-slot HBM arena.
// ------------------------------------------------------------------------------------------
struct WarpHeap {
    int2* s;  // shared memory, indices [0, H]
    int2* g;  // global memory, indexed by the same index (entries <= H unused)
    int H;
    int count;
    int length, lastlevel;
    // register copy of the LAST element (index tail_idx; valid while tail_idx == count): Heap::pop starts by moving the
    // last element to the root, and deep in the HBM arena that read is a full memory round trip at the head of every
    // pop's dependency chain.  Inserts know what they leave at the last position; a pop fetches the new last element
    // ahead of time.
    int2 tail;
    int tail_idx;
};

// (a branch-free variant -- select a generic pointer, one LD/ST -- was slower on BKT 1M x 128)
__device__ __forceinline__ int2 heap_ld(const WarpHeap& h, int i) { return i <= h.H ? h.s[i] : h.g[i]; }
__device__ __forceinline__ void heap_st(const WarpHeap& h, int i, int2 v) {
    if (i <= h.H)
        h.s[i] = v;
    else
        h.g[i] = v;
}
__device__ __forceinline__ float pair_dist(int2 v) { return __int_as_float(v.y); }
__device__ __forceinline__ int2 make_pair(int node, float d) { return make_int2(node, __float_as_int(d)); }

// Heap::Top(): slot 0 (-1, MaxDist) when empty (Heap.h:36)
__device__ __forceinline__ float heap_top_dist(const WarpHeap& h) {
    return h.count == 0 ? SPTAG_B200_MAXDIST : pair_dist(h.s[1]);
}

// Heap::insert on a FULL heap (Heap.h:43-49): the slot of the first maximum of the last level [lastlevel, length], or
// -1 when the new value is larger than that maximum and is dropped.
static __device__ __noinline__ int heap_full_slot(const int2* hs, const int2* hg, int H, int lastlevel, int length, float d, int lane) {
    float best = -1.0f;
    int besti = 0x7fffffff;
    bool have = false;
    for (int i = lastlevel + lane; i <= length; i += 32) {
        const int2 e = (i <= H) ? hs[i] : hg[i];
        const float v = __int_as_float(e.y);
        if (!have || v > best) {  // strict '<' in the reference keeps the earliest maximum
            best = v;
            besti = i;
            have = true;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(kFull, best, o);
        const int oi = __shfl_xor_sync(kFull, besti, o);
        const bool oh = __shfl_xor_sync(kFull, (int)have, o) != 0;
        if (oh && (!have || ob > best || (ob == best && oi < besti))) {
            best = ob;
            besti = oi;
            have = true;
        }
    }
    return (d > best) ? -1 : besti;
}

// The hashed visited set's table format (the search kernels and iter_grow_kernel's rehash): an id is stored as the key
// id + 1 (0 = an empty position) and probed linearly from its home position, the top log2(entries) bits of a multiplicative
// hash (shift = 32 - log2(entries)); inserts stop at half the capacity.
__host__ __device__ __forceinline__ unsigned vhash_home(unsigned id, int shift) { return (id * 2654435769u) >> shift; }

// Hashed visited set (open addressing, keys id + 1, 0 = empty, linear probing).  The per-lane probe past the home position
// is rare and kept out of line like heap_full_slot, so that it adds nothing to the kernels' register allocation; the
// warp-uniform insert has an out-of-line copy too (which one costs fewer registers depends on the kernel).
constexpr unsigned kVhashFound = 0x80000000u;  // table positions stay below 2^30
// One lane's probe for `key` after position `pos`, which holds another id (other lanes of the warp insert other keys
// concurrently): the position where the key was inserted, or its position | kVhashFound when it was there already.
static __device__ __noinline__ unsigned vhash_probe(unsigned* table, unsigned pos, unsigned key, unsigned mask) {
    for (;;) {
        pos = (pos + 1u) & mask;
        const unsigned old = atomicCAS(&table[pos], 0u, key);
        if (old == 0u) return pos;
        if (old == key) return pos | kVhashFound;
    }
}
// CheckAndSet for a warp-uniform key: every lane walks the same probe sequence from `pos`; lane 0 inserts the key and,
// with LOG, logs its position at *log_at.  True if the key was present.
template <bool LOG = true>
static __device__ __forceinline__ bool vhash_insert_uniform(unsigned* table, unsigned* log_at, unsigned pos, unsigned key,
                                                            unsigned mask, int lane) {
    unsigned cur;
    while ((cur = __ldcg(&table[pos])) != 0u && cur != key) pos = (pos + 1u) & mask;
    const bool was = cur == key;
    if (!was && lane == 0) {
        table[pos] = key;
        if (LOG) *log_at = pos;
    }
    __syncwarp();
    return was;
}
static __device__ __noinline__ bool vhash_insert_uniform_call(unsigned* table, unsigned* log_at, unsigned pos, unsigned key,
                                                              unsigned mask, int lane) {
    return vhash_insert_uniform(table, log_at, pos, key, mask, lane);
}

// Heap::insert (Heap.h:39-62).  The sift-up path (the ancestors loc>>1, loc>>2, ...) is loaded by
// one lane per level, the stop level is found with a ballot, and the shifted parents plus the new
// value are stored in one step -- the resulting array is identical to the sequential loop's.
template <bool TAIL = true>
__device__ __forceinline__ void heap_insert(WarpHeap& h, int node, float d, int lane) {
    // TAIL (fast BKT path): keep the register copy of the last element up to date
#define SPTAG_B200_HLD(i) heap_ld(h, (i))
#define SPTAG_B200_HST(i, v) heap_st(h, (i), (v))
    int loc;
    if (h.count == h.length) {
        // full heap (Heap.h:43-49): rare, and ~80 instructions per inlined copy of insert -- kept out of line because the
        // kernels are several times larger than the instruction cache
        loc = heap_full_slot(h.s, h.g, h.H, h.lastlevel, h.length, d, lane);
        if (loc < 0) return;
        if (TAIL) h.tail_idx = -1;
    } else {
        loc = ++h.count;
    }
    const int anc = loc >> (lane + 1);
    int2 av = make_int2(0, 0);
    if (anc > 0) av = SPTAG_B200_HLD(anc);
    const bool stop = (anc <= 0) || !(d < pair_dist(av));
    const int s = __ffs(__ballot_sync(kFull, stop)) - 1;  // levels 0..s-1 move down
    if (lane < s)
        SPTAG_B200_HST(loc >> lane, av);
    else if (lane == s)
        SPTAG_B200_HST(loc >> s, make_pair(node, d));
    if (TAIL && loc == h.count) {  // what now sits at the last position: the new element, or its parent moved down
        if (s == 0) {
            h.tail = make_pair(node, d);
        } else {
            h.tail.x = __shfl_sync(kFull, av.x, 0);
            h.tail.y = __shfl_sync(kFull, av.y, 0);
        }
        h.tail_idx = loc;
    }
    __syncwarp();
}
#undef SPTAG_B200_HLD
#undef SPTAG_B200_HST

// Round-1 forms, kept for every kernel except the 512-byte-row fast path: one dependent load per level and a branch per
// access.  They hold fewer values live than the paired / gathered pop below, which matters where the register cap is
// what sets the residency (768-d rows: 15 slots at 127 registers; PQ: 24 slots at 80) -- the newer forms cost those
// kernels spills and occupancy while the latency they remove is hidden there anyway.
// Heap::pop (Heap.h:73-82) + heapify (Heap.h:92-105), level by level.
__device__ __forceinline__ int2 heap_pop_seq(WarpHeap& h, int lane) {
    if (h.count == 0) return make_pair(-1, SPTAG_B200_MAXDIST);
    const int2 top = heap_ld(h, 1);
    const int2 cur = heap_ld(h, h.count);
    h.count--;
    const float cd = pair_dist(cur);
    int parent = 1, next = 2;
    while (next < h.count) {
        int2 a = heap_ld(h, next);
        const int2 b = heap_ld(h, next + 1);
        if (pair_dist(a) > pair_dist(b)) {
            next++;
            a = b;
        }
        if (pair_dist(a) < cd) {
            if (lane == 0) heap_st(h, parent, a);
            parent = next;
            next <<= 1;
        } else
            break;
    }
    if (next == h.count) {
        const int2 a = heap_ld(h, next);
        if (pair_dist(a) < cd) {
            if (lane == 0) heap_st(h, parent, a);
            parent = next;
        }
    }
    if (lane == 0 && h.count > 0) heap_st(h, parent, cur);
    __syncwarp();
    return top;
}


// Heap::pop (Heap.h:73-82) + heapify (Heap.h:92-105).  Executed redundantly by every lane (uniform loads broadcast);
// lane 0 stores.  Returns the old root.
// The two children of a node sit next to each other (indices 2p, 2p + 1 = 16 aligned bytes), so one 128-bit load
// fetches both; the host keeps H odd, which puts a pair either wholly in shared memory (2p < H) or wholly in the HBM
// arena.  The walk runs the shared-memory levels first and the arena levels second, each as a tight loop without the
// per-access "which memory" branch.
template <bool TAIL = true>
__device__ __forceinline__ int2 heap_pop(WarpHeap& h, int lane) {
    if (h.count == 0) return make_pair(-1, SPTAG_B200_MAXDIST);
    const int2 top = h.s[1];
    const int2 cur = (TAIL && h.tail_idx == h.count) ? h.tail : heap_ld(h, h.count);
    const int n = --h.count;
    const float cd = pair_dist(cur);
    int parent = 1, next = 2;
    bool placed = false;
    {   // levels whose child pair lives in shared memory
        const int lim = min(n, h.H);
        while (next < lim) {
            const int4 pr = *reinterpret_cast<const int4*>(h.s + next);
            const bool right = __int_as_float(pr.y) > __int_as_float(pr.w);  // strict: the left child wins ties (Heap.h:96)
            const int cn = right ? pr.z : pr.x, cb = right ? pr.w : pr.y;
            next += right ? 1 : 0;
            if (__int_as_float(cb) < cd) {
                if (lane == 0) h.s[parent] = make_int2(cn, cb);  // parent < next < lim <= H: always the shared-memory head
                parent = next;
                next <<= 1;
            } else {
                placed = true;
                break;
            }
        }
    }
    if (!placed) {
        if (next > h.H) {
            // Levels in the HBM arena.  Walking them one dependent load at a time costs a memory round trip per level (the
            // profile's second-largest stall); instead the whole 5-level subtree below the current node is fetched in
            // ONE gather -- lane l loads the child pair number l of the 31 pairs in breadth-first order, pair (t, o) =
            // indices (next << t) + 2 o, +1 -- every lane picks its pair's smaller child by the reference's rule, and the
            // walk is then replayed from registers with shuffles.  One round trip per 5 levels.
            while (!placed && next <= n) {
                const int t = 31 - __clz(lane + 1);
                const int o = lane + 1 - (1 << t);
                const int idx = (next << t) + 2 * o;
                const bool two = (lane < 31) && (idx < n);   // both children exist
                const bool one = (lane < 31) && (idx == n);  // a last level with a single child (Heap.h:104)
                int4 pr = make_int4(0, 0, 0, 0);
                if (two) {
                    pr = *reinterpret_cast<const int4*>(h.g + idx);
                } else if (one) {
                    const int2 a = h.g[idx];
                    pr.x = a.x;
                    pr.y = a.y;
                }
                const bool right = two && (__int_as_float(pr.y) > __int_as_float(pr.w));
                const int cn = right ? pr.z : pr.x, cb = right ? pr.w : pr.y;
                const unsigned m_two = __ballot_sync(kFull, two), m_one = __ballot_sync(kFull, one);
                const unsigned m_right = __ballot_sync(kFull, right);
                int oo = 0;
#pragma unroll
                for (int tt = 0; tt < 5; ++tt) {
                    if (placed) break;
                    const int L = (1 << tt) - 1 + oo;
                    const int pidx = (next << tt) + 2 * oo;
                    const int scn = __shfl_sync(kFull, cn, L), scb = __shfl_sync(kFull, cb, L);
                    if ((m_two >> L) & 1u) {
                        const int r = (int)((m_right >> L) & 1u);
                        if (__int_as_float(scb) < cd) {
                            if (lane == 0) heap_st(h, parent, make_int2(scn, scb));
                            parent = pidx + r;
                            oo = 2 * oo + r;
                        } else {
                            placed = true;
                        }
                    } else {
                        if (((m_one >> L) & 1u) && __int_as_float(scb) < cd) {
                            if (lane == 0) heap_st(h, parent, make_int2(scn, scb));
                            parent = pidx;
                        }
                        placed = true;  // no (further) children
                    }
                }
                next = parent << 1;  // (only used when all five levels moved up)
            }
        } else if (next == n) {  // a last level with a single child, in shared memory
            const int2 a = heap_ld(h, next);
            if (pair_dist(a) < cd) {
                if (lane == 0) heap_st(h, parent, a);
                parent = next;
            }
        }
    }
    if (lane == 0 && n > 0) heap_st(h, parent, cur);
    __syncwarp();
    if (TAIL) {
        h.tail_idx = -1;
        if (n > h.H) {  // the next pop's first read, issued now; an insert in between simply overwrites the copy
            h.tail = h.g[n];
            h.tail_idx = n;
        }
    }
    return top;
}

// ------------------------------------------------------------------------------------------
// DistPriorityQueue m_Results (WorkSpace.h:167-225): a multiset of the `cap` smallest distances
// seen so far, pre-filled with MaxDist (the reference's sentinel root plus its still-empty slots);
// insert(d) rejects iff d > worst(), otherwise replaces one maximum.  Held in registers:
// slot s = r*32 + lane.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned float_key(float f) {
    unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <int RPL>
struct MResults {
    static constexpr int G = RPL / 4;  // four groups per lane so the owner rescans one group, not the whole lane
    float m[RPL];
    float g[4];   // maximum of each group of this lane
    float lmax;   // this lane's maximum
    float worst;  // warp-wide maximum (uniform)

    __device__ __forceinline__ void reset(int cap, int lane) {
#pragma unroll
        for (int r = 0; r < RPL; ++r) m[r] = (r * 32 + lane < cap) ? SPTAG_B200_MAXDIST : -INFINITY;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v = -INFINITY;
#pragma unroll
            for (int r = 0; r < G; ++r) v = fmaxf(v, m[k * G + r]);
            g[k] = v;
        }
        lmax = fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]));
        worst = SPTAG_B200_MAXDIST;
    }
    template <int K>
    __device__ __forceinline__ void replace_in_group(float d) {
        bool done = false;
        float nm = -INFINITY;
#pragma unroll
        for (int r = 0; r < G; ++r) {
            if (!done && m[K * G + r] == lmax) {
                m[K * G + r] = d;
                done = true;
            }
            nm = fmaxf(nm, m[K * G + r]);
        }
        g[K] = nm;
    }
    __device__ __forceinline__ bool insert(float d, int lane) {
        if (d > worst) return false;
        const int owner = __ffs(__ballot_sync(kFull, lmax == worst)) - 1;
        if (lane == owner) {
            // replace ONE maximum: the first group whose maximum is the lane maximum (any one is equivalent)
            if (g[0] == lmax)
                replace_in_group<0>(d);
            else if (g[1] == lmax)
                replace_in_group<1>(d);
            else if (g[2] == lmax)
                replace_in_group<2>(d);
            else
                replace_in_group<3>(d);
            lmax = fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]));
        }
        worst = key_float(__reduce_max_sync(kFull, float_key(lmax)));
        return true;
    }
    // a suspended iterator call keeps its multiset in HBM (32 * RPL floats) until it resumes
    __device__ __forceinline__ void save(float* dst, int lane) const {
#pragma unroll
        for (int r = 0; r < RPL; ++r) dst[r * 32 + lane] = m[r];
    }
    __device__ __forceinline__ void load(const float* src, int lane) {
#pragma unroll
        for (int r = 0; r < RPL; ++r) m[r] = src[r * 32 + lane];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v = -INFINITY;
#pragma unroll
            for (int r = 0; r < G; ++r) v = fmaxf(v, m[k * G + r]);
            g[k] = v;
        }
        lmax = fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]));
        worst = key_float(__reduce_max_sync(kFull, float_key(lmax)));
    }
};

// ------------------------------------------------------------------------------------------
// Row sketches (the sketch:: kernels): a 1-byte-per-dimension copy of every float row that decides, exactly, which
// graph candidates m_Results must reject, so that their 4-byte-per-dimension rows are never fetched.
// A vector v is sketched as  scale = max|v_i| / 127,  s_i = clamp(rint(v_i / scale), -127, 127)  (all zero when scale
// is 0) plus three bounds: err >= ||v - scale s||, norm >= ||v||, nsq <= ||v||^2.  A vector with a NaN or an infinity is
// sketched as zeros with err = +inf, which no test passes.  For a query q (t, e_q) and a row x (s, e_x), I = sum t_i s_i
// is an exact integer and, by Cauchy-Schwarz,
//     q.x <= scale_q scale_x I + norm_q err_x + err_q norm_x + err_q err_x.
// sketch_lower_bound turns that into a value the reference's fp32 distance cannot fall below: every step rounds to the
// safe side, and `rel` (sketch_rel_margin) times the operands' size covers the reference's own rounding in any of its
// three summation trees.  tools/row_sketch_model.py restates all of this in numpy, operation by operation, and
// tests/test_row_sketch_bound.py holds that restatement against the reference's distance function.
// ------------------------------------------------------------------------------------------
struct RowSketchTail {
    float scale, err, norm, nsq;
};
static_assert(sizeof(RowSketchTail) == 16, "a sketch row ends in 16 bytes");
__host__ __device__ __forceinline__ int sketch_elems(int dim) { return (dim + 15) & ~15; }
__host__ __device__ __forceinline__ size_t sketch_stride(int dim) { return (size_t)sketch_elems(dim) + sizeof(RowSketchTail); }
// dim/4 additions per accumulator in the narrowest (SSE) tree, the folds, the tail, the product and the last subtraction,
// 2^-24 each, doubled
__host__ __device__ __forceinline__ float sketch_rel_margin(int dim) { return (float)(dim / 4 + 24) * 1.1920928955078125e-07f; }
constexpr float kSketchNormLimit = 1e15f;  // beyond it the reference's own sum may overflow into a NaN: no statement

// the next float above / below a non-negative finite one
__device__ __forceinline__ float f32_above(float f) { return f < INFINITY ? __uint_as_float(__float_as_uint(f) + 1u) : f; }
__device__ __forceinline__ float f32_below(float f) { return f > 0.0f ? __uint_as_float(__float_as_uint(f) - 1u) : 0.0f; }
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// The sketch of v[0..dim) by one warp: the int8 elements (zero padded to sketch_elems) to `out`, the tail returned in
// every lane.  `out` may be shared or global memory.
__device__ __forceinline__ RowSketchTail warp_sketch(const float* __restrict__ v, int dim, signed char* out, int lane) {
    float amax = 0.0f;
    double n2 = 0.0;
    bool finite = true;
    for (int i = lane; i < dim; i += 32) {
        const float x = v[i];
        finite = finite && (fabsf(x) < INFINITY);
        amax = fmaxf(amax, fabsf(x));
        n2 += (double)x * (double)x;
    }
    finite = __all_sync(kFull, finite);
    amax = finite ? __uint_as_float(__reduce_max_sync(kFull, __float_as_uint(amax))) : 0.0f;
    n2 = finite ? warp_sum(n2) : 0.0;
    const float scale = __fdiv_rn(amax, 127.0f);
    double r2 = 0.0;
    const int de = sketch_elems(dim);
    for (int i = lane; i < de; i += 32) {
        int s = 0;
        if (i < dim && finite) {
            const float x = v[i];
            if (scale > 0.0f) s = (int)fminf(fmaxf(rintf(__fdiv_rn(x, scale)), -127.0f), 127.0f);
            const double res = (double)x - (double)scale * (double)s;
            r2 += res * res;
        }
        out[i] = (signed char)s;
    }
    r2 = warp_sum(r2);
    RowSketchTail t;
    t.scale = scale;
    t.err = finite ? f32_above((float)sqrt(r2)) : INFINITY;
    t.norm = f32_above((float)sqrt(n2));
    t.nsq = f32_below(f32_below((float)n2));
    return t;
}

// A value the reference's distance of the query (tail q) to a row (tail x) with integer product I never falls below;
// -inf where nothing can be said
template <bool COSINE>
__device__ __forceinline__ float sketch_lower_bound(int I, const RowSketchTail& q, const RowSketchTail& x, float rel) {
    const float fi = __int2float_ru(I);
    const float ss = (I >= 0) ? __fmul_ru(q.scale, x.scale) : __fmul_rd(q.scale, x.scale);
    float ub = __fmul_ru(ss, fi);
    ub = __fadd_ru(ub, __fmul_ru(q.norm, x.err));
    ub = __fadd_ru(ub, __fmul_ru(q.err, x.norm));
    ub = __fadd_ru(ub, __fmul_ru(q.err, x.err));
    float lb;
    if (COSINE) {
        const float margin = __fmul_ru(rel, __fadd_ru(1.0f, __fmul_ru(q.norm, x.norm)));
        lb = __fsub_rd(__fsub_rd(1.0f, ub), margin);
    } else {
        const float nsum = __fadd_ru(q.norm, x.norm);
        const float margin = __fadd_ru(__fmul_ru(rel, __fmul_ru(nsum, nsum)), 1e-30f);
        lb = __fsub_rd(__fsub_rd(__fadd_rd(q.nsq, x.nsq), __fmul_ru(2.0f, ub)), margin);
    }
    const bool safe = __fmul_ru(q.norm, x.norm) < kSketchNormLimit && q.norm < kSketchNormLimit && x.norm < kSketchNormLimit &&
                      x.err < INFINITY && q.err < INFINITY;
    return (safe && lb == lb) ? lb : -INFINITY;
}

// ------------------------------------------------------------------------------------------
// The per-query state of one warp
// ------------------------------------------------------------------------------------------
struct BktNodeDev {
    int centerid, childStart, childEnd;
};

// HASH: the hashed visited set can be bound (search_kernel).  QHASH: the visited set is chosen per query (the iterator
// kernels): a hash table whose capacity the query carries in qmask / qshift / qlimit, or a bitmap (qmask = 0).
// BFS: the kernel seeds BKT trees breadth-first when p.bfs != 0 (the bfs:: kernels)
// SKETCH: BKT search tests a graph candidate's row sketch before it fetches the row (the sketch:: kernels)
template <int DIM, bool COSINE, int RPL, bool PQ, int ELEM, bool HASH = false, bool QHASH = false, bool BFS = false,
          bool SKETCH = false>
struct WarpSearch {
    const SearchParams& p;
    const int lane, half, j;
    // shared memory
    unsigned char* ring;
    int* cand_id;
    float* cand_dist;
    uint64_t* bars;
    float* qs;
    // HBM scratch of this slot
    unsigned int* visited;  // the bitmap, or the hash table when p.vhash is set
    unsigned int* vlog;  // nullptr when the bitmap is cleared wholesale
    int vlog_count;      // ids inserted (QHASH: the fill of the query's set, kept across calls)
    // QHASH: this query's table entries - 1 (0: its bitmap), 32 - log2(entries), and the fill at which it stops inserting
    unsigned qmask;
    int qshift, qlimit;
    bool trees_cut;      // QHASH: search_trees stopped before a pop because the table was at its limit
    // queues
    WarpHeap ng, spt;
    MResults<RPL> mres;
    // top-K: lane i holds the i-th best (dist, id) (k <= 32); larger k: unordered set in the slot's HBM arena
    int2* tk;
    float tk_d;
    int tk_id;
    float worst_d;
    int worst_id;
    int tk_count, worst_pos;  // K > 32: entries kept so far / where the worst one sits (valid once K are kept)
    // query slice
    QueryRegs<DIM> qr;
    // counters
    int checked, ndist, nexpand, ntree;
    int tree_checked, no_better;  // KDT: m_iNumberOfTreeCheckedLeaves, m_iNumOfContinuousNoBetterPropagation
    unsigned phase_bits;
    // SKETCH: the query's sketch (its elements in shared memory, 16-byte aligned) and the candidates whose rows were not
    // fetched
    const unsigned* tq;
    RowSketchTail tq_tail;
    int nskipped;

    __device__ __forceinline__ WarpSearch(const SearchParams& p_, int lane_)
        : p(p_), lane(lane_), half(lane_ >> 4), j(lane_ & 15) {}

    // The kernels' set-up: the shared-memory carve-up, the queue heads' descriptors (the caller binds their HBM arenas),
    // the ring's barriers and the queues' sentinels
    __device__ __forceinline__ void setup_warp(unsigned char* smem) {
        ring = smem;
        cand_id = reinterpret_cast<int*>(smem + p.off_cand);
        cand_dist = reinterpret_cast<float*>(smem + p.off_cand + 128);
        bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
        qs = reinterpret_cast<float*>(smem + p.off_query);
        ng.s = reinterpret_cast<int2*>(smem + p.off_ng);
        ng.H = p.h_ng;
        ng.length = p.ng_length;
        ng.lastlevel = p.ng_lastlevel;
        spt.s = reinterpret_cast<int2*>(smem + p.off_spt);
        spt.H = p.h_spt;
        spt.length = p.spt_length;
        spt.lastlevel = p.spt_lastlevel;
        phase_bits = 0;
        if (lane == 0) {
            for (int s = 0; s < p.stages; ++s) mbar_init(&bars[s], 1);
            mbar_fence_init();
            ng.s[0] = make_pair(-1, SPTAG_B200_MAXDIST);
            spt.s[0] = make_pair(-1, SPTAG_B200_MAXDIST);
        }
        __syncwarp();
    }
    // WorkSpace::Reset + ResetResult (WorkSpace.h:265-286) but the visited set's contents: no ids inserted, empty queues,
    // an m_Results of `mres_cap`, an empty top-K, zero counters
    __device__ __forceinline__ void reset_workspace(int mres_cap) {
        vlog_count = 0;
        ng.count = 0;
        spt.count = 0;
        ng.tail_idx = spt.tail_idx = -1;
        mres.reset(mres_cap, lane);
        tk_d = SPTAG_B200_MAXDIST;
        tk_id = -1;
        worst_d = SPTAG_B200_MAXDIST;
        worst_id = -1;
        if (tk != nullptr) res_reset();
        checked = ndist = nexpand = ntree = 0;
        tree_checked = no_better = 0;
    }
    // the iterator kernels: the query (element type of the index) -> shared memory
    __device__ __forceinline__ void load_query_bytes(int q) {
        const unsigned char* qb = p.queries + (size_t)q * p.query_stride_bytes;
        unsigned char* qd = reinterpret_cast<unsigned char*>(qs);
        const int qbytes = p.dim * (ELEM == 0 ? 4 : (ELEM == 3 ? 2 : 1));
        for (int i = lane; i < qbytes; i += 32) qd[i] = qb[i];
    }
    // the queue heads of a query whose queues persist in HBM: back into shared memory, and out again
    __device__ __forceinline__ void restore_queue_heads() {
        for (int i = 1 + lane; i <= min(ng.count, ng.H); i += 32) ng.s[i] = ng.g[i];
        for (int i = 1 + lane; i <= min(spt.count, spt.H); i += 32) spt.s[i] = spt.g[i];
    }
    __device__ __forceinline__ void flush_queue_heads() {
        for (int i = 1 + lane; i <= min(ng.count, ng.H); i += 32) ng.g[i] = ng.s[i];
        for (int i = 1 + lane; i <= min(spt.count, spt.H); i += 32) spt.g[i] = spt.s[i];
    }
    // result i of query q into the caller's arrays (ids shifted by the index's id offset; -1 stays -1)
    __device__ __forceinline__ void write_result(size_t q, int i, int id, float d) const {
        p.out_ids[q * p.k + i] = (id >= 0) ? id + p.id_offset : id;
        p.out_dists[q * p.k + i] = d;
    }

    // Everything but the 512-byte-row fast path keeps the round-1 step order and queue code (see heap_pop_seq): those
    // kernels' residency is set by a register cap (768-d: 15 slots at 127 registers, PQ: 24 at 80) or by the uncapped
    // register count (integer rows), and the extra live values of the newer code cost them 7-17 % on a B200.
    static constexpr bool kLean = !((DIM == 128) && (ELEM == 0) && !PQ);
    __device__ __forceinline__ void hins(WarpHeap& h, int node, float d) { heap_insert<!kLean>(h, node, d, lane); }
    __device__ __forceinline__ int2 hpop(WarpHeap& h) {
        if (kLean) return heap_pop_seq(h, lane);
        return heap_pop<true>(h, lane);
    }
    // KDT flavour: every new neighbour is inserted (8 inserts per pop), so keeping the tail copy current costs more than
    // the read it saves
    __device__ __forceinline__ void hins_k(WarpHeap& h, int node, float d) { heap_insert<false>(h, node, d, lane); }
    __device__ __forceinline__ int2 hpop_k(WarpHeap& h) {
        if (kLean) return heap_pop_seq(h, lane);
        return heap_pop<false>(h, lane);
    }

    __device__ __forceinline__ unsigned char* slot_ptr(int s) const {
        return ring + (size_t)s * p.slot_stride + (p.slot_stagger ? ((s & 1) << 6) : 0);
    }

    // the hashed visited set is bound to this launch (QHASH: to this query)
    __device__ __forceinline__ bool hashed() const { return (HASH && p.vhash != nullptr) || (QHASH && qmask != 0u); }
    __device__ __forceinline__ unsigned vhash_mask() const { return QHASH ? qmask : p.vhash_mask; }
    // hashed visited set: home position of an id in this slot's table
    __device__ __forceinline__ unsigned vhash_home(int id) const {
        return sptag_b200::vhash_home(id, QHASH ? qshift : p.vhash_shift);
    }
    // the query has filled its table to the load limit: it is abandoned (nothing counts as new any more, the search loops
    // stop) and search_kernel re-runs it on the bitmap.  Never true on the bitmap.  QHASH: the iterator kernels suspend
    // or restart the query on a larger table (iterate_kernel never reaches the limit inside a step).
    __device__ __forceinline__ bool vset_full() const {
        return (HASH && vlog_count >= p.vhash_limit) || (QHASH && vlog_count >= qlimit);
    }

    // OptHashPosVector::CheckAndSet for a warp-uniform id: true if already present.  OUTLINE: the hashed insert is a call
    // (BKT tree seeding; the KD-tree leaves inline it)
    template <bool OUTLINE = true>
    __device__ __forceinline__ bool check_and_set_uniform(int id) {
        if (hashed()) {
            if (vset_full()) return true;
            // (the iterators' tables keep no clear log)
            const bool was = QHASH     ? vhash_insert_uniform<false>(visited, nullptr, vhash_home(id), (unsigned)id + 1u, qmask, lane)
                             : OUTLINE ? vhash_insert_uniform_call(visited, vlog + vlog_count, vhash_home(id), (unsigned)id + 1u,
                                                                   p.vhash_mask, lane)
                                       : vhash_insert_uniform(visited, vlog + vlog_count, vhash_home(id), (unsigned)id + 1u,
                                                              p.vhash_mask, lane);
            if (!was) vlog_count++;
            return was;
        }
        const unsigned w = __ldcg(&visited[id >> 5]);
        const unsigned bit = 1u << (id & 31);
        const bool was = (w & bit) != 0;
        if (!was) {
            if (lane == 0) {
                visited[id >> 5] = w | bit;
                if (vlog != nullptr && vlog_count < (int)p.vlog_entries) vlog[vlog_count] = (unsigned)(id >> 5);
            }
            vlog_count++;
        }
        __syncwarp();
        return was;
    }

    // ---- K > 32: QueryResultSet in the slot's HBM arena ----
    static __device__ __forceinline__ bool res_less(int2 a, int2 b) {  // QueryResultSet.h:17-20
        const float da = __int_as_float(a.y), db = __int_as_float(b.y);
        return (da < db) || ((da == db) && (a.x < b.x));
    }
    // K > 32: the reference keeps the K best in a max-heap on (Dist, VID) (QueryResultSet.h:77-120).  What a caller can
    // observe of it is (a) the root = the worst kept entry, which gates AddPoint, and (b) the ascending list after
    // SortResult; both are functions of the SET of kept entries, not of the heap layout.  So the arena holds the set
    // unordered: an accepted point is appended while fewer than K are kept (the root is then still a (-1, MaxDist)
    // filler) and otherwise overwrites the worst entry, whose successor is found by one coalesced warp scan; the final
    // order comes from a warp-wide bitonic sort.  (A heap emulation costs ~log2 K dependent HBM round trips per AddPoint
    // and K log2 K for the sort -- 7 ms per query at K = 1001.)
    __device__ __forceinline__ void res_rescan_worst() {
        int2 best = make_pair(-1, -INFINITY);
        int bpos = 0;
        for (int i = lane; i < p.k; i += 32) {
            const int2 e = tk[i];
            if (res_less(best, e)) {
                best = e;
                bpos = i;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            int2 oth;
            oth.x = __shfl_xor_sync(kFull, best.x, o);
            oth.y = __shfl_xor_sync(kFull, best.y, o);
            const int op = __shfl_xor_sync(kFull, bpos, o);
            if (res_less(best, oth)) {
                best = oth;
                bpos = op;
            }
        }
        worst_d = __int_as_float(best.y);
        worst_id = best.x;
        worst_pos = bpos;
    }
    __device__ __forceinline__ void res_reset() { tk_count = 0; }
    // QueryResultSet::SortResult (QueryResultSet.h:89-96): ascending by (Dist, VID); unfilled slots are (-1, MaxDist)
    __device__ __forceinline__ void res_sort() {
        const int n = p.topk_pad;  // power of two >= K
        for (int i = tk_count + lane; i < n; i += 32)
            tk[i] = (i < p.k) ? make_pair(-1, SPTAG_B200_MAXDIST) : make_pair(0x7fffffff, INFINITY);
        __syncwarp();
        for (int size = 2; size <= n; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = lane; t < (n >> 1); t += 32) {
                    const int i = ((t & ~(stride - 1)) << 1) | (t & (stride - 1));  // bit `stride` clear
                    const int j = i | stride;
                    const bool ascending = (i & size) == 0;
                    const int2 a = tk[i], b = tk[j];
                    if (res_less(b, a) == ascending) {
                        tk[i] = b;
                        tk[j] = a;
                    }
                }
                __syncwarp();
            }
        }
    }

    // QueryResultSet::AddPoint (QueryResultSet.h:77-87) on the sorted register list
    __device__ __forceinline__ bool add_point(int id, float d) {
        if (!(d < worst_d || (d == worst_d && id < worst_id))) return false;
        if (tk != nullptr) {
            if (tk_count < p.k) {
                if (lane == 0) tk[tk_count] = make_pair(id, d);
                ++tk_count;
                if (tk_count == p.k) {
                    __syncwarp();
                    res_rescan_worst();
                }
            } else {
                if (lane == 0) tk[worst_pos] = make_pair(id, d);
                __syncwarp();
                res_rescan_worst();
            }
            return true;
        }
        const bool less = (lane < p.k) && ((tk_d < d) || (tk_d == d && tk_id < id));
        const int pos = __popc(__ballot_sync(kFull, less));
        const float pd = __shfl_up_sync(kFull, tk_d, 1);
        const int pi = __shfl_up_sync(kFull, tk_id, 1);
        if (lane < p.k) {
            if (lane > pos) {
                tk_d = pd;
                tk_id = pi;
            } else if (lane == pos) {
                tk_d = d;
                tk_id = id;
            }
        }
        worst_d = __shfl_sync(kFull, tk_d, p.k - 1);
        worst_id = __shfl_sync(kFull, tk_id, p.k - 1);
        return true;
    }

    __device__ __forceinline__ bool not_deleted(int id) const {
        return p.deleted == nullptr || p.deleted[id] != 1;
    }
    // StaticDispatch::CheckFilter (BKTIndex.cpp:455-458): the host evaluated the callback into one byte per vector
    __device__ __forceinline__ bool check_filter(int id) const { return p.filter == nullptr || p.filter[id] != 0; }

    __device__ __forceinline__ void issue_stage(int t, int cnt) {
        const int base = t * p.stage_rows;
        const int rows = min(p.stage_rows, cnt - base);
        const int st = t & (p.stages - 1);  // the host keeps `stages` a power of two
        if (lane == 0) mbar_arrive_expect_tx(&bars[st], (uint32_t)rows * (uint32_t)p.row_bytes);
        __syncwarp();
        if (lane < rows) {
            const int id = cand_id[base + lane];
            tma_load_1d(slot_ptr(st * p.stage_rows + lane), p.vectors + (size_t)id * p.row_stride_bytes,
                        (uint32_t)p.row_bytes, &bars[st]);
        }
    }

    // distances of the query to cand_id[0..cnt) -> cand_dist[0..cnt).  cnt <= 32.
    const float* pq_table;
    // one table entry.  Ordinary loads for both tables: an ADC table was written by this warp a moment ago, and a
    // per-look-up choice between ld.global and ld.global.nc made ptxas emit BOTH address computations and both loads,
    // predicated, for every look-up (14 instructions per look-up instead of 5).
    // (an L2 evict_last policy on these look-ups was slower at 2M x 100)
    static __device__ __forceinline__ float pq_ld(const float* tb, unsigned idx) { return tb[idx]; }

    // PQ rows: all (<= 32) code rows of the step are staged by one TMA batch, then lane r sums the M
    // table entries of candidate r in subvector order -- the reference's single float accumulator
    // (PQQuantizer::L2Distance, PQQuantizer.h:110-128), one candidate per lane.
    __device__ __forceinline__ void compute_dists_pq(int cnt) {
        __syncwarp();
        fence_proxy_async();
        if (lane == 0) mbar_arrive_expect_tx(&bars[0], (uint32_t)cnt * (uint32_t)p.row_bytes);
        __syncwarp();
        if (lane < cnt)
            tma_load_1d(ring + (size_t)lane * p.slot_stride, p.vectors + (size_t)cand_id[lane] * p.row_stride_bytes,
                        (uint32_t)p.row_bytes, &bars[0]);
        mbar_wait(&bars[0], phase_bits & 1u);
        phase_bits ^= 1u;
        if (lane < cnt) {
            const unsigned char* row = ring + (unsigned)lane * (unsigned)p.slot_stride;
            // row offsets of the query's table rows (< M * Ks * Ks, fits 32 bits): unsigned indices keep every address
            // one IMAD.WIDE.U32; the offsets are read four at a time; a code byte is one PRMT
            const unsigned* qoff = reinterpret_cast<const unsigned*>(qs);
            const float* tb = pq_table;  // the shared SDC table, or this slot's ADC table of the current query
            float acc = 0.0f;
            // 16 look-ups in flight per lane (their addresses do not depend on the running sum), then the sum in
            // sub-vector order
            const int m16 = p.pq_m & ~15;
            int i = 0;
            for (; i < m16; i += 16) {
                const uint4 w = *reinterpret_cast<const uint4*>(row + i);
                const unsigned ws[4] = {w.x, w.y, w.z, w.w};
                float t[16];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint4 qo = *reinterpret_cast<const uint4*>(qoff + i + 4 * c);
                    t[4 * c + 0] = pq_ld(tb, qo.x + __byte_perm(ws[c], 0u, 0x4440u));
                    t[4 * c + 1] = pq_ld(tb, qo.y + __byte_perm(ws[c], 0u, 0x4441u));
                    t[4 * c + 2] = pq_ld(tb, qo.z + __byte_perm(ws[c], 0u, 0x4442u));
                    t[4 * c + 3] = pq_ld(tb, qo.w + __byte_perm(ws[c], 0u, 0x4443u));
                }
#pragma unroll
                for (int b = 0; b < 16; ++b) acc = __fadd_rn(acc, t[b]);
            }
            const int m4 = p.pq_m & ~3;
            for (; i < m4; i += 4) {
                const unsigned w = *reinterpret_cast<const unsigned*>(row + i);
                const float t0 = pq_ld(tb, qoff[i] + __byte_perm(w, 0u, 0x4440u));
                const float t1 = pq_ld(tb, qoff[i + 1] + __byte_perm(w, 0u, 0x4441u));
                const float t2 = pq_ld(tb, qoff[i + 2] + __byte_perm(w, 0u, 0x4442u));
                const float t3 = pq_ld(tb, qoff[i + 3] + __byte_perm(w, 0u, 0x4443u));
                acc = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(acc, t0), t1), t2), t3);
            }
            for (; i < p.pq_m; ++i) acc = __fadd_rn(acc, pq_ld(tb, qoff[i] + (unsigned)row[i]));
            cand_dist[lane] = acc;
        }
        __syncwarp();
        ndist += cnt;
    }

    // ------------------------------------------------------------------------------------------------------------
    // 512-byte float rows (DIM == 128): the fast path.  The generic path is bound by instruction issue and per-step
    // latency, not by HBM: a large share of the warp instructions managed the run-time-shaped TMA ring or were the
    // half-warp distance with its shuffle tree, and the longest stall was the wait for the visited-bitmap atomics BEFORE the row fetch could even be issued.  Here
    //   * the ring shape is a compile-time constant: 2 stages x 8 rows, row slots 576 B apart (64 mod 128);
    //   * a quarter-warp (4 lanes) owns a row: lane q keeps accumulators 4q..4q+3 of the reference's 16, reads one
    //     conflict-free LDS.128 per 16-element chunk, and the 16 -> 8 -> 4 folds are two xor-shuffle rounds
    //     (acc256[j] = acc512[j] + acc512[j+8] pairs lanes q and q^2, acc128[j] = acc256[j] + acc256[j+4] pairs q and
    //     q^1; fp32 addition is commutative, so every lane holds the reference's bits) -- 8 rows per pass;
    // (Fetching ALL valid neighbours' rows before the bitmap atomics return was tried and was slower: only
    //  56 % of a row's neighbours are new on average at 1M x 128, so the extra row traffic outweighs the hidden latency.)
    // ------------------------------------------------------------------------------------------------------------
    static constexpr bool kFast = (DIM == 128) && (ELEM == 0) && !PQ;
    static constexpr int kFastRows = 8;
    static constexpr int kFastStride = 128 * 4 + 64;
    static constexpr int kFastRowBytes = 128 * 4;

    __device__ __forceinline__ unsigned char* fast_slot(int st, int r) const {
        return ring + (st * kFastRows + r) * kFastStride;
    }
    // rows [8t, 8t + rows) of the step: lane r of the first `rows` lanes fetches the row of vector `id`
    __device__ __forceinline__ void fast_issue(int st, int rows, int id) {
        if (lane == 0) mbar_arrive_expect_tx(&bars[st], (uint32_t)rows * (uint32_t)kFastRowBytes);
        __syncwarp();
        if (lane < rows)
            tma_load_1d(fast_slot(st, lane), p.vectors + (size_t)id * p.row_stride_bytes, (uint32_t)kFastRowBytes, &bars[st]);
    }
    // distance of the query to the 8 rows of stage `st`; lane 4r + q returns row r's value (all four lanes of a row)
    template <bool COS = COSINE>
    __device__ __forceinline__ float fast_dist8(int st) const {
        const int r = lane >> 2, q = lane & 3;
        const float4* row = reinterpret_cast<const float4*>(fast_slot(st, r)) + q;
        const float4* qv = reinterpret_cast<const float4*>(qs) + q;
        float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float4 x = qv[4 * c];
            const float4 y = row[4 * c];
            a0 = __fadd_rn(a0, dist_term<COS>(x.x, y.x));
            a1 = __fadd_rn(a1, dist_term<COS>(x.y, y.y));
            a2 = __fadd_rn(a2, dist_term<COS>(x.z, y.z));
            a3 = __fadd_rn(a3, dist_term<COS>(x.w, y.w));
        }
        // diff256 = lo(diff512) + hi(diff512): accumulators j and j + 8 live in lanes q and q ^ 2
        a0 = __fadd_rn(a0, __shfl_xor_sync(kFull, a0, 2));
        a1 = __fadd_rn(a1, __shfl_xor_sync(kFull, a1, 2));
        a2 = __fadd_rn(a2, __shfl_xor_sync(kFull, a2, 2));
        a3 = __fadd_rn(a3, __shfl_xor_sync(kFull, a3, 2));
        // diff128 = lo(diff256) + hi(diff256): j and j + 4 live in lanes q and q ^ 1
        a0 = __fadd_rn(a0, __shfl_xor_sync(kFull, a0, 1));
        a1 = __fadd_rn(a1, __shfl_xor_sync(kFull, a1, 1));
        a2 = __fadd_rn(a2, __shfl_xor_sync(kFull, a2, 1));
        a3 = __fadd_rn(a3, __shfl_xor_sync(kFull, a3, 1));
        const float sum = __fadd_rn(__fadd_rn(__fadd_rn(a0, a1), a2), a3);
        return COS ? __fsub_rn(1.0f, sum) : sum;
    }
    // cand_id[0..cnt) -> cand_dist[0..cnt).  p.stages = 2: the ring holds two 8-row stages (the copy of pass t + 1 overlaps
    // the arithmetic of pass t); p.stages = 1: one stage -- half the shared memory per slot, which is what lets 20-24
    // query slots fit on an SM (the other warps fill the gap instead of this warp's second stage)
    __device__ __forceinline__ void fast_compute_dists(int cnt) {
        __syncwarp();
        fence_proxy_async();
        const int nst = (cnt + kFastRows - 1) >> 3;
        const bool two = p.stages == 2;
        const int myid = (lane < 16 && lane < cnt) ? cand_id[lane] : 0;
        fast_issue(0, min(kFastRows, cnt), __shfl_sync(kFull, myid, lane & 7));
        if (two && nst > 1) fast_issue(1, min(kFastRows, cnt - kFastRows), __shfl_sync(kFull, myid, 8 + (lane & 7)));
        // the rows that do not fit the ring start their trip from HBM to L2 now, so that their TMA copy -- issued when a
        // ring stage frees up -- finds them there
        if (lane >= (two ? 2 * kFastRows : kFastRows) && lane < cnt)
            tma_prefetch_l2(p.vectors + (size_t)cand_id[lane] * p.row_stride_bytes, (uint32_t)kFastRowBytes);
        for (int t = 0; t < nst; ++t) {
            const int st = two ? (t & 1) : 0;
            mbar_wait(&bars[st], (phase_bits >> st) & 1u);
            phase_bits ^= (1u << st);
            const float d = fast_dist8(st);
            const int ri = kFastRows * t + (lane >> 2);
            if ((lane & 3) == 0 && ri < cnt) cand_dist[ri] = d;
            __syncwarp();
            const int nt = two ? t + 2 : t + 1;  // the pass that reuses this stage
            if (nt < nst) {
                fence_proxy_async();
                const int base = kFastRows * nt;
                fast_issue(st, min(kFastRows, cnt - base), (base + (lane & 7) < cnt) ? cand_id[base + (lane & 7)] : 0);
            }
        }
        __syncwarp();
        ndist += cnt;
    }
    __device__ __forceinline__ void compute_dists(int cnt) {
        if (cnt <= 0) return;
        if (PQ) {
            compute_dists_pq(cnt);
            return;
        }
        if (kFast) {  // compile-time
            fast_compute_dists(cnt);
            return;
        }
        __syncwarp();
        fence_proxy_async();  // earlier generic-proxy reads of the ring precede the async writes
        // stage count without an integer division (runtime divisor = a ~20-instruction emulation on the step's critical path)
        int nst = 0;
        for (int covered = 0; covered < cnt; covered += p.stage_rows) ++nst;
        const int pre = min(nst, p.stages);
        for (int t = 0; t < pre; ++t) issue_stage(t, cnt);
        for (int t = 0; t < nst; ++t) {
            const int st = t & (p.stages - 1);  // the host keeps `stages` a power of two
            mbar_wait(&bars[st], (phase_bits >> st) & 1u);
            phase_bits ^= (1u << st);
            const int base = t * p.stage_rows;
            const int rows = min(p.stage_rows, cnt - base);
            int pr = 0;
            const bool narrow = p.simd_width != 16;  // AVX / SSE trees: generic one-pair loop below
            for (; ELEM == 0 && !narrow && 2 * pr + 2 < rows; pr += 2) {  // two row pairs per pass: 2 independent chains per lane
                const int r0 = 2 * pr + half, r1 = r0 + 2;
                const float* const rws[2] = {reinterpret_cast<const float*>(slot_ptr(st * p.stage_rows + r0)),
                                             reinterpret_cast<const float*>(slot_ptr(st * p.stage_rows + r1))};
                float d2[2];
                half_warp_distance_n<DIM, COSINE, 2>(rws, qr, qs, p.dim, j, d2);
                if (j == 0) {
                    cand_dist[base + r0] = d2[0];
                    if (r1 < rows) cand_dist[base + r1] = d2[1];
                }
            }
            for (; 2 * pr < rows; ++pr) {
                const int r = 2 * pr + half;
                float d;
                if (ELEM == 0) {
                    const float* row = reinterpret_cast<const float*>(slot_ptr(st * p.stage_rows + r));
                    if (narrow)
                        d = half_warp_distance_w<COSINE>(row, qs, p.dim, j, p.simd_width);
                    else
                        d = half_warp_distance<DIM, COSINE>(row, qr, qs, p.dim, j);
                } else {
                    d = half_warp_distance_elem_w<COSINE, ELEM>(slot_ptr(st * p.stage_rows + r),
                                                                reinterpret_cast<const unsigned char*>(qs), p.dim, j, p.simd_width);
                }
                if (j == 0 && r < rows) cand_dist[base + r] = d;
            }
            __syncwarp();
            if (t + p.stages < nst) {
                fence_proxy_async();
                issue_stage(t + p.stages, cnt);
            }
        }
        __syncwarp();
        ndist += cnt;
    }

    // BKTree::InitSearchTrees (BKTree.h:696-769), m_bfs == 0
    __device__ __forceinline__ void push_children(int cs, int ce) {
        for (int base = cs; base < ce; base += 32) {
            const int cnt = min(32, ce - base);
            __syncwarp();
            if (lane < cnt) cand_id[lane] = p.nodes[3 * (base + lane)];
            ntree += cnt;
            compute_dists(cnt);
            for (int r = 0; r < cnt; ++r) hins(spt, base + r, cand_dist[r]);
        }
    }

    __device__ __forceinline__ void init_search_trees() {
        for (int t = 0; t < p.tree_num; ++t) {
            const int start = p.tree_starts[t];
            const int centerid = p.nodes[3 * start], cs = p.nodes[3 * start + 1], ce = p.nodes[3 * start + 2];
            ntree++;
            if (cs < 0) {
                __syncwarp();
                if (lane == 0) cand_id[0] = centerid;
                compute_dists(1);
                hins(spt, start, cand_dist[0]);
            } else {
                // (a compile-time branch: a dead call alone changes the other kernels' code)
                if constexpr (BFS) {
                    if (p.bfs != 0) {
                        init_search_trees_bfs(cs, ce);
                        continue;
                    }
                }
                push_children(cs, ce);
            }
        }
    }

    // ---- BKTree::InitSearchTrees, m_bfs != 0 (BKTree.h:703-758) ----
    // m_currBSPTQueue / m_nextBSPTQueue: Heap<NodeDistPair> of MaxBFSNodes entries, held wholly in HBM at the end of this
    // query's SPTQueue arena (s = g, so every access is a plain global load / store) and emulated by the same insert and
    // pop as the queues.  They live only while a tree is seeded.
    __device__ __forceinline__ WarpHeap bfs_heap(int which) const {
        WarpHeap h;
        h.s = h.g = spt.g + p.spt_spill_entries - (size_t)(2 - which) * kBfsHeapEntries;
        h.H = kBfsMaxNodes;
        h.count = 0;
        h.length = kBfsMaxNodes;
        h.lastlevel = 64;  // never read: admission keeps count below length, so insert never takes the full-heap branch
        h.tail_idx = -1;
        return h;
    }
    // The children [cs, ce) in child order: into `q` while dist <= 1.1f * q.Top() (an fp32 product) and q holds fewer than
    // MaxBFSNodes, into SPTQueue otherwise.  Top() of the empty heap is the 1e9 the reference writes into heap[0]; the
    // top after an insert is the new pair exactly when it is smaller than the old top (the sift-up compares with <).
    __device__ __forceinline__ void bfs_admit(WarpHeap& q, int cs, int ce) {
        float top = q.count == 0 ? 1e9f : pair_dist(heap_ld(q, 1));
        for (int base = cs; base < ce; base += 32) {
            const int cnt = min(32, ce - base);
            __syncwarp();
            if (lane < cnt) cand_id[lane] = p.nodes[3 * (base + lane)];
            ntree += cnt;
            compute_dists(cnt);
            for (int r = 0; r < cnt; ++r) {
                const float d = cand_dist[r];
                if (d <= __fmul_rn(1.1f, top) && q.count < kBfsMaxNodes) {
                    if (q.count == 0 || d < top) top = d;
                    heap_insert<false>(q, base + r, d, lane);
                } else {
                    hins(spt, base + r, d);
                }
            }
        }
    }
    // One tree whose root has children [cs, ce).  Levels run while `curr` holds nodes: once it is empty every later level
    // of the reference's m_bfs loop does nothing.  A popped leaf goes to SPTQueue (no CheckAndSet, not counted); a popped
    // internal node's centre enters NGQueue if new (not counted as a checked leaf) and its children are admitted to `next`.
    __device__ __forceinline__ void init_search_trees_bfs(int cs, int ce) {
        WarpHeap curr = bfs_heap(0), next = bfs_heap(1);
        bfs_admit(curr, cs, ce);
        for (int level = 1; level <= p.bfs && curr.count != 0; ++level) {
            while (curr.count != 0) {
                const int2 tmp = heap_pop_seq(curr, lane);
                const int tcenter = p.nodes[3 * tmp.x], tcs = p.nodes[3 * tmp.x + 1], tce = p.nodes[3 * tmp.x + 2];
                ntree++;
                if (tcs < 0) {
                    hins(spt, tmp.x, pair_dist(tmp));
                } else {
                    if (!check_and_set_uniform(tcenter)) hins(ng, tcenter, pair_dist(tmp));
                    bfs_admit(next, tcs, tce);
                }
            }
            const WarpHeap t = curr;
            curr = next;
            next = t;
        }
        while (curr.count != 0) {
            const int2 e = heap_pop_seq(curr, lane);
            hins(spt, e.x, pair_dist(e));
        }
    }

    // the table is at its limit before a SearchTrees pop (each pop inserts at most one centre): QHASH records the cut, at
    // which an iterator call suspends
    __device__ __forceinline__ bool trees_full() {
        if (!vset_full()) return false;
        if (QHASH) trees_cut = true;
        return true;
    }

    // BKTree::SearchTrees (BKTree.h:771-799)
    __device__ __forceinline__ void search_trees(int limit) {
        while (spt.count != 0 && !trees_full()) {
            const int2 bcell = hpop(spt);
            const int centerid = p.nodes[3 * bcell.x], cs = p.nodes[3 * bcell.x + 1], ce = p.nodes[3 * bcell.x + 2];
            ntree++;
            // leaf or internal node alike: a centre that was not visited yet enters NGQueue (BKTree.h:780-795); only new
            // LEAVES count as checked
            if (!check_and_set_uniform(centerid)) {
                if (cs < 0) checked++;
                hins(ng, centerid, pair_dist(bcell));
            }
            if (cs < 0) {
                if (checked >= limit) break;
            } else {
                push_children(cs, ce);
            }
        }
    }

    // The visited-set update of one 32-wide chunk of a graph row (OptHashPosVector::CheckAndSet per neighbour, in
    // neighbour order): the scan stops at the first negative entry (BKTIndex.cpp:333-336); a repeated id inside the row is
    // "visited" by the time its second copy is reached, so only the first occurrence (the leader) touches the bitmap.
    // issue_mark starts the atomics and returns without reading their result; the caller overlaps other work with the
    // round trip and asks for the verdict later.
    // Hashed set: the first probe is an atomicCAS at the home position (leaders hold distinct ids and the table is this
    // warp's own, so only lanes of this warp race); `bit` holds the position and `old` what the CAS found.
    struct RowMark {
        int first_neg;
        bool leader;
        unsigned bit, old;
    };
    __device__ __forceinline__ RowMark issue_mark(int nn, bool in_row) {
        RowMark m;
        const unsigned negmask = __ballot_sync(kFull, in_row && nn < 0) | ~__ballot_sync(kFull, in_row);
        m.first_neg = negmask ? (__ffs(negmask) - 1) : 32;
        const bool active = lane < m.first_neg;
        const unsigned same = __match_any_sync(kFull, active ? nn : (-1 - lane));
        m.leader = active && ((__ffs(same) - 1) == lane);
        m.old = 0xffffffffu;
        if (hashed()) {
            m.leader = m.leader && !vset_full();
            m.bit = vhash_home(nn);
            if (m.leader) m.old = atomicCAS(&visited[m.bit], 0u, (unsigned)nn + 1u);
        } else {
            m.bit = 1u << (nn & 31);
            if (m.leader) m.old = atomicOr(&visited[nn >> 5], m.bit);
        }
        return m;
    }
    // the verdict of issue_mark: this lane's id was not visited before.  Hashed set: the probe continues past positions
    // that hold other ids (another lane's id may have just taken the home position); `bit` ends at the id's position.
    __device__ __forceinline__ bool mark_fresh(RowMark& m, int nn) {
        if (!hashed()) return m.leader && (m.old & m.bit) == 0;
        if (!m.leader || m.old == (unsigned)nn + 1u) return false;
        if (m.old == 0u) return true;
        const unsigned r = vhash_probe(visited, m.bit, (unsigned)nn + 1u, vhash_mask());
        m.bit = r & ~kVhashFound;
        return (r & kVhashFound) == 0;
    }
    // what the clear log records for a fresh id: its bitmap word, or its table position
    __device__ __forceinline__ unsigned mark_word(const RowMark& m, int nn) const {
        return hashed() ? m.bit : (unsigned)(nn >> 5);
    }
    // L2 prefetch of the bitmap words (table home positions) the next step will update (no data returns to the SM)
    __device__ __forceinline__ void prefetch_marks(int nn) {
        if (nn >= 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(visited + (hashed() ? vhash_home(nn) : (unsigned)(nn >> 5))));
    }

    // One graph-row chunk after issue_mark: its fresh ids compacted into cand_id in neighbour order (and logged), and their
    // distances in cand_dist.  Returns how many there are.  The iterator kernels bind no clear log (vlog = nullptr: their
    // sets persist across calls), so the log store compiles away there; binding one would add it to every chunk.
    // GATED: the caller drops every candidate whose distance is above mres.worst (BKT Search), so the sketch may stand in
    // for the row of such a candidate
    template <bool GATED = false>
    __device__ __forceinline__ int expand_chunk(RowMark& mark, int nn) {
        const bool fresh = mark_fresh(mark, nn);
        const unsigned freshmask = __ballot_sync(kFull, fresh);
        const int cnt = __popc(freshmask);
        __syncwarp();
        if (fresh) {
            const int rank = __popc(freshmask & ((1u << lane) - 1u));
            cand_id[rank] = nn;
            if (vlog != nullptr && vlog_count + rank < (int)p.vlog_entries) vlog[vlog_count + rank] = mark_word(mark, nn);
        }
        vlog_count += cnt;
        if constexpr (GATED && SKETCH)
            compute_dists_gated(cnt);
        else
            compute_dists(cnt);
        return cnt;
    }

    // compute_dists for candidates that only matter while their distance is <= mres.worst.  Pass 1 stages the candidates'
    // sketch rows, tail included, through the row ring, which the row pass cannot use before the bounds exist: one TMA
    // batch of p.sketch_batch rows against bars[0] per round trip, while the rows of the later batches are prefetched
    // into L2.  From shared memory the warp multiplies two rows at a time with the query's sketch (lane l the 16-byte
    // vectors l, l + 32, ... of a row: conflict-free), and lane r bounds candidate r's distance from below as soon as its
    // batch is done.  Pass 2 fetches the rows of the others only, compacted in neighbour order, and their distances are
    // the reference's bits; a candidate that was proven above worst gets its bound as its distance.  worst never
    // increases, so the caller drops it wherever the true distance would have been dropped, and every counter advances
    // as if the row had been read.  Until m_Results is full its worst is MaxDist and nothing is skipped.
    // (Two rows per group and the bound per batch keep every sketch kernel within its register cap without spills.)
    __device__ __forceinline__ void compute_dists_gated(int cnt) {
        if (cnt <= 0) return;
        __syncwarp();
        const int myid = (lane < cnt) ? cand_id[lane] : 0;
        const float worst = mres.worst;
        float lb = -INFINITY;
        if (worst < SPTAG_B200_MAXDIST) {  // (warp-uniform)
            const int stride = (int)sketch_stride(p.dim);
            const int nvec = ((DIM > 0) ? sketch_elems(DIM) : sketch_elems(p.dim)) >> 4;  // 16-byte vectors per row
            const int batch = p.sketch_batch;
            if (lane >= batch && lane < cnt) tma_prefetch_l2(p.sketch + (size_t)myid * stride, (uint32_t)stride);
            for (int b0 = 0; b0 < cnt; b0 += batch) {
                const int nb = min(batch, cnt - b0);
                const bool in_batch = lane >= b0 && lane < b0 + nb;
                __syncwarp();
                fence_proxy_async();  // earlier generic-proxy reads of the ring precede the async writes
                if (lane == 0) mbar_arrive_expect_tx(&bars[0], (uint32_t)(nb * stride));
                __syncwarp();
                if (in_batch) tma_load_1d(ring + (lane - b0) * stride, p.sketch + (size_t)myid * stride, (uint32_t)stride, &bars[0]);
                mbar_wait(&bars[0], phase_bits & 1u);
                phase_bits ^= 1u;
                int myI = 0;
                for (int r0 = 0; r0 < nb; r0 += 2) {
                    const unsigned* const rw[2] = {reinterpret_cast<const unsigned*>(ring + r0 * stride),
                                                   reinterpret_cast<const unsigned*>(ring + min(r0 + 1, nb - 1) * stride)};
                    int acc[2] = {0, 0};
                    for (int v = lane; v < nvec; v += 32) {
                        unsigned t[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) t[e] = tq[4 * v + e];
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
#pragma unroll
                            for (int e = 0; e < 4; ++e) acc[u] = __dp4a((int)rw[u][4 * v + e], (int)t[e], acc[u]);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int I = __reduce_add_sync(kFull, acc[u]);
                        if (r0 + u < nb && lane == b0 + r0 + u) myI = I;
                    }
                }
                if (in_batch)
                    lb = sketch_lower_bound<COSINE>(myI, tq_tail, *reinterpret_cast<const RowSketchTail*>(ring + (lane - b0) * stride + 16 * nvec),
                                                    sketch_rel_margin(p.dim));
            }
        }
        const bool keep = (lane < cnt) && !(lb > worst);
        const unsigned keepmask = __ballot_sync(kFull, keep);
        const int nkeep = __popc(keepmask);
        const int rank = __popc(keepmask & ((1u << lane) - 1u));
        __syncwarp();
        if (keep) cand_id[rank] = myid;
        compute_dists(nkeep);
        const float d = keep ? cand_dist[rank] : lb;
        __syncwarp();
        if (lane < cnt) {
            cand_id[lane] = myid;
            cand_dist[lane] = d;
        }
        __syncwarp();
        ndist += cnt - nkeep;
        nskipped += cnt - nkeep;
    }

    // BKT Search's accept of the popped node (BKTIndex.cpp:292-320): a node whose last graph entry `checkNode` points back
    // to a duplicate group (< -1) offers every live member of that group to m_Results at its distance
    __device__ __forceinline__ void add_node_or_group(int tmpNode, float gdist, int checkNode) {
        if (checkNode < -1) {
            const int tn = -2 - checkNode;
            const int tcs = p.nodes[3 * tn + 1], tce = p.nodes[3 * tn + 2];
            int i = -tcs;
            do {
                if (not_deleted(tmpNode)) {
                    if (check_filter(tmpNode)) {
                        if (!add_point(tmpNode, gdist) || p.never_dup) break;
                    }
                }
                if (i <= 0) break;
                tmpNode = p.nodes[3 * i];
            } while (i++ < tce);
        } else {
            if (not_deleted(tmpNode) && check_filter(tmpNode)) add_point(tmpNode, gdist);
        }
    }

    // BKT::Index<T>::Search<notDeleted, CheckDup, AlwaysTrue> (BKTIndex.cpp:268-352).
    // One step's memory round trips are data-dependent (queue root -> graph row -> visited set -> vectors), so the order
    // inside a step is chosen to overlap them: the root of NGQueue is the popped node before the sift-down runs, so the
    // accept / stop logic (which never looks at the queue) and the visited-set atomics are issued first and Heap::pop's
    // sift-down runs while they are in flight; the graph row of the node that is on top AFTER the pop is fetched a step
    // ahead (the CPU does the same with _mm_prefetch, BKTIndex.cpp:283-288), and when it is still on top at the end of
    // the step the bitmap words of its neighbours are prefetched into L2.
    __device__ __forceinline__ void bkt_search_fast() {
        init_search_trees();
        const int checkPos = p.degree - 1;
        int pre_id = -1, pre_nn = -1;
        // (search_trees appears once in the code: the kernels are far larger than the instruction cache.  First trip:
        //  SearchTrees(NumberOfInitialDynamicPivots) before the loop; later trips: the re-seeding test at the end of a step)
        bool reseed = true;
        int tree_limit = p.initial_pivots;
        for (;;) {
            if (reseed) search_trees(tree_limit);
            if (pre_id >= 0 && ng.count != 0 && ng.s[1].x == pre_id) prefetch_marks(pre_nn);
            if (ng.count == 0 || vset_full()) break;
            const int2 gnode = ng.s[1];  // what Heap::pop will return
            int tmpNode = gnode.x;
            const float gdist = pair_dist(gnode);
            const int* node = p.graph + (size_t)tmpNode * p.degree;
            nexpand++;
            // lane i holds neighbour i of the first 32-wide chunk
            int nn;
            if (tmpNode == pre_id)
                nn = pre_nn;
            else
                nn = (lane <= checkPos) ? node[lane] : -1;

            bool stop = false;
            if (gdist <= worst_d) {
                add_node_or_group(tmpNode, gdist, (checkPos < 32) ? __shfl_sync(kFull, nn, checkPos) : node[checkPos]);
            } else {
                if (not_deleted(tmpNode)) stop = (gdist > mres.worst || checked > p.max_check);
            }

            RowMark mark;
            mark.first_neg = 0;
            mark.leader = false;
            mark.bit = mark.old = 0u;
            if (!stop) mark = issue_mark(nn, lane <= checkPos);
            hpop(ng);  // sift-down, while the atomics are in flight (the reference pops before it looks at the node)
            if (stop) return;
            if (!kLean) {
                pre_id = (ng.count != 0) ? ng.s[1].x : -1;
                pre_nn = (pre_id >= 0 && lane <= checkPos) ? p.graph[(size_t)pre_id * p.degree + lane] : -1;
            }

            for (int cbase = 0; cbase <= checkPos; cbase += 32) {
                if (cbase > 0) {
                    nn = (cbase + lane <= checkPos) ? node[cbase + lane] : -1;
                    mark = issue_mark(nn, cbase + lane <= checkPos);
                }
                const int cnt = expand_chunk(mark, nn);
                // m_Results.worst() never increases, so a candidate above the current worst is rejected
                // whenever its turn comes; only the others are replayed in neighbour order (BKTIndex.cpp:338-344)
                const float myd = (lane < cnt) ? cand_dist[lane] : SPTAG_B200_MAXDIST;
                const int myid = (lane < cnt) ? cand_id[lane] : -1;
                checked += cnt;
                unsigned maybe = __ballot_sync(kFull, lane < cnt && !(myd > mres.worst));
                while (maybe) {
                    const int r = __ffs(maybe) - 1;
                    maybe &= maybe - 1;
                    const float d = __shfl_sync(kFull, myd, r);
                    const int id = __shfl_sync(kFull, myid, r);
                    if (mres.insert(d, lane)) hins(ng, id, d);
                }
                if (mark.first_neg < 32) break;
            }
            reseed = heap_top_dist(ng) > heap_top_dist(spt);
            tree_limit = p.other_pivots + checked;
        }
    }

    // BKT::Index<T>::Search<notDeleted, CheckDup, AlwaysTrue> (BKTIndex.cpp:268-352), round-1 step order (pop, row, visited, rows)
    __device__ __forceinline__ void bkt_search_legacy() {
        init_search_trees();
        const int checkPos = p.degree - 1;
        // (one copy of search_trees in the code: first trip = SearchTrees(NumberOfInitialDynamicPivots), later trips = the
        //  re-seeding test at the end of a step)
        bool reseed = true;
        int tree_limit = p.initial_pivots;
        for (;;) {
            if (reseed) search_trees(tree_limit);
            if (ng.count == 0 || vset_full()) break;
            const int2 gnode = hpop(ng);
            int tmpNode = gnode.x;
            const float gdist = pair_dist(gnode);
            const int* node = p.graph + (size_t)tmpNode * p.degree;
            nexpand++;
            // lane i reads neighbour i of the first 32-wide chunk while the accept logic runs
            int nn = (lane <= checkPos) ? node[lane] : -1;

            if (gdist <= worst_d) {
                add_node_or_group(tmpNode, gdist, node[checkPos]);
            } else {
                if (not_deleted(tmpNode)) {
                    if (gdist > mres.worst || checked > p.max_check) return;
                }
            }

            for (int cbase = 0; cbase <= checkPos; cbase += 32) {
                if (cbase > 0) nn = (cbase + lane <= checkPos) ? node[cbase + lane] : -1;
                // the scan stops at the first negative entry (BKTIndex.cpp:333-336); a repeated id inside the row is
                // "visited" by the time its second copy is reached
                RowMark mark = issue_mark(nn, cbase + lane <= checkPos);
                const int cnt = expand_chunk<true>(mark, nn);
                // m_Results.worst() never increases, so a candidate above the current worst is rejected
                // whenever its turn comes; only the others are replayed in neighbour order (BKTIndex.cpp:338-344)
                const float myd = (lane < cnt) ? cand_dist[lane] : SPTAG_B200_MAXDIST;
                const int myid = (lane < cnt) ? cand_id[lane] : -1;
                checked += cnt;
                unsigned maybe = __ballot_sync(kFull, lane < cnt && !(myd > mres.worst));
                while (maybe) {
                    const int r = __ffs(maybe) - 1;
                    maybe &= maybe - 1;
                    const float d = __shfl_sync(kFull, myd, r);
                    const int id = __shfl_sync(kFull, myid, r);
                    if (mres.insert(d, lane)) hins(ng, id, d);
                }
                if (mark.first_neg < 32) break;
            }
            reseed = heap_top_dist(ng) > heap_top_dist(spt);
            tree_limit = p.other_pivots + checked;
        }
    }

    __device__ __forceinline__ void bkt_search() {
        if (kLean)
            bkt_search_legacy();
        else
            bkt_search_fast();
    }
    __device__ __forceinline__ void kdt_search() {
        if (kLean)
            kdt_search_legacy();
        else
            kdt_search_fast();
    }

    // ------------------------------------------------------------------------------------
    // BKT::Index<T>::SearchIterative<notDeleted, isDup> (BKTIndex.cpp:354-427): the resumable loop behind
    // ResultIterator::Next.  Differences from Search: every popped live node is a result (at most `batch` per call),
    // neighbours enter NGQueue unconditionally (m_Results only feeds the relaxed-monotonicity flag), duplicate-group
    // members get their own distance and enter NGQueue, and there is no stop rule besides `count >= batch`.
    // Results are appended to this query's arena `tk` (sorted afterwards); `count` is resultCount.
    // A query on a hash table (QHASH) suspends where its state can be saved instead of losing an insert: at the top of a
    // step that could take the fill past the limit (`margin` = degree + largest duplicate group + 1 bounds what one step
    // inserts), and before a SearchTrees pop at the limit.  `at` enters as where the call starts (kIterFirst, kIterStep) or
    // resumes, and leaves as kIterDone or the resume point; `limit` is the pending SearchTrees limit.
    // ------------------------------------------------------------------------------------
    __device__ __forceinline__ void bkt_search_iterative(int& at, int batch, int& relaxed, int& count, int& limit,
                                                         int margin) {
        if (at == kIterFirst) {
            init_search_trees();
            at = kIterInitTrees;
            limit = p.initial_pivots;
        }
        if (at != kIterStep) {  // the first call's trees, or a resumed in-step SearchTrees
            trees_cut = false;
            search_trees(limit);
            if (QHASH && trees_cut) return;
            if (at == kIterStepTrees && count >= batch) {
                at = kIterDone;
                return;
            }
        }
        const int checkPos = p.degree - 1;
        while (ng.count != 0) {
            if (QHASH && vlog_count + margin > qlimit) {
                at = kIterStep;
                return;
            }
            const int2 gnode = hpop(ng);
            const int popped = gnode.x;
            const float gdist = pair_dist(gnode);
            const int* node = p.graph + (size_t)popped * p.degree;
            nexpand++;
            int nn = (lane <= checkPos) ? node[lane] : -1;
            if (not_deleted(popped)) {
                if (lane == 0) tk[tk_count] = make_pair(popped, gdist);
                ++tk_count;
                ++count;
                if (gdist > mres.worst || checked > p.max_check) relaxed = 1;
            }
            const int checkNode = node[checkPos];
            if (checkNode < -1) {
                const int tn = -2 - checkNode;
                const int tcs = p.nodes[3 * tn + 1], tce = p.nodes[3 * tn + 2];
                for (int base = -tcs; base < tce; base += 32) {
                    const int i = base + lane;
                    const int id = (i < tce) ? p.nodes[3 * i] : -1;
                    const bool live = (i < tce) && not_deleted(id);
                    const unsigned livemask = __ballot_sync(kFull, live);
                    const int cnt = __popc(livemask);
                    __syncwarp();
                    if (live) cand_id[__popc(livemask & ((1u << lane) - 1u))] = id;
                    compute_dists(cnt);
                    for (int r = 0; r < cnt; ++r) {  // the distance is taken first, CheckAndSet second (:394-401)
                        const int mid = cand_id[r];
                        const float md = cand_dist[r];
                        if (!check_and_set_uniform(mid)) hins(ng, mid, md);
                    }
                    __syncwarp();
                }
            }
            for (int cbase = 0; cbase <= checkPos; cbase += 32) {
                if (cbase > 0) nn = (cbase + lane <= checkPos) ? node[cbase + lane] : -1;
                RowMark mark = issue_mark(nn, cbase + lane <= checkPos);
                const int cnt = expand_chunk(mark, nn);
                checked += cnt;
                for (int r = 0; r < cnt; ++r) {
                    const int id = cand_id[r];
                    const float d = cand_dist[r];
                    hins(ng, id, d);
                    mres.insert(d, lane);
                }
                __syncwarp();
                if (mark.first_neg < 32) break;
            }
            if (heap_top_dist(ng) > heap_top_dist(spt)) {
                limit = p.other_pivots + checked;
                trees_cut = false;
                search_trees(limit);
                if (QHASH && trees_cut) {
                    at = kIterStepTrees;
                    return;
                }
            }
            if (count >= batch) break;
        }
        at = kIterDone;
    }

    // SearchIndexIterativeFromNeareast, first call (BKTIndex.cpp:549-572): one result of the finished search is marked
    // visited and its not-yet-visited graph neighbours enter NGQueue with their distances (no budget accounting, no
    // m_Results)
    __device__ __forceinline__ void seed_from_result(int result) {
        check_and_set_uniform(result);
        const int checkPos = p.degree - 1;
        const int* node = p.graph + (size_t)result * p.degree;
        for (int cbase = 0; cbase <= checkPos; cbase += 32) {
            const bool in_row = (cbase + lane <= checkPos);
            const int nn = in_row ? node[cbase + lane] : -1;
            RowMark mark = issue_mark(nn, in_row);
            const int cnt = expand_chunk(mark, nn);
            for (int r = 0; r < cnt; ++r) hins(ng, cand_id[r], cand_dist[r]);
            __syncwarp();
            if (mark.first_neg < 32) break;
        }
    }

    // ------------------------------------------------------------------------------------
    // KDT flavour: KDTree::KDTSearch (KDTree.h:233-271, tail recursion as a loop),
    // InitSearchTrees/SearchTrees (KDTree.h:213-231), KDT::Index<T>::Search (KDTIndex.cpp:182-241)
    // ------------------------------------------------------------------------------------
    __device__ __forceinline__ void kdt_search_node(int node, float distBound) {
        for (;;) {
            if (node < 0) {
                const int index = -node - 1;
                if (index >= p.n) return;
                if (check_and_set_uniform<false>(index)) return;
                ++tree_checked;
                ++checked;
                __syncwarp();
                if (lane == 0) cand_id[0] = index;
                compute_dists(1);
                hins_k(ng, index, cand_dist[0]);
                return;
            }
            const int4 tn = __ldg(reinterpret_cast<const int4*>(p.nodes) + node);  // {left, right, split_dim, split_value}
            ntree++;
            // the split test reads the raw query (KDTree.h:255); `distBound + diff*diff` is one FMA in the
            // reference's g++ -O3 build (see oracle/sptag_oracle.c kdt_search_node)
            float qv;
            if (ELEM == 0)
                qv = qs[tn.z];
            else
                qv = int_query_elem<ELEM>(qs, tn.z);
            const float diff = __fsub_rn(qv, __int_as_float(tn.w));
            const float distanceBound = __fmaf_rn(diff, diff, distBound);
            int otherChild, bestChild;
            if (diff < 0) {
                bestChild = tn.x;
                otherChild = tn.y;
            } else {
                otherChild = tn.x;
                bestChild = tn.y;
            }
            hins_k(spt, otherChild, distanceBound);
            node = bestChild;
        }
    }

    __device__ __forceinline__ void kdt_search_trees(int limit) {
        while (spt.count != 0 && checked < limit && !vset_full()) {
            const int2 tcell = hpop_k(spt);
            kdt_search_node(tcell.x, pair_dist(tcell));
        }
    }

    __device__ __forceinline__ void kdt_search_fast() {
        for (int t = 0; t < p.tree_num; ++t) kdt_search_node(p.tree_starts[t], 0.0f);
        kdt_search_trees(p.initial_pivots);
        int pre_id = -1, pre_nn = -1;  // graph row of NGQueue's new top, fetched one step ahead (see bkt_search)
        while (ng.count != 0 && !vset_full()) {
            const int2 gnode = ng.s[1];  // what Heap::pop will return
            const float gdist = pair_dist(gnode);
            const int* node = p.graph + (size_t)gnode.x * p.degree;
            nexpand++;
            int nn;
            if (gnode.x == pre_id)
                nn = pre_nn;
            else
                nn = (lane < p.degree) ? node[lane] : -1;
            if (not_deleted(gnode.x)) {
                if (!add_point(gnode.x, gdist) && checked > p.max_check) {
                    hpop_k(ng);
                    return;
                }
            }
            const float upperBound = fmaxf(worst_d, gdist);
            bool bLocalOpt = true;
            RowMark mark = issue_mark(nn, lane < p.degree);
            hpop_k(ng);  // sift-down, while the atomics are in flight
            pre_id = (ng.count != 0) ? ng.s[1].x : -1;
            pre_nn = (pre_id >= 0 && lane < p.degree) ? p.graph[(size_t)pre_id * p.degree + lane] : -1;
            for (int cbase = 0; cbase < p.degree; cbase += 32) {
                if (cbase > 0) {
                    nn = (cbase + lane < p.degree) ? node[cbase + lane] : -1;
                    mark = issue_mark(nn, cbase + lane < p.degree);
                }
                const int cnt = expand_chunk(mark, nn);
                // every new neighbour enters NGQueue, in neighbour order (KDTIndex.cpp:212-223)
                const float myd = (lane < cnt) ? cand_dist[lane] : SPTAG_B200_MAXDIST;
                const int myid = (lane < cnt) ? cand_id[lane] : -1;
                if (__any_sync(kFull, lane < cnt && myd <= upperBound)) bLocalOpt = false;
                checked += cnt;
                for (int r = 0; r < cnt; ++r) hins_k(ng, __shfl_sync(kFull, myid, r), __shfl_sync(kFull, myd, r));
                if (mark.first_neg < 32) break;
            }
            if (bLocalOpt)
                no_better++;
            else
                no_better = 0;
            if (no_better > p.no_better_threshold) {
                if (tree_checked <= checked / 10) {
                    kdt_search_trees(p.other_pivots + checked);
                } else if (gdist > worst_d) {
                    break;
                }
            }
            if (pre_id >= 0 && ng.count != 0 && ng.s[1].x == pre_id) prefetch_marks(pre_nn);
        }
    }

    __device__ __forceinline__ void kdt_search_legacy() {
        for (int t = 0; t < p.tree_num; ++t) kdt_search_node(p.tree_starts[t], 0.0f);
        kdt_search_trees(p.initial_pivots);
        while (ng.count != 0 && !vset_full()) {
            const int2 gnode = hpop(ng);
            const float gdist = pair_dist(gnode);
            const int* node = p.graph + (size_t)gnode.x * p.degree;
            nexpand++;
            int nn = (lane < p.degree) ? node[lane] : -1;
            if (not_deleted(gnode.x)) {
                if (!add_point(gnode.x, gdist) && checked > p.max_check) return;
            }
            const float upperBound = fmaxf(worst_d, gdist);
            bool bLocalOpt = true;
            for (int cbase = 0; cbase < p.degree; cbase += 32) {
                if (cbase > 0) nn = (cbase + lane < p.degree) ? node[cbase + lane] : -1;
                RowMark mark = issue_mark(nn, cbase + lane < p.degree);
                const int cnt = expand_chunk(mark, nn);
                for (int r = 0; r < cnt; ++r) {
                    const float d = cand_dist[r];
                    if (d <= upperBound) bLocalOpt = false;
                    checked++;
                    hins(ng, cand_id[r], d);
                }
                if (mark.first_neg < 32) break;
            }
            if (bLocalOpt)
                no_better++;
            else
                no_better = 0;
            if (no_better > p.no_better_threshold) {
                if (tree_checked <= checked / 10) {
                    kdt_search_trees(p.other_pivots + checked);
                } else if (gdist > worst_d) {
                    break;
                }
            }
        }
    }
};

// The per-query visited set of an iterator kernel: its table or bitmap, and the table's capacity
template <typename W>
__device__ __forceinline__ void bind_iter_visited(W& w, const SearchParams& p, const IterVisited& iv, int q, int bits) {
    w.visited = iv.tables ? iv.tables[q] : p.visited + (size_t)q * p.visited_words;
    w.qmask = bits ? (1u << bits) - 1u : 0u;
    w.qshift = 32 - bits;
    w.qlimit = bits ? 1 << (bits - 1) : INT_MAX;
}
// The next query of an iterator launch: every query, or those on the resume list; -1 when none is left
__device__ __forceinline__ int next_iter_query(const SearchParams& p, const IterVisited& iv, int lane) {
    unsigned i = 0;
    if (lane == 0) i = atomicAdd(p.work_counter, 1u);
    i = __shfl_sync(kFull, i, 0);
    if (iv.list) return i < iv.list[0] ? (int)iv.list[kIterListHeader + i] : -1;
    return i < (unsigned)p.nq ? (int)i : -1;
}
// Append q to the suspension list; `kind` (1 or 2) counts it as a step or a tree suspension, 0 not at all
__device__ __forceinline__ void suspend_iter_query(const IterVisited& iv, int q, int kind, int lane) {
    if (lane == 0) {
        iv.suspended[kIterListHeader + atomicAdd(iv.suspended, 1u)] = (unsigned)q;
        if (kind) atomicAdd(iv.suspended + kind, 1u);
    }
}

// The kernels: search_kernel, iterate_kernel and nearest_first_kernel as they are, and the same text in namespace bfs with
// breadth-first tree seeding (EnableBfs != 0), instantiated for the generic-dimension, integer and PQ rows only
// and once more in namespace sketch with the row-sketch test in BKT search's graph step (search_kernel only is instantiated)
#define SPTAG_B200_SKETCH false
#define SPTAG_B200_BFS false
#include "search_kernel_defs.cuh"
#undef SPTAG_B200_BFS
namespace bfs {
#define SPTAG_B200_BFS true
#include "search_kernel_defs.cuh"
#undef SPTAG_B200_BFS
}  // namespace bfs
#undef SPTAG_B200_SKETCH
namespace sketch {
#define SPTAG_B200_SKETCH true
#define SPTAG_B200_BFS false
#include "search_kernel_defs.cuh"
#undef SPTAG_B200_BFS
#undef SPTAG_B200_SKETCH
}  // namespace sketch

}  // namespace sptag_b200
