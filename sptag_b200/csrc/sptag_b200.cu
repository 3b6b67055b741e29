// sptag_b200.cu -- C-ABI implementation (include/sptag_b200.h) over the sm_90a search kernels.
//
// Host side of the drop-in boundary: index upload (the arrays BKT::Index<T> keeps in m_pSamples /
// m_pGraph / m_pTrees / m_deletedID, AnnService/inc/Core/BKT/Index.h), the reference's on-disk
// folder reader (VectorIndex.cpp:617-681), parameter handling with the reference's names
// (BKT/ParameterDefinitionList.h:44-49), per-slot scratch management and the kernel launches.
// No torch, no CPU fallback: a search either runs the CUDA kernels or returns an error code.
#include "../../include/sptag_b200.h"
#include "aux_kernels.cuh"
#include "kernel_select.h"

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <mutex>
#include <sys/stat.h>
#include <sstream>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

using namespace sptag_b200;

namespace {

thread_local std::string g_last_error;
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define CUDA_OK(expr)                                                                            \
    do {                                                                                         \
        cudaError_t e__ = (expr);                                                                \
        if (e__ != cudaSuccess)                                                                  \
            return fail(SPTAG_B200_FAIL, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                        __FILE__, __LINE__);                                                     \
    } while (0)

// An owned device allocation.  Its owner is destroyed with the allocation's device current (DeviceGuard); release()
// frees it earlier.
struct DeviceBuffer {
    void* ptr = nullptr;
    size_t bytes = 0;
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : ptr(std::exchange(o.ptr, nullptr)), bytes(std::exchange(o.bytes, 0)) {}
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        if (this != &o) {
            release();
            ptr = std::exchange(o.ptr, nullptr);
            bytes = std::exchange(o.bytes, 0);
        }
        return *this;
    }
    ~DeviceBuffer() { release(); }
    int ensure(size_t need) {
        if (need <= bytes) return 0;
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
        cudaError_t e = cudaMalloc(&ptr, need);
        if (e != cudaSuccess) return fail(SPTAG_B200_MEMORY_OVERFLOW, "cudaMalloc(%zu) failed: %s", need,
                                          cudaGetErrorString(e));
        bytes = need;
        return 0;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
    }
};

size_t value_size(int vt) {
    switch (vt) {
    case SPTAG_B200_VT_INT8:
    case SPTAG_B200_VT_UINT8: return 1;
    case SPTAG_B200_VT_INT16: return 2;
    case SPTAG_B200_VT_FLOAT: return 4;
    }
    return 0;
}

size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

struct sptag_b200_index {
    int device = 0;
    int algo = 0, value_type = SPTAG_B200_VT_FLOAT, metric = 0;
    int n = 0, dim = 0, degree = 0, tree_num = 0, node_count = 0, num_deleted = 0, id_offset = 0;
    size_t row_stride = 0;  // bytes, multiple of 16
    // device-resident index
    DeviceBuffer d_vectors, d_graph, d_nodes, d_tree_starts, d_deleted;
    int search_deleted = 0;   // handle-wide default of p_searchDeleted (parameter "SearchDeleted"); per-call value: sptag_b200_search_ex
    // search parameters (reference names)
    int max_check = 8192, max_check_refine = 8192, initial_pivots = 50, other_pivots = 4, no_better_threshold = 3;
    // graph-update parameters (reference names, BKT/ParameterDefinitionList.h:28-31): AddIndex's refine budget, the
    // result count of DeleteIndex(vectors), RebuildNeighbors' factor
    int add_cef = 500, cef = 1000;
    float rng_factor = 1.0f;
    int open_iterators = 0;  // their per-query bitmaps are sized to n: mutations are refused while any is open
    DeviceBuffer d_mut, d_first;  // mutation scratch: ids / codes / counter, and the per-id first batch position
    // B200 tuning knobs
    int queries_per_sm = 0;  // 0 = auto
    int stage_rows = 0;      // 0 = auto
    int stages = 2;
    bool stages_set = false;  // B200.Stages was set explicitly
    // Small queue caches + a small ring: the kernel is latency-bound per warp, so resident queries per
    // SM matter more than on-chip queue capacity.  0 = auto.
    int h_ng = 0, h_spt = 0;
    int simd_width = 16;
    int slot_scheme = 0;          // 0 auto, 1 = 128-multiple stride + staggered odd slots, 2 = stride 64 mod 128
    int visited_log = -1;         // -1 auto (bitmap > 256 KB per slot), 0 clear per query, 1 log + selective clear
    int visited_log_entries = 0;  // 0 = auto
    // PQ / OPQ quantizer (null when q_type == 0)
    int q_type = 0, q_rtype = SPTAG_B200_VT_FLOAT, q_m = 0, q_ks = 0, q_dsub = 0;
    int q_adc = 0;  // IQuantizer::SetEnableADC (not serialized by the reference either)
    DeviceBuffer d_codebooks, d_rotation_t, d_rotation, d_sdc, d_raw;
    DeviceBuffer d_rec;  // refine on a quantized index: the batch's reconstructed rows
    // scratch
    // Everything a search launch writes besides its outputs.  Two sets: a launch normally takes set 0; when set 0 is
    // still busy with a launch from ANOTHER stream the new launch takes set 1 (allocated on first use), so two batches
    // can be in flight -- the second kernel's CTAs take over SM by SM as the first kernel's persistent warps run out of
    // queries, which hides the tail of a batch.
    struct Scratch {
        DeviceBuffer d_visited, d_ng_spill, d_spt_spill, d_counter, d_vlog, d_topk, d_codes, d_adc;
        bool visited_clean = false;   // the whole d_visited buffer is known to be zero
        cudaEvent_t ev_done = nullptr;  // recorded after every kernel that uses this set; the next launch on it waits
        cudaStream_t last_stream = nullptr;
        bool used = false;
        void release() {  // early free: set 1 did not fit in HBM and the launch falls back to set 0
            d_visited.release(); d_ng_spill.release(); d_spt_spill.release(); d_counter.release(); d_vlog.release();
            d_topk.release(); d_codes.release(); d_adc.release();
        }
    } scratch[2];
    DeviceBuffer d_ids, d_dists;                      // refine pass: per-batch result lists
    // Host-buffer entry points: two staging sets, each with its own stream, so that one caller's H2D / D2H overlaps
    // another caller's kernel (the kernels themselves share the per-slot scratch and are ordered by ev_done)
    struct Staging {
        std::mutex mu;
        cudaStream_t stream = nullptr;
        DeviceBuffer d_queries, d_ids, d_dists, d_stats, d_filter;
    } staging[2];
    std::atomic<unsigned> staging_rr{0};
    DeviceBuffer d_graph_new;                         // sptag_b200_refine_graph: the pass's output rows
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_aux = nullptr;
    double refine_search_ms = 0.0, refine_rebuild_ms = 0.0;  // device time of the last sptag_b200_refine_graph call
    bool timed = false;
    int num_sms = 0;
    size_t smem_optin = 0;
    std::mutex mu;
};

// One ResultIterator per query of a batch (VectorIndex::GetIterator, BKTIndex.cpp:650-657): the rented WorkSpace of
// each query lives in HBM for the iterator's lifetime.
struct sptag_b200_iterator {
    sptag_b200_index* h = nullptr;
    int nq = 0;
    // sampled at open, like the reference's WorkSpace::Initialize + Reset at RentWorkSpace (BKTIndex.cpp:686-696)
    int max_check = 0, ng_length = 0, ng_lastlevel = 0, spt_length = 0, spt_lastlevel = 0;
    size_t visited_words = 0, ng_entries = 0, spt_entries = 0;
    int topk_pad = 0;
    int search_deleted = 0;  // GetIterator(p_target, p_searchDeleted)
    int nearest_k = 0;       // > 0 once sptag_b200_iterator_next_from_nearest ran: the head QueryResult's size
    bool stepped = false;    // a Next of either kind has run
    DeviceBuffer d_queries, d_visited, d_ng, d_spt, d_state, d_topk, d_ids, d_dists, d_counts, d_relaxed;
};

namespace {

int heap_lastlevel(int size) {
    // Heap::Resize: lastlevel = int(pow(2.0, floor(log2((float)size))))  (Heap.h:24)
    return (int)std::pow(2.0, std::floor(std::log2((float)size)));
}

// The kernel instantiation for this index / parameter set (nullptr: unsupported m_Results capacity); the
// instantiations live in kern_*.cu (kernel_select.h)
SearchKernelFn pick_kernel(const sptag_b200_index* h, int mres_cap, int slots = 0) {
    const bool kdt = (h->algo == SPTAG_B200_ALGO_KDT);
    if (h->q_type != 0) return pick_pq_kernel(mres_cap);  // quantized: BKT + L2 only (PQQuantizer.h:130-136)
    const bool l2 = (h->metric == SPTAG_B200_METRIC_L2);
    if (h->value_type == SPTAG_B200_VT_INT8) return pick_int8_kernel(false, !l2, mres_cap, kdt);
    if (h->value_type == SPTAG_B200_VT_UINT8) return pick_int8_kernel(true, !l2, mres_cap, kdt);
    if (h->value_type == SPTAG_B200_VT_INT16) return pick_int16_kernel(!l2, mres_cap, kdt);
    const int kdim = (h->simd_width == 16) ? h->dim : 0;  // the 128- / 768-d specialisations are AVX-512 trees
    return l2 ? pick_float_kernel_l2(kdim, mres_cap, kdt, slots) : pick_float_kernel_cosine(kdim, mres_cap, kdt, slots);
}

// What one call may override (the reference passes these per call: p_searchDeleted of SearchIndex / GetIterator,
// maxCheck + filterFunc of SearchIndexWithFilter, MaxCheckForRefineGraph of RefineSearchIndex).  Nothing here is ever
// written into the handle, so concurrent callers cannot see each other's settings.
struct CallOpts {
    int max_check = 0;          // 0 = the index's MaxCheck
    int search_deleted = -1;    // -1 = the handle's "SearchDeleted" default, else 0 / 1
    const unsigned char* d_filter = nullptr;  // device byte map (0 = never added to the results) or nullptr
    size_t refine_query_stride = 0;  // refine flavour: bytes between queries (index rows: the padded row stride)
    // test the tombstone map even while the host's count is 0: DeleteIndex(vectors) tombstones on the device between two
    // of its searches (an all-zero map rejects nothing, so this equals the reference's Count() == 0 dispatch)
    bool tombstones_live = false;
};

// Slots of a result heap kept in HBM for k results: a power of two (the final sort is bitonic), at least 64
int topk_pad_for(int k) {
    int pad = 64;
    while (pad < k) pad <<= 1;
    return pad;
}

// One search-kernel launch: parameters, instantiation and geometry
struct SearchLaunch {
    SearchParams p;
    SearchKernelFn kern = nullptr;
    int grid = 0;
    int per_sm = 0;   // resident query slots per SM
    size_t smem = 0;  // dynamic shared memory per slot
};

// What the search kernels support for this handle and k.  The iterators refuse the same combinations.
int check_supported(const sptag_b200_index* h, int k) {
    if (h->algo != SPTAG_B200_ALGO_BKT && h->algo != SPTAG_B200_ALGO_KDT)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported index algorithm %d", h->algo);
    const bool pq = (h->q_type != 0);
    if (pq) {
        if (h->value_type != SPTAG_B200_VT_UINT8 || h->dim != h->q_m)
            return fail(SPTAG_B200_DIMENSION_MISMATCH, "quantizer has %d sub-vectors but the index rows are %d x type %d",
                        h->q_m, h->dim, h->value_type);
        if (h->algo != SPTAG_B200_ALGO_BKT || h->metric != SPTAG_B200_METRIC_L2)
            return fail(SPTAG_B200_LACK_OF_INPUTS, "quantized indexes are searchable as BKT + L2 only");
    } else if (h->value_type == SPTAG_B200_VT_INT16) {
        // int16: every rounding step of the AVX-512 variants is reproduced (no exact-integer argument needed)
    } else if (h->value_type != SPTAG_B200_VT_FLOAT) {
        // int8 / uint8: every partial sum must stay an exactly representable integer for the kernel's and the
        // reference's summation orders to be interchangeable in the scalar tails; true for the supported range
        const int maxterm = (h->value_type == SPTAG_B200_VT_INT8) ? (h->metric == SPTAG_B200_METRIC_L2 ? 254 * 254 : 127 * 127)
                                                                   : 255 * 255;
        if ((long long)h->dim * maxterm >= (1ll << 31))
            return fail(SPTAG_B200_LACK_OF_INPUTS, "dimension %d too large for the integer distance kernels", h->dim);
    }
    if (h->simd_width != 16 && h->simd_width != 8 && h->simd_width != 4)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "B200.SimdWidth %d: 16 (AVX-512), 8 (AVX / AVX2) or 4 (SSE)", h->simd_width);
    if (h->simd_width != 16 && (pq || h->value_type == SPTAG_B200_VT_INT16))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "B200.SimdWidth %d: the AVX / SSE summation trees are built for float, int8 and uint8 "
                                              "rows (int16 and the quantizer tables exist in the AVX-512 form only)", h->simd_width);
    if (k < 1 || k > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside the supported range [1, 2048]", k);
    return 0;
}

// SearchParams from the handle and the call's options, including the per-slot arena sizes; the shared-memory layout
// (lay_out) and the scratch pointers (bind_scratch) come later
void fill_params(const sptag_b200_index* h, int k, const CallOpts& opts, SearchParams& p) {
    const int eff_max_check = opts.max_check > 0 ? opts.max_check : h->max_check;
    const int eff_search_deleted = opts.search_deleted >= 0 ? opts.search_deleted : h->search_deleted;
    const bool pq = (h->q_type != 0);
    memset(&p, 0, sizeof(p));
    p.vectors = (const unsigned char*)h->d_vectors.ptr;
    p.row_stride_bytes = h->row_stride;
    p.row_bytes = (int)h->row_stride;
    p.n = h->n;
    p.dim = h->dim;
    p.graph = (const int*)h->d_graph.ptr;
    p.degree = h->degree;
    p.nodes = (const int*)h->d_nodes.ptr;
    p.tree_starts = (const int*)h->d_tree_starts.ptr;
    p.tree_num = h->tree_num;
    p.node_count = h->node_count;
    // flags += (m_deletedID.Count() == 0 || p_searchDeleted) << 2  (BKTIndex.cpp:473, KDTIndex.cpp:260)
    p.deleted = ((h->num_deleted > 0 || opts.tombstones_live) && !eff_search_deleted) ? (const signed char*)h->d_deleted.ptr
                                                                                       : nullptr;
    p.filter = opts.d_filter;
    p.k = k;
    p.id_offset = h->id_offset;
    p.max_check = eff_max_check;
    p.initial_pivots = h->initial_pivots;
    p.other_pivots = h->other_pivots;
    p.no_better_threshold = h->no_better_threshold;
    // a fresh thread's WorkSpace: Initialize(max(MaxCheck, MaxCheckForRefineGraph)) then
    // Reset(MaxCheck, K) (BKTIndex.cpp:600-605, WorkSpace.h:243-278)
    const int alloc_check = std::max(eff_max_check, h->max_check_refine);
    p.ng_length = alloc_check * 30;
    p.ng_lastlevel = heap_lastlevel(p.ng_length);
    p.spt_length = alloc_check * 10;
    p.spt_lastlevel = heap_lastlevel(p.spt_length);
    p.mres_cap = std::max(eff_max_check / 16, k);
    p.simd_width = h->simd_width;
    p.sdc = (const float*)h->d_sdc.ptr;
    p.pq_m = h->q_m;
    p.pq_ks = h->q_ks;
    p.pq_adc = (pq && h->q_adc) ? 1 : 0;
    p.pq_dsub = h->q_dsub;
    p.codebooks = (const float*)h->d_codebooks.ptr;

    // ---- per-slot arena sizes ----
    p.visited_words = round_up(((size_t)h->n + 1 + 31) / 32, 4);
    // (even entry counts keep every slot's arena 16-byte aligned for the paired child loads)
    p.ng_spill_entries = round_up((size_t)std::min<long long>((long long)p.ng_length, (long long)h->n + 2) + 2, 2);
    p.spt_spill_entries = round_up((size_t)std::min<long long>((long long)p.spt_length, (long long)h->node_count + 2) + 2, 2);
    const bool use_log = h->visited_log < 0 ? (p.visited_words * 4 > 256 * 1024) : (h->visited_log != 0);
    if (use_log) {
        const size_t entries = h->visited_log_entries > 0 ? (size_t)h->visited_log_entries
                                                          : (size_t)std::max(65536, 8 * alloc_check);
        p.vlog_entries = std::min(entries, (size_t)h->n + 2);
    }
    if (k > 32) p.topk_pad = topk_pad_for(k);  // result heap of the reference in HBM, one arena per slot
}

// Shared-memory layout of a query slot, kernel instantiation, residency and grid.  Unless the queue heads are sized
// explicitly, the shared memory a slot has spare at that residency goes to them, and the layout is made once more.
int lay_out(const sptag_b200_index* h, int nq, SearchLaunch& L) {
    SearchParams& p = L.p;
    const bool pq = (h->q_type != 0);
    int stage_rows = h->stage_rows;
    if (stage_rows <= 0) {
        stage_rows = (int)(5120 / round_up(h->row_stride + 64, 128));  // 768-d: 2 rows, 128-d: 8 rows (sweeps)
        stage_rows = std::max(2, std::min(16, stage_rows));
    }
    stage_rows &= ~1;
    if (stage_rows < 2) stage_rows = 2;
    if (stage_rows > 32) stage_rows = 32;
    int stages = std::max(1, std::min(8, h->stages));
    while (stages & (stages - 1)) stages &= stages - 1;  // power of two (the kernel masks instead of dividing)
    // ring slot stride: the two rows of a pair must start 64 B apart modulo 128 (disjoint banks for the two
    // half-warps); either a 128-multiple stride with odd slots staggered, or a stride that is 64 mod 128
    {
        const size_t a = round_up(h->row_stride + 64, 128), b = round_up(h->row_stride, 128) + 64;
        p.slot_stagger = (a <= b) ? 1 : 0;
        if (h->slot_scheme == 1) p.slot_stagger = 1;
        if (h->slot_scheme == 2) p.slot_stagger = 0;
        p.slot_stride = (int)(p.slot_stagger ? a : b);
    }
    // 512-byte float rows run the fixed-shape fast path (search_kernels.cuh kFast): 2 stages x 8 rows, slots 576 B apart;
    // must mirror WarpSearch::kFast
    const bool fast128 = !pq && h->value_type == SPTAG_B200_VT_FLOAT && h->dim == 128 && h->simd_width == 16;
    // ... with register-capped kernel variants for more than 16 query slots per SM (B200.QueriesPerSM); those run a
    // one-stage ring (B200.Stages = 1 selects it at any residency) so that the slot's shared memory still fits
    // Default residency for 512-byte rows: all warps start together and a query costs about the same for every warp,
    // so a batch runs in ceil(nq / slots) near-lockstep rounds and a mostly empty last round is lost time.  Pick the slot
    // count in [14, 20] whose last round is fullest, weighted by the per-slot-count throughput (saturates at 17+).
    int want_slots = fast128 ? h->queries_per_sm : 0;
    if (fast128 && want_slots <= 0) {
        static const double weight[7] = {0.88, 0.92, 0.97, 1.0, 1.0, 1.0, 1.0};  // 14 .. 20 slots
        double best = -1.0;
        for (int s = 14; s <= 20; ++s) {
            const long long slots = (long long)h->num_sms * s;
            const long long rounds = ((long long)nq + slots - 1) / slots;
            const double score = weight[s - 14] * (double)nq / (double)(rounds * slots);
            if (score > best + 1e-9) {
                best = score;
                want_slots = s;
            }
        }
        if ((long long)nq <= (long long)h->num_sms * 14) want_slots = 14;  // one round: fewer slots, larger queue heads
    }
    if (fast128) {
        stage_rows = 8;
        // one 8-row stage unless B200.Stages = 2 is asked for at <= 16 slots: the second stage's 4.6 KB serve better as
        // queue heads
        stages = (h->stages_set && h->stages == 2 && want_slots <= 16) ? 2 : 1;
        p.slot_stride = 128 * 4 + 64;
        p.slot_stagger = 0;
    }
    if (pq) {  // every candidate row of a step in one TMA batch; rows are M bytes
        stage_rows = 32;
        stages = 1;
        p.slot_stride = (int)h->row_stride + ((h->row_stride % 128 == 0) ? 16 : 0);
        p.slot_stagger = 0;
    }
    p.stage_rows = stage_rows;
    p.stages = stages;
    const bool big_rows = h->row_stride >= 2048;
    int extra_ng = 0, extra_spt = 0;
    for (int pass = 0;; ++pass) {
        // odd: a node's two children (indices 2p, 2p + 1) are fetched with one 128-bit load, so a pair must not straddle
        // the shared-memory head and the HBM arena (heap_pop)
        p.h_ng = ((h->h_ng > 0 ? h->h_ng : (big_rows ? 64 : 128)) + extra_ng) | 1;
        p.h_spt = ((h->h_spt > 0 ? h->h_spt : (big_rows ? 32 : 64)) + extra_spt) | 1;
        size_t off = (size_t)stage_rows * stages * p.slot_stride;
        p.off_ng = (int)off;
        off += round_up((size_t)(p.h_ng + 1) * 8, 16);
        p.off_spt = (int)off;
        off += round_up((size_t)(p.h_spt + 1) * 8, 16);
        p.off_cand = (int)off;
        off += 256;
        p.off_bar = (int)off;
        off += round_up((size_t)stages * 8, 16);
        p.off_query = (int)off;
        const bool query_in_regs_only = !pq && h->value_type == SPTAG_B200_VT_FLOAT && h->algo == SPTAG_B200_ALGO_BKT &&
                                        h->dim == 768 && h->simd_width == 16;  // must mirror kRegsOnly in search_kernel
        off += query_in_regs_only ? 16 : round_up((size_t)h->dim * 4 + 16, 16);  // float query, or M row offsets for PQ
        L.smem = round_up(off, 128);
        if (L.smem > h->smem_optin)
            return fail(SPTAG_B200_MEMORY_OVERFLOW, "shared memory per query slot %zu exceeds %zu", L.smem, h->smem_optin);

        L.kern = pick_kernel(h, p.mres_cap, want_slots);
        if (!L.kern)
            return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, K) = %d exceeds what this index type supports (2048; quantized: 1024)", p.mres_cap);
        CUDA_OK(cudaFuncSetAttribute((const void*)L.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
        // resident single-warp CTAs per SM allowed by registers + shared memory for this instantiation
        int fit = 0;
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, (const void*)L.kern, 32, L.smem));
        if (fit < 1) return fail(SPTAG_B200_MEMORY_OVERFLOW, "search kernel does not fit on an SM (smem %zu)", L.smem);
        int per_sm = h->queries_per_sm;
        if (per_sm <= 0) per_sm = fit;  // the kernel is latency-bound per warp: fill the SM
        if (h->queries_per_sm <= 0 && big_rows) per_sm = std::min(per_sm, 14);  // 3 KB rows: 14 beats 15 (HBM-bound)
        // 512 B rows: 14 slots leave 2 KB more shared memory per queue head than 16 and shorten the tail of a 10k-query batch
        if (h->queries_per_sm <= 0 && fast128) per_sm = std::min(per_sm, want_slots);
        L.per_sm = std::max(1, std::min(per_sm, fit));
        if (pass > 0 || h->h_ng > 0 || h->h_spt > 0) break;
        // Spare shared memory of a slot (at this residency) goes to the queue heads: 3/4 NGQueue, 1/4 SPTQueue
        const size_t per_slot = (size_t)(227 * 1024) / L.per_sm - 1024;
        if (per_slot <= L.smem + 512) break;
        const size_t spare_entries = (per_slot - L.smem) / 8;
        extra_ng = (int)std::min<size_t>(spare_entries * 3 / 4, 4096);
        extra_spt = (int)std::min<size_t>(spare_entries / 4, 2048);
        extra_ng &= ~1;
        extra_spt &= ~1;
        if (extra_ng + extra_spt < 64) break;
    }
    L.grid = std::max(1, std::min(nq, h->num_sms * L.per_sm));
    return 0;
}

// Everything of a search launch but its scratch: the refusals, SearchParams, layout, kernel and grid
int plan_search(const sptag_b200_index* h, int k, int nq, const CallOpts& opts, SearchLaunch& L) {
    if (int rc = check_supported(h, k)) return rc;
    fill_params(h, k, opts, L.p);
    return lay_out(h, nq, L);
}

// Point the launch at scratch set `set`, allocated for every resident slot (grown, never shrunk).  Caller holds h->mu.
int bind_scratch(sptag_b200_index* h, SearchLaunch& L, int set) {
    sptag_b200_index::Scratch& sc = h->scratch[set];
    SearchParams& p = L.p;
    const size_t alloc_slots = (size_t)h->num_sms * L.per_sm;
    {
        const size_t before = sc.d_visited.bytes;
        if (int rc = sc.d_visited.ensure(alloc_slots * p.visited_words * 4)) return rc;
        if (sc.d_visited.bytes != before) sc.visited_clean = false;
    }
    if (p.vlog_entries) {
        if (int rc = sc.d_vlog.ensure(alloc_slots * p.vlog_entries * 4)) return rc;
        p.vlog = (unsigned int*)sc.d_vlog.ptr;
        if (!sc.visited_clean) {  // log mode relies on every query leaving its bitmap zeroed
            CUDA_OK(cudaMemset(sc.d_visited.ptr, 0, sc.d_visited.bytes));
            sc.visited_clean = true;
        }
    } else {
        sc.visited_clean = false;  // clear-per-query mode leaves the last query's bits behind
    }
    if (int rc = sc.d_ng_spill.ensure(alloc_slots * p.ng_spill_entries * 8)) return rc;
    if (int rc = sc.d_spt_spill.ensure(alloc_slots * p.spt_spill_entries * 8)) return rc;
    if (int rc = sc.d_counter.ensure(256)) return rc;
    if (p.pq_adc) {  // one M x Ks fp32 table per resident query
        if (int rc = sc.d_adc.ensure(alloc_slots * (size_t)h->q_m * h->q_ks * 4)) return rc;
        p.adc_tables = (float*)sc.d_adc.ptr;
    }
    if (p.topk_pad) {
        if (int rc = sc.d_topk.ensure(alloc_slots * (size_t)p.topk_pad * 8)) return rc;
        p.topk = (int2*)sc.d_topk.ptr;
    }
    p.visited = (unsigned int*)sc.d_visited.ptr;
    p.ng_spill = (int2*)sc.d_ng_spill.ptr;
    p.spt_spill = (int2*)sc.d_spt_spill.ptr;
    p.work_counter = (unsigned int*)sc.d_counter.ptr;
    return 0;
}

size_t query_bytes(const sptag_b200_index* h) {
    if (h->q_type != 0) return (size_t)h->q_m * h->q_dsub * value_size(h->q_rtype);
    return (size_t)h->dim * value_size(h->value_type);
}

int quantize_device(sptag_b200_index* h, const void* d_raw, int n, unsigned char* d_codes, cudaStream_t stream,
                    float* d_rotated = nullptr) {
    const int dim = h->q_m * h->q_dsub;
    const size_t smem = (size_t)dim * 2 * sizeof(float);
    if (smem > 48 * 1024)
        CUDA_OK(cudaFuncSetAttribute(pq_quantize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pq_quantize_kernel<<<n, 128, smem, stream>>>((const unsigned char*)d_raw, h->q_rtype, (long long)query_bytes(h), n,
                                                  (const float*)h->d_codebooks.ptr,
                                                  h->q_type == 2 ? (const float*)h->d_rotation_t.ptr : nullptr, h->q_m,
                                                  h->q_ks, h->q_dsub, d_codes, d_rotated);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return 0;
}

// Every kernel that touches the handle's shared scratch (visited bitmaps, queue arenas, work counter, quantized-query
// buffer) is ordered after the previous one, whatever stream it was launched on: the caller's stream waits on ev_done
// before the launch sequence and records it afterwards.  Caller holds h->mu.
int scratch_acquire(sptag_b200_index* h, cudaStream_t stream, int set = 0) {
    if (h->scratch[set].used) CUDA_OK(cudaStreamWaitEvent(stream, h->scratch[set].ev_done, 0));
    return 0;
}
int scratch_release(sptag_b200_index* h, cudaStream_t stream, int set = 0) {
    CUDA_OK(cudaEventRecord(h->scratch[set].ev_done, stream));
    h->scratch[set].used = true;
    h->scratch[set].last_stream = stream;
    return 0;
}
// Set 0 unless it is still busy with a launch from another stream (then set 1, if that one is free or also busy on
// this very stream).  Single-stream callers therefore never allocate the second set.
int pick_scratch(sptag_b200_index* h, cudaStream_t stream) {
    sptag_b200_index::Scratch& a = h->scratch[0];
    if (!a.used || a.last_stream == stream || cudaEventQuery(a.ev_done) == cudaSuccess) return 0;
    sptag_b200_index::Scratch& b = h->scratch[1];
    if (!b.used || b.last_stream == stream || cudaEventQuery(b.ev_done) == cudaSuccess) return 1;
    return 0;  // both busy elsewhere: queue behind set 0
}

// refine = true: the RefineSearchIndex flavour (BKTIndex.cpp:698-711) -- queries are base rows of the index itself
// (stride = the padded row stride), duplicate groups are not expanded, ids come back local (no shard offset); the
// caller passes MaxCheckForRefineGraph as opts.max_check.  Caller holds h->mu.
int search_device_impl(sptag_b200_index* h, const void* d_queries, int nq, int k, int* d_ids, float* d_dists,
                       int* d_stats, cudaStream_t stream, bool refine = false, const CallOpts& opts = CallOpts()) {
    if (nq <= 0) return SPTAG_B200_SUCCESS;
    int set = refine ? 0 : pick_scratch(h, stream);
    SearchLaunch L;
    if (int rc = plan_search(h, k, nq, opts, L)) return rc;
    if (int rc = bind_scratch(h, L, set)) {
        if (set == 0) return rc;
        // the second scratch set did not fit in HBM: run behind the first one instead
        h->scratch[1].release();
        cudaGetLastError();
        set = 0;
        if (int rc0 = bind_scratch(h, L, set)) return rc0;
    }
    SearchParams& p = L.p;
    sptag_b200_index::Scratch& sc = h->scratch[set];
    if (int rc = scratch_acquire(h, stream, set)) return rc;
    p.queries = (const unsigned char*)d_queries;
    p.query_stride_bytes = (size_t)h->dim * value_size(h->value_type);
    if (h->q_type != 0) {
        // QueryResultSet::SetTarget -> IQuantizer::QuantizeVector (QueryResultSet.h:46-60): raw -> M code bytes
        if (h->q_adc) {  // ADC: the kernel needs the rotated float vector, not codes
            const size_t dimq = (size_t)h->q_m * h->q_dsub;
            if (int rc = sc.d_codes.ensure((size_t)nq * dimq * 4)) return rc;
            if (int rc = quantize_device(h, d_queries, nq, nullptr, stream, (float*)sc.d_codes.ptr)) return rc;
            p.queries = (const unsigned char*)sc.d_codes.ptr;
            p.query_stride_bytes = dimq * 4;
        } else {
            if (int rc = sc.d_codes.ensure((size_t)nq * h->q_m)) return rc;
            if (int rc = quantize_device(h, d_queries, nq, (unsigned char*)sc.d_codes.ptr, stream)) return rc;
            p.queries = (const unsigned char*)sc.d_codes.ptr;
            p.query_stride_bytes = (size_t)h->q_m;
        }
    }
    if (refine) {
        if (opts.refine_query_stride) p.query_stride_bytes = opts.refine_query_stride;
        p.never_dup = 1;
        p.id_offset = 0;
    }
    p.nq = nq;
    p.out_ids = d_ids;
    p.out_dists = d_dists;
    p.out_stats = d_stats;
    CUDA_OK(cudaMemsetAsync(p.work_counter, 0, 4, stream));
    CUDA_OK(cudaEventRecord(h->ev_start, stream));
    L.kern<<<L.grid, 32, L.smem, stream>>>(p);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaEventRecord(h->ev_stop, stream));
    h->timed = true;
    return scratch_release(h, stream, set);
}

// An iterator step's search set-up: the search kernel's refusals and launch shape for k results over the iterator's
// queries, with the budget and tombstone choice the iterator was opened with.  Caller holds h->mu.
int plan_iterator_step(const sptag_b200_iterator* it, int k, SearchLaunch& L) {
    CallOpts iopts;
    iopts.max_check = it->max_check;  // the rented WorkSpace keeps the budget it was reset with
    iopts.search_deleted = it->search_deleted;
    return plan_search(it->h, k, it->nq, iopts, L);
}

// Run one iterator step planned by plan_iterator_step.  The iterator's queue lengths and per-query arenas replace the
// per-slot scratch of a search; of scratch set 0 only the work counter is used, with the same ordering as a search.
// The grid stays the search kernel's.  launch(p, grid, smem, stream) enqueues the iterate or nearest-first kernel;
// `what` names k in the refusal.  Caller holds h->mu.
template <typename LaunchFn>
int run_iterator_step(sptag_b200_iterator* it, int k, const char* what, SearchLaunch& L, int32_t* out_ids,
                      float* out_dists, int32_t* out_counts, uint8_t* out_relaxed_mono, LaunchFn&& launch) {
    sptag_b200_index* h = it->h;
    if (it->topk_pad == 0) {  // the first Next creates the QueryResult: its size bounds every later batch
        it->topk_pad = topk_pad_for(k);
        if (int rc = it->d_topk.ensure((size_t)it->nq * it->topk_pad * 8)) return rc;
    } else if (k > it->topk_pad) {
        // e.g. Next(batch) after SearchIndexIterativeFromNeareast(k) reset the slot cap: the per-query result arena
        // was sized by the first call
        return fail(SPTAG_B200_LACK_OF_INPUTS, "%s = %d exceeds the iterator's result arena (%d, sized by its first call)",
                    what, k, it->topk_pad);
    }
    const size_t rn = (size_t)it->nq * k;
    if (int rc = it->d_ids.ensure(rn * 4)) return rc;
    if (int rc = it->d_dists.ensure(rn * 4)) return rc;
    if (int rc = h->scratch[0].d_counter.ensure(256)) return rc;
    SearchParams& p = L.p;
    // generic-DIM kernel: the query is read from shared memory (lay_out sized the slot for the static variants)
    p.off_query = (int)round_up((size_t)p.off_bar + round_up((size_t)p.stages * 8, 16), 16);
    const size_t smem = round_up((size_t)p.off_query + round_up((size_t)h->dim * 4 + 16, 16), 128);
    p.queries = (const unsigned char*)it->d_queries.ptr;
    p.query_stride_bytes = query_bytes(h);
    p.nq = it->nq;
    p.max_check = it->max_check;
    p.ng_length = it->ng_length;
    p.ng_lastlevel = it->ng_lastlevel;
    p.spt_length = it->spt_length;
    p.spt_lastlevel = it->spt_lastlevel;
    p.visited = (unsigned int*)it->d_visited.ptr;
    p.visited_words = it->visited_words;
    p.ng_spill = (int2*)it->d_ng.ptr;
    p.ng_spill_entries = it->ng_entries;
    p.spt_spill = (int2*)it->d_spt.ptr;
    p.spt_spill_entries = it->spt_entries;
    p.topk = (int2*)it->d_topk.ptr;
    p.topk_pad = it->topk_pad;
    p.out_ids = (int*)it->d_ids.ptr;
    p.out_dists = (float*)it->d_dists.ptr;
    p.work_counter = (unsigned int*)h->scratch[0].d_counter.ptr;
    if (smem > h->smem_optin) return fail(SPTAG_B200_MEMORY_OVERFLOW, "shared memory per query slot %zu exceeds %zu", smem, h->smem_optin);
    cudaStream_t stream = nullptr;
    if (int rc = scratch_acquire(h, stream)) return rc;
    CUDA_OK(cudaMemsetAsync(p.work_counter, 0, 4, stream));
    CUDA_OK(cudaEventRecord(h->ev_start, stream));
    if (int rc = launch(p, L.grid, smem, stream)) return rc;
    g_launches++;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaEventRecord(h->ev_stop, stream));
    h->timed = true;
    if (int rc = scratch_release(h, stream)) return rc;
    CUDA_OK(cudaMemcpyAsync(out_ids, it->d_ids.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_dists, it->d_dists.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    if (out_counts) CUDA_OK(cudaMemcpyAsync(out_counts, it->d_counts.ptr, (size_t)it->nq * 4, cudaMemcpyDeviceToHost, stream));
    if (out_relaxed_mono)
        CUDA_OK(cudaMemcpyAsync(out_relaxed_mono, it->d_relaxed.ptr, (size_t)it->nq, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    it->stepped = true;
    return SPTAG_B200_SUCCESS;
}

// Element type of the index rows as the aux kernels' ELEM parameter takes it: 0 float, 1 int8, 2 uint8, 3 int16
template <typename T, int EL>
struct Elem : std::integral_constant<int, EL> {
    typedef T type;
};

// Calls f(Elem<T, EL>()) for the index's value type
template <typename F>
void with_elem(const sptag_b200_index* h, F&& f) {
    switch (h->value_type) {
    case SPTAG_B200_VT_INT8: f(Elem<int8_t, 1>()); break;
    case SPTAG_B200_VT_UINT8: f(Elem<uint8_t, 2>()); break;
    case SPTAG_B200_VT_INT16: f(Elem<int16_t, 3>()); break;
    default: f(Elem<float, 0>()); break;
    }
}

// Calls f(cos, el) with the index's metric as a compile-time bool (true for every metric but L2) and its Elem; the
// caller launches the <cos, el> instantiations of its kernels inside f
template <typename F>
void with_metric_elem(const sptag_b200_index* h, F&& f) {
    with_elem(h, [&](auto el) {
        if (h->metric == SPTAG_B200_METRIC_L2)
            f(std::false_type(), el);
        else
            f(std::true_type(), el);
    });
}

// Make d_graph_new, rows of `degree` entries, the index's graph.  BuildGraph re-attaches the duplicate-group
// back-pointers after its refine passes (NeighborhoodGraph.h:395-401); the new rows may be wider or narrower than the
// current ones (RefineGraph's schedule, :460-492).  Caller holds h->mu.
int install_graph(sptag_b200_index* h, int degree, cudaStream_t stream) {
    const long long n = h->n;
    carry_backpointers_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const int*)h->d_graph.ptr,
                                                                               (int*)h->d_graph_new.ptr, h->n, h->degree,
                                                                               degree);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaStreamSynchronize(stream));
    std::swap(h->d_graph, h->d_graph_new);
    h->degree = degree;
    return 0;
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        int cur = -1;
        cudaGetDevice(&cur);
        if (prev >= 0 && cur != prev) cudaSetDevice(prev);
    }
};

bool read_file(const std::string& path, std::vector<char>& out) {
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) return false;
    std::streamsize sz = f.tellg();
    f.seekg(0);
    out.resize((size_t)sz);
    return (bool)f.read(out.data(), sz);
}

// Shape of an index and where its arrays come from: host arrays (sptag_b200_create) or the reference's files
// streamed through pinned chunks (sptag_b200_load).  Exactly one of (ptr, file) is set per array.
struct ArraySource {
    const void* ptr = nullptr;
    FILE* file = nullptr;
    long long offset = 0;  // body offset in the file
};

// Chunked upload: rows of `row_bytes` from `src` to a device array with `dst_stride` bytes between rows.  Files are
// read into two pinned buffers alternately, so the read of chunk i+1 overlaps the H2D copy of chunk i and no
// full-file host copy ever exists (f1: the 10 GB codes / 12.8 GB graph of config C4 used to sit twice in host memory).
int upload_rows(const ArraySource& src, void* dst, size_t rows, size_t row_bytes, size_t dst_stride, cudaStream_t stream) {
    if (rows == 0 || row_bytes == 0) return 0;
    if (src.ptr != nullptr) {
        if (dst_stride == row_bytes)
            CUDA_OK(cudaMemcpyAsync(dst, src.ptr, rows * row_bytes, cudaMemcpyHostToDevice, stream));
        else
            CUDA_OK(cudaMemcpy2DAsync(dst, dst_stride, src.ptr, row_bytes, row_bytes, rows, cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        return 0;
    }
    const size_t chunk_bytes = (size_t)32 << 20;
    const size_t rows_per_chunk = std::max<size_t>(1, chunk_bytes / row_bytes);
    void* pinned[2] = {nullptr, nullptr};
    cudaEvent_t freed[2] = {nullptr, nullptr};
    int rc = 0;
    for (int i = 0; i < 2 && rc == 0; ++i) {
        if (cudaMallocHost(&pinned[i], rows_per_chunk * row_bytes) != cudaSuccess ||
            cudaEventCreateWithFlags(&freed[i], cudaEventDisableTiming) != cudaSuccess)
            rc = fail(SPTAG_B200_MEMORY_OVERFLOW, "pinned staging buffer (%zu bytes) failed", rows_per_chunk * row_bytes);
    }
    if (rc == 0 && fseeko(src.file, (off_t)src.offset, SEEK_SET) != 0) rc = fail(SPTAG_B200_FAIL, "seek failed");
    size_t done = 0;
    for (int c = 0; rc == 0 && done < rows; ++c) {
        const int b = c & 1;
        const size_t nr = std::min(rows_per_chunk, rows - done);
        if (c >= 2 && cudaEventSynchronize(freed[b]) != cudaSuccess) rc = fail(SPTAG_B200_FAIL, "upload failed");
        if (rc == 0 && fread(pinned[b], row_bytes, nr, src.file) != nr) rc = fail(SPTAG_B200_FAIL, "file truncated");
        if (rc) break;
        unsigned char* d = (unsigned char*)dst + done * dst_stride;
        cudaError_t e = (dst_stride == row_bytes)
                            ? cudaMemcpyAsync(d, pinned[b], nr * row_bytes, cudaMemcpyHostToDevice, stream)
                            : cudaMemcpy2DAsync(d, dst_stride, pinned[b], row_bytes, row_bytes, nr, cudaMemcpyHostToDevice, stream);
        if (e == cudaSuccess) e = cudaEventRecord(freed[b], stream);
        if (e != cudaSuccess) rc = fail(SPTAG_B200_FAIL, "upload failed: %s", cudaGetErrorString(e));
        done += nr;
    }
    if (cudaStreamSynchronize(stream) != cudaSuccess && rc == 0) rc = fail(SPTAG_B200_FAIL, "upload failed");
    for (int i = 0; i < 2; ++i) {
        if (pinned[i]) cudaFreeHost(pinned[i]);
        if (freed[i]) cudaEventDestroy(freed[i]);
    }
    return rc;
}

// Range checks a kernel relies on: graph ids in [-1, n) (last slot: a duplicate back-pointer -2-node), tree starts and
// BKT child ranges inside the node array.  Runs on the device copy, so it also covers streamed files.
__global__ void validate_graph_kernel(const int* __restrict__ graph, long long entries, int degree, int n, int node_count,
                                      int* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= entries) return;
    const int v = graph[i];
    const bool last = (int)(i % degree) == degree - 1;
    bool ok = (v >= -1 && v < n);
    if (!ok && last && v < -1) ok = (-2 - v) < node_count;
    if (!ok) atomicAdd(bad, 1);
}
__global__ void validate_bkt_kernel(const int* __restrict__ nodes, int node_count, int n, int* __restrict__ bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= node_count) return;
    const int c = nodes[3 * i], cs = nodes[3 * i + 1], ce = nodes[3 * i + 2];
    bool ok = (c >= -1 && c <= n);
    if (cs >= 0) ok = ok && (cs <= ce && ce <= node_count);
    else if (cs < -1) ok = ok && (-cs <= node_count && ce <= node_count);  // duplicate-group head: members at [-cs, ce)
    if (!ok) atomicAdd(bad, 1);
}
__global__ void validate_kdt_kernel(const int4* __restrict__ nodes, int node_count, int n, int* __restrict__ bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= node_count) return;
    const int4 t = nodes[i];
    // children: node index, or -(vector id)-1 (KDTree.h:283,293)
    const bool ok = (t.x < node_count && t.y < node_count && -t.x - 1 <= n && -t.y - 1 <= n);
    if (!ok) atomicAdd(bad, 1);
}

struct IndexShape {
    int device = -1, algo = 0, value_type = 0, metric = 0, n = 0, dim = 0, degree = 0, tree_num = 0, node_count = 0,
        num_deleted = 0, id_offset = 0;
};

int build_handle(const IndexShape& sh, const ArraySource& vectors, const ArraySource& graph, const int32_t* tree_starts,
                 const ArraySource& nodes, const ArraySource& deleted, sptag_b200_handle* out) {
    *out = nullptr;
    if (sh.n <= 0) return fail(SPTAG_B200_EMPTY_INDEX, "empty index");
    if (sh.dim <= 0 || sh.degree <= 0 || sh.tree_num <= 0 || sh.node_count <= 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "bad index shape");
    const size_t vs = value_size(sh.value_type);
    if (vs == 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "bad value type %d", sh.value_type);
    if (sh.algo != SPTAG_B200_ALGO_BKT && sh.algo != SPTAG_B200_ALGO_KDT)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported index algorithm %d", sh.algo);
    for (int t = 0; t < sh.tree_num; ++t)
        if (tree_starts[t] < 0 || tree_starts[t] >= sh.node_count)
            return fail(SPTAG_B200_FAIL, "tree start %d = %d outside the %d tree nodes", t, tree_starts[t], sh.node_count);

    int device = sh.device;
    if (device < 0) CUDA_OK(cudaGetDevice(&device));
    DeviceGuard guard(device);
    CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)  // sm_90a code loads on compute capability 9.0 only
        return fail(SPTAG_B200_FAIL, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                    prop.major, prop.minor);

    auto* h = new sptag_b200_index();
    h->device = device;
    h->num_sms = prop.multiProcessorCount;
    h->smem_optin = prop.sharedMemPerBlockOptin;
    h->algo = sh.algo;
    h->value_type = sh.value_type;
    h->metric = sh.metric;
    h->n = sh.n;
    h->dim = sh.dim;
    h->degree = sh.degree;
    h->tree_num = sh.tree_num;
    h->node_count = sh.node_count;
    h->num_deleted = (deleted.ptr || deleted.file) ? sh.num_deleted : 0;
    h->id_offset = sh.id_offset;
    const size_t row_bytes = (size_t)h->dim * vs;
    h->row_stride = round_up(row_bytes, 16);  // TMA bulk copies need 16-byte aligned rows and sizes

    auto destroy_on_fail = [&](int rc) {
        sptag_b200_destroy(h);
        return rc;
    };
    if (cudaEventCreate(&h->ev_start) != cudaSuccess || cudaEventCreate(&h->ev_stop) != cudaSuccess ||
        cudaEventCreate(&h->ev_aux) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->scratch[0].ev_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->scratch[1].ev_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreate(&h->staging[0].stream) != cudaSuccess || cudaStreamCreate(&h->staging[1].stream) != cudaSuccess)
        return destroy_on_fail(fail(SPTAG_B200_FAIL, "cudaEventCreate / cudaStreamCreate failed"));
    cudaStream_t up = h->staging[0].stream;
    // one spare row so a 16-byte padded read of the last row stays in bounds
    if (int rc = h->d_vectors.ensure(((size_t)h->n + 1) * h->row_stride)) return destroy_on_fail(rc);
    if (h->row_stride != row_bytes) cudaMemsetAsync(h->d_vectors.ptr, 0, ((size_t)h->n + 1) * h->row_stride, up);
    if (int rc = upload_rows(vectors, h->d_vectors.ptr, (size_t)h->n, row_bytes, h->row_stride, up)) return destroy_on_fail(rc);
    const size_t graph_row = (size_t)h->degree * 4;
    if (int rc = h->d_graph.ensure((size_t)h->n * graph_row)) return destroy_on_fail(rc);
    if (int rc = upload_rows(graph, h->d_graph.ptr, (size_t)h->n, graph_row, graph_row, up)) return destroy_on_fail(rc);
    const size_t node_sz = (h->algo == SPTAG_B200_ALGO_BKT) ? 12 : 16;
    const size_t node_bytes = (size_t)h->node_count * node_sz;
    // BKT: one extra sentinel node (the reference's LoadTrees appends (-1,-1,-1), BKTree.h:662)
    if (int rc = h->d_nodes.ensure(node_bytes + 16)) return destroy_on_fail(rc);
    cudaMemsetAsync(h->d_nodes.ptr, 0xff, node_bytes + 16, up);
    if (int rc = upload_rows(nodes, h->d_nodes.ptr, (size_t)h->node_count, node_sz, node_sz, up)) return destroy_on_fail(rc);
    if (int rc = h->d_tree_starts.ensure((size_t)h->tree_num * 4)) return destroy_on_fail(rc);
    cudaMemcpy(h->d_tree_starts.ptr, tree_starts, (size_t)h->tree_num * 4, cudaMemcpyHostToDevice);
    if (h->num_deleted > 0) {
        if (int rc = h->d_deleted.ensure((size_t)h->n)) return destroy_on_fail(rc);
        if (int rc = upload_rows(deleted, h->d_deleted.ptr, 1, (size_t)h->n, (size_t)h->n, up)) return destroy_on_fail(rc);
    }
    // ids the kernels index with must be in range: a corrupt file fails here, not as a stray device read later
    {
        if (int rc = h->scratch[0].d_counter.ensure(256)) return destroy_on_fail(rc);
        int* bad = (int*)h->scratch[0].d_counter.ptr + 8;
        cudaMemsetAsync(bad, 0, 8, up);
        const long long entries = (long long)h->n * h->degree;
        validate_graph_kernel<<<(unsigned)((entries + 255) / 256), 256, 0, up>>>((const int*)h->d_graph.ptr, entries, h->degree,
                                                                                 h->n, h->node_count, bad);
        if (h->algo == SPTAG_B200_ALGO_BKT)
            validate_bkt_kernel<<<(h->node_count + 255) / 256, 256, 0, up>>>((const int*)h->d_nodes.ptr, h->node_count, h->n, bad + 1);
        else
            validate_kdt_kernel<<<(h->node_count + 255) / 256, 256, 0, up>>>((const int4*)h->d_nodes.ptr, h->node_count, h->n, bad + 1);
        g_launches += 2;
        int hb[2] = {0, 0};
        if (cudaMemcpyAsync(hb, bad, 8, cudaMemcpyDeviceToHost, up) != cudaSuccess || cudaStreamSynchronize(up) != cudaSuccess)
            return destroy_on_fail(fail(SPTAG_B200_FAIL, "index upload failed: %s", cudaGetErrorString(cudaGetLastError())));
        if (hb[0] || hb[1])
            return destroy_on_fail(fail(SPTAG_B200_FAIL, "index is corrupt: %d graph entries and %d tree nodes out of range", hb[0], hb[1]));
    }
    if (cudaDeviceSynchronize() != cudaSuccess || cudaGetLastError() != cudaSuccess)
        return destroy_on_fail(fail(SPTAG_B200_FAIL, "index upload failed"));
    *out = h;
    return SPTAG_B200_SUCCESS;
}

}  // namespace

extern "C" {

const char* sptag_b200_last_error(void) { return g_last_error.c_str(); }

int64_t sptag_b200_launch_count(void) { return (int64_t)g_launches.load(); }

int sptag_b200_create(const sptag_b200_index_desc* desc, sptag_b200_handle* out) {
    if (!desc || !out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null descriptor");
    *out = nullptr;
    if (desc->struct_size != (int32_t)sizeof(sptag_b200_index_desc))
        return fail(SPTAG_B200_FAIL, "descriptor size mismatch: %d vs %zu", desc->struct_size,
                    sizeof(sptag_b200_index_desc));
    if (desc->num_vectors <= 0 || !desc->vectors || !desc->graph || !desc->tree_nodes || !desc->tree_starts)
        return fail(SPTAG_B200_EMPTY_INDEX, "empty index");
    IndexShape sh;
    sh.device = desc->device;
    sh.algo = desc->algo;
    sh.value_type = desc->value_type;
    sh.metric = desc->metric;
    sh.n = desc->num_vectors;
    sh.dim = desc->dim;
    sh.degree = desc->graph_degree;
    sh.tree_num = desc->tree_num;
    sh.node_count = desc->node_count;
    sh.num_deleted = desc->deleted ? desc->num_deleted : 0;
    sh.id_offset = desc->id_offset;
    ArraySource v, g, t, d;
    v.ptr = desc->vectors;
    g.ptr = desc->graph;
    t.ptr = desc->tree_nodes;
    d.ptr = sh.num_deleted > 0 ? desc->deleted : nullptr;
    return build_handle(sh, v, g, desc->tree_starts, t, d, out);
}

void sptag_b200_destroy(sptag_b200_handle h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (auto& sc : h->scratch)
        if (sc.ev_done) cudaEventDestroy(sc.ev_done);
    for (auto& st : h->staging)
        if (st.stream) cudaStreamDestroy(st.stream);
    if (h->ev_start) cudaEventDestroy(h->ev_start);
    if (h->ev_stop) cudaEventDestroy(h->ev_stop);
    if (h->ev_aux) cudaEventDestroy(h->ev_aux);
    delete h;  // frees the device buffers, with the index's device current
}

namespace {
struct FileCloser {
    std::vector<FILE*> files;
    FILE* open(const std::string& path) {
        FILE* f = std::fopen(path.c_str(), "rb");
        if (f) files.push_back(f);
        return f;
    }
    ~FileCloser() {
        for (FILE* f : files) std::fclose(f);
    }
};
long long file_size(FILE* f) {
    if (fseeko(f, 0, SEEK_END) != 0) return -1;
    const long long sz = (long long)ftello(f);
    fseeko(f, 0, SEEK_SET);
    return sz;
}
}  // namespace

int sptag_b200_load(const char* folder, int32_t device, int32_t id_offset, sptag_b200_handle* out) {
    if (!folder || !out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    *out = nullptr;
    const std::string dir(folder);
    // indexloader.ini: "[Index]" section of Name=Value lines (VectorIndex.cpp:197-222, :617-681)
    std::ifstream ini(dir + "/indexloader.ini");
    if (!ini) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot open %s/indexloader.ini", folder);
    std::map<std::string, std::string> kv;
    std::string line;
    while (std::getline(ini, line)) {
        while (!line.empty() && (line.back() == '\r' || line.back() == ' ')) line.pop_back();
        if (line.empty() || line[0] == '[' || line[0] == ';' || line[0] == '#') continue;
        size_t eq = line.find('=');
        if (eq == std::string::npos) continue;
        kv[line.substr(0, eq)] = line.substr(eq + 1);
    }
    auto get = [&](const char* name, const char* def) {
        auto it = kv.find(name);
        return it == kv.end() ? std::string(def) : it->second;
    };
    IndexShape sh;
    sh.device = device;
    sh.id_offset = id_offset;
    const std::string algo = get("IndexAlgoType", "BKT");
    if (algo == "BKT")
        sh.algo = SPTAG_B200_ALGO_BKT;
    else if (algo == "KDT")
        sh.algo = SPTAG_B200_ALGO_KDT;
    else
        return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported IndexAlgoType %s", algo.c_str());
    const std::string vt = get("ValueType", "Float");
    if (vt == "Float")
        sh.value_type = SPTAG_B200_VT_FLOAT;
    else if (vt == "Int8")
        sh.value_type = SPTAG_B200_VT_INT8;
    else if (vt == "UInt8")
        sh.value_type = SPTAG_B200_VT_UINT8;
    else if (vt == "Int16")
        sh.value_type = SPTAG_B200_VT_INT16;
    else
        return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported ValueType %s", vt.c_str());
    const std::string dm = get("DistCalcMethod", "Cosine");  // reference default is Cosine
    sh.metric = (dm == "L2") ? SPTAG_B200_METRIC_L2
                             : (dm == "InnerProduct" ? SPTAG_B200_METRIC_INNERPRODUCT : SPTAG_B200_METRIC_COSINE);
    // the kernels implement the default seeding only (BKTree.h:696-769 with m_bfs == 0); a BFS-seeded index would
    // return different neighbours than the reference, so refuse it
    if (std::atoi(get("EnableBfs", "0").c_str()) != 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "EnableBfs != 0 (BFS tree seeding, BKTree.h:703-758) is not built");

    FileCloser fc;
    FILE* fv = fc.open(dir + "/" + get("VectorFilePath", "vectors.bin"));
    FILE* fg = fc.open(dir + "/" + get("GraphFilePath", "graph.bin"));
    FILE* ft = fc.open(dir + "/" + get("TreeFilePath", "tree.bin"));
    if (!fv) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read vectors file in %s", folder);
    if (!fg) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read graph file in %s", folder);
    if (!ft) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read tree file in %s", folder);
    FILE* fd = fc.open(dir + "/" + get("DeleteVectorFilePath", "deletes.bin"));

    // vectors.bin: int32 rows, int32 cols, rows*cols*T (Dataset.h:146-180)
    int32_t hdr[2];
    if (std::fread(hdr, 4, 2, fv) != 2) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read vectors file in %s", folder);
    sh.n = hdr[0];
    sh.dim = hdr[1];
    if (sh.n <= 0 || sh.dim <= 0) return fail(SPTAG_B200_EMPTY_INDEX, "empty index");
    if (file_size(fv) < 8 + (long long)sh.n * sh.dim * (long long)value_size(sh.value_type))
        return fail(SPTAG_B200_FAIL, "vectors file truncated");
    // graph.bin: int32 N, int32 degree, N*degree int32 (NeighborhoodGraph.h:606-615)
    if (std::fread(hdr, 4, 2, fg) != 2) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read graph file in %s", folder);
    if (hdr[0] != sh.n) return fail(SPTAG_B200_FAIL, "graph rows %d != vectors %d", hdr[0], sh.n);
    sh.degree = hdr[1];
    if (sh.degree <= 0 || file_size(fg) < 8 + (long long)sh.n * sh.degree * 4) return fail(SPTAG_B200_FAIL, "graph file truncated");
    // tree.bin: int32 treeNumber, starts[], int32 nodeCount, nodes[] (BKTree.h:635-645, KDTree.h:123-133)
    const long long tsz = file_size(ft);
    if (std::fread(hdr, 4, 1, ft) != 1) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read tree file in %s", folder);
    sh.tree_num = hdr[0];
    if (sh.tree_num <= 0 || (long long)sh.tree_num > (tsz - 8) / 4)
        return fail(SPTAG_B200_FAIL, "tree file: bad tree count %d", sh.tree_num);
    std::vector<int32_t> starts((size_t)sh.tree_num);
    if (std::fread(starts.data(), 4, starts.size(), ft) != starts.size() || std::fread(hdr, 4, 1, ft) != 1)
        return fail(SPTAG_B200_FAIL, "tree file truncated");
    sh.node_count = hdr[0];
    const long long node_sz = sh.algo == SPTAG_B200_ALGO_BKT ? 12 : 16;
    const long long nodes_off = (long long)(2 + sh.tree_num) * 4;
    if (sh.node_count <= 0 || tsz < nodes_off + (long long)sh.node_count * node_sz) return fail(SPTAG_B200_FAIL, "tree file truncated");
    // deletes.bin: int32 count, then Dataset<int8> (int32 rows, int32 cols, bytes) (Labelset.h:78-83)
    ArraySource v, g, t, d;
    if (fd) {
        int32_t dh[3];
        if (std::fread(dh, 4, 3, fd) != 3) return fail(SPTAG_B200_FAIL, "deletes file truncated");
        sh.num_deleted = dh[0];
        if (sh.num_deleted > 0) {
            // a short payload would silently resurrect every deleted vector: refuse it
            if (file_size(fd) < 12 + (long long)sh.n) return fail(SPTAG_B200_FAIL, "deletes file truncated (%d tombstones declared)", sh.num_deleted);
            d.file = fd;
            d.offset = 12;
        }
    }
    v.file = fv;
    v.offset = 8;
    g.file = fg;
    g.offset = 8;
    t.file = ft;
    t.offset = nodes_off;
    sptag_b200_handle h = nullptr;
    if (int rc = build_handle(sh, v, g, starts.data(), t, d, &h)) return rc;
    {
        auto it = kv.find("QuantizerFilePath");  // [Quantizer] section (VectorIndex.cpp:188-192)
        if (it != kv.end() && !it->second.empty()) {
            std::vector<char> qb;
            if (!read_file(dir + "/" + it->second, qb)) {
                sptag_b200_destroy(h);
                return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read quantizer file %s", it->second.c_str());
            }
            if (int rc = sptag_b200_set_quantizer(h, qb.data(), (int64_t)qb.size())) {
                sptag_b200_destroy(h);
                return rc;
            }
        }
    }
    static const char* names[] = {"MaxCheck", "MaxCheckForRefineGraph", "NumberOfInitialDynamicPivots",
                                  "NumberOfOtherDynamicPivots", "ThresholdOfNumberOfContinuousNoBetterPropagation",
                                  "AddCEF", "CEF", "RNGFactor"};
    for (const char* nm : names) {
        auto it = kv.find(nm);
        if (it != kv.end()) sptag_b200_set_param(h, nm, it->second.c_str());
    }
    *out = h;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_set_quantizer(sptag_b200_handle h, const void* blob, int64_t blob_bytes) {
    if (!h || !blob || blob_bytes < 14) return fail(SPTAG_B200_LACK_OF_INPUTS, "null or short quantizer blob");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    const unsigned char* b = (const unsigned char*)blob;
    const int qtype = b[0], rtype = b[1];
    int32_t hdr[3];
    memcpy(hdr, b + 2, 12);
    const int m = hdr[0], ks = hdr[1], dsub = hdr[2];
    if (qtype != 1 && qtype != 2) return fail(SPTAG_B200_LACK_OF_INPUTS, "unknown quantizer type %d", qtype);
    if (qtype == 1 && rtype != SPTAG_B200_VT_FLOAT)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "PQQuantizer<T> is supported for T = float only (reconstruct type %d)", rtype);
    if (rtype < 0 || rtype > 3 || m <= 0 || ks <= 0 || ks > 256 || dsub <= 0)
        return fail(SPTAG_B200_FAILED_PARSE_VALUE, "bad quantizer header (M %d Ks %d Dsub %d type %d)", m, ks, dsub, rtype);
    const size_t dim = (size_t)m * dsub;
    const size_t cb_bytes = (size_t)m * ks * dsub * 4;
    const size_t need = 14 + cb_bytes + (qtype == 2 ? dim * dim * 4 : 0);
    if ((size_t)blob_bytes < need) return fail(SPTAG_B200_FAILED_PARSE_VALUE, "quantizer blob truncated (%lld < %zu)",
                                              (long long)blob_bytes, need);
    if (int rc = h->d_codebooks.ensure(cb_bytes)) return rc;
    CUDA_OK(cudaMemcpy(h->d_codebooks.ptr, b + 14, cb_bytes, cudaMemcpyHostToDevice));
    if (qtype == 2) {
        // m_InitMatrixTranspose (OPQQuantizer.h:84-94): the rows the query is multiplied with
        const float* rot = (const float*)(b + 14 + cb_bytes);
        std::vector<float> rt(dim * dim);
        for (size_t i = 0; i < dim; ++i)
            for (size_t j = 0; j < dim; ++j) {
                float v;
                memcpy(&v, (const char*)rot + (j * dim + i) * 4, 4);
                rt[i * dim + j] = v;
            }
        if (int rc = h->d_rotation_t.ensure(dim * dim * 4)) return rc;
        CUDA_OK(cudaMemcpy(h->d_rotation_t.ptr, rt.data(), dim * dim * 4, cudaMemcpyHostToDevice));
        // m_OPQMatrix as stored: the rows ReconstructVector multiplies with (OPQQuantizer.h:124-131)
        if (int rc = h->d_rotation.ensure(dim * dim * 4)) return rc;
        CUDA_OK(cudaMemcpy(h->d_rotation.ptr, rot, dim * dim * 4, cudaMemcpyHostToDevice));
    }
    // InitializeDistanceTables (PQQuantizer.h:333-348) on the device, same summation tree as the reference
    const size_t entries = (size_t)m * ks * ks;
    if (int rc = h->d_sdc.ensure(entries * 4)) return rc;
    sdc_table_kernel<<<(unsigned)((entries + 255) / 256), 256>>>((const float*)h->d_codebooks.ptr, m, ks, dsub,
                                                                (float*)h->d_sdc.ptr);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaDeviceSynchronize());
    h->q_type = qtype;
    h->q_rtype = rtype;
    h->q_m = m;
    h->q_ks = ks;
    h->q_dsub = dsub;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_quantize(sptag_b200_handle h, const void* raw_vectors, int32_t num, uint8_t* codes_out) {
    if (!h || !raw_vectors || !codes_out || num <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (h->q_type == 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "index has no quantizer");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    const size_t rbytes = (size_t)num * query_bytes(h);
    if (int rc = h->d_raw.ensure(rbytes)) return rc;
    DeviceBuffer& d_codes = h->scratch[0].d_codes;
    if (int rc = d_codes.ensure((size_t)num * h->q_m)) return rc;
    CUDA_OK(cudaMemcpy(h->d_raw.ptr, raw_vectors, rbytes, cudaMemcpyHostToDevice));
    if (int rc = scratch_acquire(h, nullptr, 0)) return rc;
    if (int rc = quantize_device(h, h->d_raw.ptr, num, (unsigned char*)d_codes.ptr, nullptr)) return rc;
    if (int rc = scratch_release(h, nullptr, 0)) return rc;
    CUDA_OK(cudaMemcpy(codes_out, d_codes.ptr, (size_t)num * h->q_m, cudaMemcpyDeviceToHost));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_set_param(sptag_b200_handle h, const char* name, const char* value) {
    if (!h || !name || !value) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    char* end = nullptr;
    const long v = strtol(value, &end, 10);
    if (end == value) return fail(SPTAG_B200_FAILED_PARSE_VALUE, "cannot parse '%s' for %s", value, name);
    std::lock_guard<std::mutex> lock(h->mu);
    const std::string n(name);
    if (n == "MaxCheck") h->max_check = (int)v;
    else if (n == "MaxCheckForRefineGraph") h->max_check_refine = (int)v;
    else if (n == "AddCEF") h->add_cef = (int)v;
    else if (n == "CEF") h->cef = (int)v;
    else if (n == "RNGFactor") h->rng_factor = strtof(value, nullptr);
    else if (n == "SearchDeleted") h->search_deleted = (v != 0) ? 1 : 0;
    else if (n == "NumberOfInitialDynamicPivots") h->initial_pivots = (int)v;
    else if (n == "NumberOfOtherDynamicPivots") h->other_pivots = (int)v;
    else if (n == "ThresholdOfNumberOfContinuousNoBetterPropagation") h->no_better_threshold = (int)v;
    else if (n == "B200.QueriesPerSM") h->queries_per_sm = (int)v;
    else if (n == "B200.StageRows") h->stage_rows = (int)v;
    else if (n == "B200.Stages") { h->stages = (int)v; h->stages_set = true; }
    else if (n == "B200.NGCacheEntries") h->h_ng = (int)v;
    else if (n == "B200.SPTCacheEntries") h->h_spt = (int)v;
    else if (n == "B200.SimdWidth") h->simd_width = (int)v;
    else if (n == "B200.VisitedLog") h->visited_log = (int)v;
    else if (n == "B200.VisitedLogEntries") h->visited_log_entries = (int)v;
    else if (n == "B200.SlotScheme") h->slot_scheme = (int)v;
    else if (n == "EnableADC") h->q_adc = (v != 0);  // VectorIndex::SetQuantizerADC (VectorIndex.h:136-138)
    else return fail(SPTAG_B200_PARAM_NOT_FOUND, "unknown parameter %s", name);
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_get_param(sptag_b200_handle h, const char* name, char* value_out, int32_t capacity) {
    if (!h || !name || !value_out || capacity <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    std::lock_guard<std::mutex> lock(h->mu);
    const std::string n(name);
    long v;
    if (n == "RNGFactor") {  // float, printed like the reference's ini (ConvertToString)
        snprintf(value_out, (size_t)capacity, "%f", h->rng_factor);
        return SPTAG_B200_SUCCESS;
    }
    if (n == "MaxCheck") v = h->max_check;
    else if (n == "MaxCheckForRefineGraph") v = h->max_check_refine;
    else if (n == "AddCEF") v = h->add_cef;
    else if (n == "CEF") v = h->cef;
    else if (n == "SearchDeleted") v = h->search_deleted;
    else if (n == "NumberOfInitialDynamicPivots") v = h->initial_pivots;
    else if (n == "NumberOfOtherDynamicPivots") v = h->other_pivots;
    else if (n == "ThresholdOfNumberOfContinuousNoBetterPropagation") v = h->no_better_threshold;
    else if (n == "B200.QueriesPerSM") v = h->queries_per_sm;
    else if (n == "B200.StageRows") v = h->stage_rows;
    else if (n == "B200.Stages") v = h->stages;
    else if (n == "B200.NGCacheEntries") v = h->h_ng;
    else if (n == "B200.SPTCacheEntries") v = h->h_spt;
    else if (n == "B200.SimdWidth") v = h->simd_width;
    else if (n == "B200.VisitedLog") v = h->visited_log;
    else if (n == "B200.VisitedLogEntries") v = h->visited_log_entries;
    else if (n == "B200.SlotScheme") v = h->slot_scheme;
    else if (n == "EnableADC") v = h->q_adc;
    else if (n == "B200.LastRefineSearchUs") v = (long)(h->refine_search_ms * 1000.0);    // read-only: device time
    else if (n == "B200.LastRefineRebuildUs") v = (long)(h->refine_rebuild_ms * 1000.0);  // of the last refine pass
    else return fail(SPTAG_B200_PARAM_NOT_FOUND, "unknown parameter %s", name);
    snprintf(value_out, (size_t)capacity, "%ld", v);
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_search_device(sptag_b200_handle h, const void* d_queries, int32_t num_queries, int32_t k,
                             int32_t* d_out_ids, float* d_out_dists, int32_t* d_out_stats, void* cuda_stream) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && (!d_queries || !d_out_ids || !d_out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    return search_device_impl(h, d_queries, num_queries, k, d_out_ids, d_out_dists, d_out_stats,
                              (cudaStream_t)cuda_stream);
}

namespace {
// Host-buffer search: staging set, H2D, launch (under h->mu), D2H.  refine = the RefineSearchIndex flavour.
int search_host_impl(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k, CallOpts opts,
                     const uint8_t* allowed, bool refine, int32_t* out_ids, float* out_dists, int32_t* out_stats) {
    if (num_queries == 0) return SPTAG_B200_SUCCESS;
    // a staging set of our own for the whole call: the one that is free, else wait for the next in turn
    sptag_b200_index::Staging* st = nullptr;
    std::unique_lock<std::mutex> slock;
    for (auto& cand : h->staging) {
        std::unique_lock<std::mutex> l(cand.mu, std::try_to_lock);
        if (l.owns_lock()) {
            st = &cand;
            slock = std::move(l);
            break;
        }
    }
    if (!st) {
        st = &h->staging[h->staging_rr.fetch_add(1) & 1u];
        slock = std::unique_lock<std::mutex>(st->mu);
    }
    DeviceGuard guard(h->device);
    const size_t qbytes = (size_t)num_queries * query_bytes(h);
    const size_t rn = (size_t)num_queries * k;
    if (int rc = st->d_queries.ensure(qbytes)) return rc;
    if (int rc = st->d_ids.ensure(rn * 4)) return rc;
    if (int rc = st->d_dists.ensure(rn * 4)) return rc;
    if (out_stats)
        if (int rc = st->d_stats.ensure((size_t)num_queries * kStatsPerQuery * 4)) return rc;
    cudaStream_t stream = st->stream;
    CUDA_OK(cudaMemcpyAsync(st->d_queries.ptr, queries, qbytes, cudaMemcpyHostToDevice, stream));
    int map_n = 0;
    if (allowed) {
        // SearchIndexWithFilter: the caller evaluated filterFunc once per vector; the map is this call's own copy
        {
            std::lock_guard<std::mutex> lock(h->mu);
            map_n = h->n;
        }
        if (int rc = st->d_filter.ensure((size_t)map_n)) return rc;
        CUDA_OK(cudaMemcpyAsync(st->d_filter.ptr, allowed, (size_t)map_n, cudaMemcpyHostToDevice, stream));
        opts.d_filter = (const unsigned char*)st->d_filter.ptr;
    }
    {
        std::lock_guard<std::mutex> lock(h->mu);  // launch set-up + enqueue only; the copies above / below overlap other callers' kernels
        if (allowed && h->n != map_n) {  // an add ran in between: the map no longer covers every vector
            cudaStreamSynchronize(stream);
            return fail(SPTAG_B200_FAIL, "the index grew from %d to %d vectors during the filtered search", map_n, h->n);
        }
        if (int rc = search_device_impl(h, st->d_queries.ptr, num_queries, k, (int*)st->d_ids.ptr, (float*)st->d_dists.ptr,
                                        out_stats ? (int*)st->d_stats.ptr : nullptr, stream, refine, opts)) {
            cudaStreamSynchronize(stream);
            return rc;
        }
    }
    CUDA_OK(cudaMemcpyAsync(out_ids, st->d_ids.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_dists, st->d_dists.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    if (out_stats)
        CUDA_OK(cudaMemcpyAsync(out_stats, st->d_stats.ptr, (size_t)num_queries * kStatsPerQuery * 4,
                                cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    return SPTAG_B200_SUCCESS;
}
}  // namespace

int sptag_b200_search_ex(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                         const sptag_b200_search_options* options, int32_t* out_ids, float* out_dists,
                         int32_t* out_stats) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && (!queries || !out_ids || !out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    CallOpts opts;
    const uint8_t* allowed = nullptr;
    if (options) {
        if (options->struct_size != (int32_t)sizeof(sptag_b200_search_options))
            return fail(SPTAG_B200_FAIL, "options size mismatch: %d vs %zu", options->struct_size, sizeof(sptag_b200_search_options));
        opts.search_deleted = options->search_deleted ? 1 : 0;
        opts.max_check = options->max_check > 0 ? options->max_check : 0;
        allowed = options->allowed;
        if (allowed && h->algo != SPTAG_B200_ALGO_BKT) return fail(SPTAG_B200_FAIL, "Not Support Filter on KDT Index!");
    }
    return search_host_impl(h, queries, num_queries, k, opts, allowed, false, out_ids, out_dists, out_stats);
}

int sptag_b200_refine_search(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                             int32_t search_deleted, int32_t* out_ids, float* out_dists) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && (!queries || !out_ids || !out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (h->q_type != 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "refine on a quantized index (reconstruct + re-quantize) is not built");
    CallOpts opts;
    {
        std::lock_guard<std::mutex> lock(h->mu);
        opts.max_check = h->max_check_refine;  // workSpace->Reset(m_pGraph.m_iMaxCheckForRefineGraph, K)
    }
    opts.search_deleted = search_deleted ? 1 : 0;
    return search_host_impl(h, queries, num_queries, k, opts, nullptr, true, out_ids, out_dists, nullptr);
}

int sptag_b200_search(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k, int32_t* out_ids,
                      float* out_dists, int32_t* out_stats) {
    return sptag_b200_search_ex(h, queries, num_queries, k, nullptr, out_ids, out_dists, out_stats);
}

int sptag_b200_search_filtered(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t k,
                               const uint8_t* allowed, int32_t max_check, int32_t* out_ids, float* out_dists,
                               int32_t* out_stats) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!allowed) return fail(SPTAG_B200_LACK_OF_INPUTS, "null filter map");
    sptag_b200_search_options o;
    memset(&o, 0, sizeof(o));
    o.struct_size = (int32_t)sizeof(o);
    {
        std::lock_guard<std::mutex> lock(h->mu);
        o.search_deleted = h->search_deleted;  // the handle-wide default, as sptag_b200_search reads it
    }
    o.max_check = max_check;  // workSpace->Reset(maxCheck == 0 ? m_iMaxCheck : maxCheck, K)
    o.allowed = allowed;
    return sptag_b200_search_ex(h, queries, num_queries, k, &o, out_ids, out_dists, out_stats);
}

int sptag_b200_refine_graph(sptag_b200_handle h, int32_t first_node, int32_t num_nodes, int32_t cef,
                            int32_t neighborhood_size, float rng_factor, int32_t* out_graph, int32_t* out_res_ids,
                            float* out_res_dists, int32_t install) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    const bool pq = (h->q_type != 0);
    if (pq && h->q_adc)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "refine on a quantized index with ADC on: the reference's RebuildNeighbors reads a "
                                              "code row as a distance table there (PQQuantizer.h:114-119); turn ADC off");
    if (first_node < 0 || num_nodes < 0 || (long long)first_node + num_nodes > h->n)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "node range [%d, %d) outside the index", first_node, first_node + num_nodes);
    if (cef < 1 || cef + 1 > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "CEF = %d outside [1, 2047]", cef);
    if (neighborhood_size < 1 || neighborhood_size > 1024)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "neighbourhood size %d outside [1, 1024]", neighborhood_size);
    if (install && (first_node != 0 || num_nodes != h->n))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "install needs a full pass over the index");
    if (num_nodes == 0) return SPTAG_B200_SUCCESS;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    const int k = cef + 1;
    const int batch = std::min(num_nodes, 32768);  // 32768 x 1001 result pairs = 262 MB of scratch (524 MB at CEF 2000)
    if (int rc = h->d_ids.ensure((size_t)batch * k * 4)) return rc;
    if (int rc = h->d_dists.ensure((size_t)batch * k * 4)) return rc;
    if (int rc = h->d_graph_new.ensure((size_t)num_nodes * neighborhood_size * 4)) return rc;
    cudaStream_t stream = nullptr;
    CallOpts ropts;
    ropts.max_check = h->max_check_refine;  // workSpace->Reset(m_pGraph.m_iMaxCheckForRefineGraph, CEF + 1)
    ropts.search_deleted = 0;               // RefineNode(index, node, false, searchDeleted = false, CEF)
    ropts.refine_query_stride = h->row_stride;  // the queries are the index's own (padded) rows
    int rc = SPTAG_B200_SUCCESS;
    h->refine_search_ms = h->refine_rebuild_ms = 0.0;
    const unsigned char* dv = (const unsigned char*)h->d_vectors.ptr;
    if (pq) {
        // RefineNode on a quantized index (NeighborhoodGraph.h:538-543): the query is NOT the stored code row but what
        // SetTarget makes of its reconstruction, so each batch is reconstructed into packed raw vectors and goes through
        // the ordinary raw-query path of search_device_impl (QuantizeVector on the device)
        ropts.refine_query_stride = 0;
        if (int rc2 = h->d_rec.ensure((size_t)batch * query_bytes(h))) return rc2;
    }
    for (int done = 0; done < num_nodes && rc == SPTAG_B200_SUCCESS; done += batch) {
        const int nb = std::min(batch, num_nodes - done);
        const int first = first_node + done;
        const unsigned char* queries = dv + (size_t)first * h->row_stride;
        if (pq) {
            const size_t rsmem = (size_t)h->q_m * h->q_dsub * sizeof(float);
            if (rsmem > 48 * 1024)
                CUDA_OK(cudaFuncSetAttribute(pq_reconstruct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rsmem));
            pq_reconstruct_kernel<<<nb, 128, rsmem, stream>>>(queries, h->row_stride, nb, (const float*)h->d_codebooks.ptr,
                                                            h->q_type == 2 ? (const float*)h->d_rotation.ptr : nullptr,
                                                            h->q_m, h->q_ks, h->q_dsub, h->q_rtype,
                                                            (unsigned char*)h->d_rec.ptr);
            g_launches++;
            CUDA_OK(cudaGetLastError());
            queries = (const unsigned char*)h->d_rec.ptr;
        }
        rc = search_device_impl(h, queries, nb, k, (int*)h->d_ids.ptr, (float*)h->d_dists.ptr,
                                nullptr, stream, /*refine=*/true, ropts);
        if (rc) break;
        const int warps_per_block = 4;
        const unsigned blocks = (unsigned)((nb + warps_per_block - 1) / warps_per_block);
        const size_t smem = (size_t)warps_per_block * neighborhood_size * 4;
        int* rows = (int*)h->d_graph_new.ptr + (size_t)done * neighborhood_size;
        if (pq) {
            rebuild_neighbors_pq_kernel<<<blocks, warps_per_block * 32, smem, stream>>>(
                dv, h->row_stride, h->q_m, h->q_ks, (const float*)h->d_sdc.ptr, first, nb, (const int*)h->d_ids.ptr,
                (const float*)h->d_dists.ptr, k, neighborhood_size, rng_factor, rows);
        } else {
            with_metric_elem(h, [&](auto cos, auto el) {
                rebuild_neighbors_kernel<cos, el><<<blocks, warps_per_block * 32, smem, stream>>>(
                    dv, h->row_stride, h->dim, first, nb, (const int*)h->d_ids.ptr, (const float*)h->d_dists.ptr, k,
                    neighborhood_size, rng_factor, rows, h->simd_width);
            });
        }
        g_launches++;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaEventRecord(h->ev_aux, stream);
        if (e == cudaSuccess && out_res_ids)
            e = cudaMemcpyAsync(out_res_ids + (size_t)done * k, h->d_ids.ptr, (size_t)nb * k * 4, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess && out_res_dists)
            e = cudaMemcpyAsync(out_res_dists + (size_t)done * k, h->d_dists.ptr, (size_t)nb * k * 4, cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (e == cudaSuccess) {
            float ms_s = 0.f, ms_r = 0.f;
            cudaEventElapsedTime(&ms_s, h->ev_start, h->ev_stop);
            cudaEventElapsedTime(&ms_r, h->ev_stop, h->ev_aux);
            h->refine_search_ms += ms_s;
            h->refine_rebuild_ms += ms_r;
        }
        if (e != cudaSuccess) rc = fail(SPTAG_B200_FAIL, "refine pass failed: %s", cudaGetErrorString(e));
    }
    if (rc) return rc;
    if (out_graph)
        CUDA_OK(cudaMemcpy(out_graph, h->d_graph_new.ptr, (size_t)num_nodes * neighborhood_size * 4, cudaMemcpyDeviceToHost));
    return install ? install_graph(h, neighborhood_size, stream) : SPTAG_B200_SUCCESS;
}

int sptag_b200_rebuild_graph(sptag_b200_handle h, int32_t* out_graph, int32_t install) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    const int stride = h->degree, ns = h->degree / 2;
    if ((h->degree & 1) || ns < 2 || ns > 1024)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "RebuildGraph needs rows of 2 x N candidates, N in [2, 1024] (degree is %d)", h->degree);
    const long long n = h->n;
    DeviceBuffer d_indegree;
    if (int rc = d_indegree.ensure((size_t)std::max<long long>(n, 1) * 4)) return rc;
    if (int rc = h->d_graph_new.ensure((size_t)n * ns * 4)) return rc;
    cudaStream_t stream = nullptr;
    cudaError_t e = cudaMemsetAsync(d_indegree.ptr, 0, (size_t)n * 4, stream);
    if (e == cudaSuccess) {
        const long long total = n * ns;
        indegree_count_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const int*)h->d_graph.ptr, n, stride, ns,
                                                                                  (int*)d_indegree.ptr);
        rebuild_graph_kernel<<<1, 32, 0, stream>>>((const int*)h->d_graph.ptr, (int)n, stride, ns, (int*)d_indegree.ptr,
                                                  (int*)h->d_graph_new.ptr);
        g_launches += 2;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "rebuild graph failed: %s", cudaGetErrorString(e));
    if (out_graph) CUDA_OK(cudaMemcpy(out_graph, h->d_graph_new.ptr, (size_t)n * ns * 4, cudaMemcpyDeviceToHost));
    return install ? install_graph(h, ns, stream) : SPTAG_B200_SUCCESS;
}

int sptag_b200_refine_schedule(sptag_b200_handle h, int32_t refine_iterations, int32_t cef, float cef_scale,
                                 int32_t neighborhood_size, float neighborhood_scale, float rng_factor) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (refine_iterations < 0 || cef < 1 || neighborhood_size < 1 || !(cef_scale > 0.f) || !(neighborhood_scale > 0.f))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "bad refine schedule");
    // NeighborhoodGraph::BuildGraph runs its passes on rows of NeighborhoodSize x NeighborhoodScale entries
    // (m_iNeighborhoodSize is that product while the graph is built); RefineGraph (NeighborhoodGraph.h:460-492):
    //   passes 0 .. RefineIterations-2: RefineNode(..., (int)(CEF * CEFScale)) on the wide rows,
    //   then m_iNeighborhoodSize = (int)(m_iNeighborhoodSize / NeighborhoodScale) and one pass with CEF.
    const int wide = (int)(neighborhood_size * neighborhood_scale);
    const int big_cef = (int)(cef * cef_scale);
    const int narrow = (int)(wide / neighborhood_scale);
    for (int iter = 0; iter < refine_iterations - 1; ++iter)
        if (int rc = sptag_b200_refine_graph(h, 0, h->n, big_cef, wide, rng_factor, nullptr, nullptr, nullptr, 1)) return rc;
    if (refine_iterations > 0)
        if (int rc = sptag_b200_refine_graph(h, 0, h->n, cef, narrow, rng_factor, nullptr, nullptr, nullptr, 1)) return rc;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_get_graph(sptag_b200_handle h, int32_t* out_graph) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!out_graph) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    CUDA_OK(cudaMemcpy(out_graph, h->d_graph.ptr, (size_t)h->n * h->degree * 4, cudaMemcpyDeviceToHost));
    return SPTAG_B200_SUCCESS;
}

int32_t sptag_b200_graph_degree(sptag_b200_handle h) { return h ? h->degree : 0; }

int sptag_b200_iterator_open(sptag_b200_handle h, const void* queries, int32_t num_queries, sptag_b200_iter* out) {
    return sptag_b200_iterator_open_ex(h, queries, num_queries, -1, out);
}

int sptag_b200_iterator_open_ex(sptag_b200_handle h, const void* queries, int32_t num_queries, int32_t search_deleted,
                                sptag_b200_iter* out) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!out || !queries || num_queries <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    *out = nullptr;
    if (h->algo != SPTAG_B200_ALGO_BKT) return fail(SPTAG_B200_FAIL, "ITERATIVE NOT SUPPORT FOR KDT");
    if (h->q_type != 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "iterators on quantized indexes are not built");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    SearchLaunch L;
    if (int rc = plan_search(h, 1, num_queries, CallOpts(), L)) return rc;  // the search's refusals, queue lengths, arena sizes
    const SearchParams& p = L.p;
    auto* it = new sptag_b200_iterator();
    it->h = h;
    it->nq = num_queries;
    it->max_check = h->max_check;
    it->search_deleted = search_deleted < 0 ? h->search_deleted : (search_deleted ? 1 : 0);
    it->ng_length = p.ng_length;
    it->ng_lastlevel = p.ng_lastlevel;
    it->spt_length = p.spt_length;
    it->spt_lastlevel = p.spt_lastlevel;
    it->visited_words = p.visited_words;
    // NGQueue arena: a plain scan inserts every node at most once (n + 2 bounds it), but after
    // SearchIndexIterativeFromNeareast's nodeCheckStatus.clear() the leftovers of the finished search stay queued while
    // every node may enter once more, so 2 (n + 2) is the bound; Heap::insert itself stops at `length`
    it->ng_entries = round_up((size_t)std::min<long long>((long long)p.ng_length, 2 * ((long long)h->n + 2)) + 2, 2);
    it->spt_entries = p.spt_spill_entries;
    const size_t qbytes = (size_t)num_queries * query_bytes(h);
    int rc = 0;
    if ((rc = it->d_queries.ensure(qbytes)) || (rc = it->d_visited.ensure((size_t)num_queries * it->visited_words * 4)) ||
        (rc = it->d_ng.ensure((size_t)num_queries * it->ng_entries * 8)) ||
        (rc = it->d_spt.ensure((size_t)num_queries * it->spt_entries * 8)) ||
        (rc = it->d_state.ensure((size_t)num_queries * kIterStateInts * 4)) ||
        (rc = it->d_counts.ensure((size_t)num_queries * 4)) || (rc = it->d_relaxed.ensure((size_t)num_queries))) {
        delete it;
        return rc;
    }
    std::vector<int> st((size_t)num_queries * kIterStateInts, 0);
    for (int q = 0; q < num_queries; ++q) {
        st[(size_t)q * kIterStateInts + 2] = 1;   // first call: InitSearchTrees + SearchTrees
        st[(size_t)q * kIterStateInts + 4] = -1;  // no QueryResult yet: the first Next sets the slot count
    }
    cudaError_t e = cudaMemcpy(it->d_queries.ptr, queries, qbytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(it->d_visited.ptr, 0, it->d_visited.bytes);
    if (e == cudaSuccess) e = cudaMemcpy(it->d_state.ptr, st.data(), st.size() * 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        delete it;
        return fail(SPTAG_B200_FAIL, "iterator set-up failed: %s", cudaGetErrorString(e));
    }
    h->open_iterators++;  // sptag_b200_iterator_close gives it back
    *out = it;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_iterator_next(sptag_b200_iter it, int32_t batch, int32_t* out_ids, float* out_dists, int32_t* out_counts,
                             uint8_t* out_relaxed_mono) {
    if (!it || !it->h) return fail(SPTAG_B200_EMPTY_INDEX, "null iterator");
    if (!out_ids || !out_dists) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (batch < 1 || batch > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "batch = %d outside [1, 1024]", batch);
    sptag_b200_index* h = it->h;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    SearchLaunch L;
    if (int rc = plan_iterator_step(it, batch, L)) return rc;
    IterateKernelFn kern = pick_iterate_kernel_for(h->value_type, h->metric != SPTAG_B200_METRIC_L2, L.p.mres_cap);
    if (!kern) return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, batch) = %d exceeds the supported 1024", L.p.mres_cap);
    return run_iterator_step(it, batch, "batch", L, out_ids, out_dists, out_counts, out_relaxed_mono,
                             [&](const SearchParams& p, int grid, size_t smem, cudaStream_t stream) {
                                 CUDA_OK(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                                 kern<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr, (int*)it->d_counts.ptr,
                                                                  (unsigned char*)it->d_relaxed.ptr);
                                 return 0;
                             });
}

int sptag_b200_iterator_next_from_nearest(sptag_b200_iter it, int32_t k, int32_t* out_ids, float* out_dists,
                                          uint8_t* out_found) {
    if (!it || !it->h) return fail(SPTAG_B200_EMPTY_INDEX, "null iterator");
    if (!out_ids || !out_dists) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (k < 1 || k > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside [1, 1024]", k);
    const bool first = (it->nearest_k == 0);
    if (first && it->stepped)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "the first SearchIndexIterativeFromNeareast call needs a freshly opened iterator");
    if (!first && k != it->nearest_k)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d differs from the head QueryResult's %d slots", k, it->nearest_k);
    sptag_b200_index* h = it->h;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    SearchLaunch L;
    if (int rc = plan_iterator_step(it, k, L)) return rc;
    const bool cosine = h->metric != SPTAG_B200_METRIC_L2;
    NearestFirstKernelFn kfirst = pick_nearest_first_kernel_for(h->value_type, cosine, L.p.mres_cap);
    IterateKernelFn knext = pick_iterate_kernel_for(h->value_type, cosine, L.p.mres_cap);
    if (!kfirst || !knext)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, k) = %d exceeds the supported 1024", L.p.mres_cap);
    const int rc = run_iterator_step(
        it, k, "k", L, out_ids, out_dists, nullptr, nullptr, [&](const SearchParams& p, int grid, size_t smem, cudaStream_t stream) {
            if (first) {
                CUDA_OK(cudaFuncSetAttribute((const void*)kfirst, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                kfirst<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr);
            } else {
                // the caller Reset()s a QueryResult that keeps its k slots (SPANNIndex.cpp:284): no cap from the previous count
                CUDA_OK(cudaMemset2DAsync((int*)it->d_state.ptr + 4, (size_t)kIterStateInts * 4, 0xFF, 4, (size_t)it->nq, stream));
                CUDA_OK(cudaFuncSetAttribute((const void*)knext, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                knext<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr, (int*)it->d_counts.ptr, (unsigned char*)it->d_relaxed.ptr);
            }
            return 0;
        });
    if (rc) return rc;
    if (out_found)  // the reference's return value: is the first result slot a real vector
        for (int q = 0; q < it->nq; ++q) out_found[q] = out_ids[(size_t)q * k] >= 0 ? 1 : 0;
    it->nearest_k = k;
    return SPTAG_B200_SUCCESS;
}

void sptag_b200_iterator_close(sptag_b200_iter it) {
    if (!it) return;
    if (it->h) {
        std::lock_guard<std::mutex> lock(it->h->mu);
        DeviceGuard guard(it->h->device);
        it->h->open_iterators--;
        delete it;  // frees the per-query arenas, with the index's device current
        return;
    }
    delete it;
}

int sptag_b200_distance_batch(sptag_b200_handle h, const void* queries, int32_t num_queries, const int32_t* ids,
                              int32_t ids_per_query, float* out) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!queries || !ids || !out || num_queries <= 0 || ids_per_query <= 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (h->q_type != 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "distance_batch handles raw (un-quantized) vectors only");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    const size_t qrow = (size_t)h->dim * value_size(h->value_type);
    const size_t qstride = (qrow + 3) & ~(size_t)3;  // integer rows: 4-byte aligned queries (2-/4-byte loads per lane)
    const size_t qbytes = (size_t)num_queries * qstride;
    const size_t total = (size_t)num_queries * ids_per_query;
    DeviceBuffer dq, di, dout;
    int rc = 0;
    if ((rc = dq.ensure(qbytes)) || (rc = di.ensure(total * 4)) || (rc = dout.ensure(total * 4))) return rc;
    if (qrow == qstride)
        cudaMemcpy(dq.ptr, queries, qbytes, cudaMemcpyHostToDevice);
    else
        cudaMemcpy2D(dq.ptr, qstride, queries, qrow, qrow, (size_t)num_queries, cudaMemcpyHostToDevice);
    cudaMemcpy(di.ptr, ids, total * 4, cudaMemcpyHostToDevice);
    const long long halfwarps = (long long)((total + 1) / 2) * 2;
    const int threads = 256;
    const long long blocks = (halfwarps * 16 + threads - 1) / threads;
    const unsigned char* dv = (const unsigned char*)h->d_vectors.ptr;
    with_metric_elem(h, [&](auto cos, auto el) {
        distance_batch_kernel<cos, el><<<(unsigned)blocks, threads>>>(dv, h->row_stride, h->n, h->dim, dq.ptr, num_queries,
                                                                      (const int*)di.ptr, ids_per_query, (float*)dout.ptr,
                                                                      h->simd_width);
    });
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpy(out, dout.ptr, total * 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "distance_batch failed: %s", cudaGetErrorString(e));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_merge_topk(int32_t device, const int32_t* d_ids, const float* d_dists, int32_t num_lists,
                          int32_t num_queries, int32_t k, int32_t* d_out_ids, float* d_out_dists, void* cuda_stream) {
    if (!d_ids || !d_dists || !d_out_ids || !d_out_dists) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (num_lists < 1 || num_lists > 16) return fail(SPTAG_B200_LACK_OF_INPUTS, "num_lists %d outside [1,16]", num_lists);
    if (num_queries <= 0 || k <= 0) return SPTAG_B200_SUCCESS;
    if (device < 0) CUDA_OK(cudaGetDevice(&device));
    DeviceGuard guard(device);
    const int threads = 128;
    merge_topk_kernel<<<(num_queries + threads - 1) / threads, threads, 0, (cudaStream_t)cuda_stream>>>(
        d_ids, d_dists, num_lists, num_queries, k, d_out_ids, d_out_dists);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return SPTAG_B200_SUCCESS;
}

// ---------------------------------------------------------------------------------------------------------------
// Vector-partition shards of ONE process (SURVEY.md 8e; the reference's Aggregator deployment,
// AggregatorService.cpp:215-412, fans a query out to its index servers and merges the lists): every shard is an
// ordinary handle on its own GPU with its id_offset; a group search runs all shards at once and merges on the first
// shard's GPU by reading the other GPUs' result lists through NVLink peer access inside the merge kernel.
// ---------------------------------------------------------------------------------------------------------------
struct sptag_b200_shard_group {
    std::vector<sptag_b200_index*> shards;
    struct PerShard {
        cudaStream_t stream = nullptr;
        cudaEvent_t done = nullptr;
        DeviceBuffer d_queries, d_ids, d_dists;
    };
    std::vector<PerShard> per;
    DeviceBuffer d_out_ids, d_out_dists;  // on shards[0]'s device
    cudaEvent_t ev_q = nullptr;
    std::mutex mu;
};

int sptag_b200_group_create(const sptag_b200_handle* shards, int32_t num_shards, sptag_b200_group* out) {
    if (!shards || !out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    *out = nullptr;
    if (num_shards < 1 || num_shards > 16) return fail(SPTAG_B200_LACK_OF_INPUTS, "num_shards %d outside [1, 16]", num_shards);
    for (int i = 0; i < num_shards; ++i) {
        if (!shards[i]) return fail(SPTAG_B200_EMPTY_INDEX, "shard %d is null", i);
        if (shards[i]->dim != shards[0]->dim || shards[i]->value_type != shards[0]->value_type ||
            shards[i]->metric != shards[0]->metric || shards[i]->q_type != shards[0]->q_type)
            return fail(SPTAG_B200_DIMENSION_MISMATCH, "shard %d differs from shard 0 in dimension, value type, metric or quantizer", i);
    }
    auto* g = new sptag_b200_shard_group();
    g->shards.assign(shards, shards + num_shards);
    g->per.resize((size_t)num_shards);
    const int home = shards[0]->device;
    for (int i = 0; i < num_shards; ++i) {
        DeviceGuard guard(shards[i]->device);
        if (cudaStreamCreate(&g->per[(size_t)i].stream) != cudaSuccess ||
            cudaEventCreateWithFlags(&g->per[(size_t)i].done, cudaEventDisableTiming) != cudaSuccess) {
            sptag_b200_group_destroy(g);
            return fail(SPTAG_B200_FAIL, "stream / event creation failed on device %d", shards[i]->device);
        }
        if (shards[i]->device != home) {  // the merge kernel on `home` dereferences this shard's result lists
            int can = 0;
            cudaDeviceCanAccessPeer(&can, home, shards[i]->device);
            if (!can) {
                sptag_b200_group_destroy(g);
                return fail(SPTAG_B200_FAIL, "device %d cannot access device %d (no NVLink / P2P path)", home, shards[i]->device);
            }
            DeviceGuard hg(home);
            const cudaError_t e = cudaDeviceEnablePeerAccess(shards[i]->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                sptag_b200_group_destroy(g);
                return fail(SPTAG_B200_FAIL, "cudaDeviceEnablePeerAccess(%d -> %d): %s", home, shards[i]->device, cudaGetErrorString(e));
            }
            cudaGetLastError();
        }
    }
    {
        DeviceGuard guard(home);
        if (cudaEventCreateWithFlags(&g->ev_q, cudaEventDisableTiming) != cudaSuccess) {
            sptag_b200_group_destroy(g);
            return fail(SPTAG_B200_FAIL, "event creation failed");
        }
    }
    *out = g;
    return SPTAG_B200_SUCCESS;
}

void sptag_b200_group_destroy(sptag_b200_group g) {
    if (!g) return;
    for (size_t i = 0; i < g->per.size(); ++i) {
        DeviceGuard guard(g->shards[i]->device);
        cudaDeviceSynchronize();
        g->per[i].d_queries.release();
        g->per[i].d_ids.release();
        g->per[i].d_dists.release();
        if (g->per[i].stream) cudaStreamDestroy(g->per[i].stream);
        if (g->per[i].done) cudaEventDestroy(g->per[i].done);
    }
    if (!g->shards.empty()) {
        DeviceGuard guard(g->shards[0]->device);
        g->d_out_ids.release();
        g->d_out_dists.release();
        if (g->ev_q) cudaEventDestroy(g->ev_q);
    }
    delete g;
}

int sptag_b200_group_search(sptag_b200_group g, const void* queries, int32_t num_queries, int32_t k, int32_t* out_ids,
                            float* out_dists) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null group");
    if (num_queries < 0 || (num_queries > 0 && (!queries || !out_ids || !out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (num_queries == 0) return SPTAG_B200_SUCCESS;
    std::lock_guard<std::mutex> glock(g->mu);
    const int ns = (int)g->shards.size();
    const size_t qbytes = (size_t)num_queries * query_bytes(g->shards[0]);
    const size_t rn = (size_t)num_queries * k;
    ShardLists lists;
    memset(&lists, 0, sizeof(lists));
    // fan out: every GPU gets the batch and starts its own search; nothing here waits for a device
    for (int i = 0; i < ns; ++i) {
        sptag_b200_index* h = g->shards[(size_t)i];
        auto& ps = g->per[(size_t)i];
        DeviceGuard guard(h->device);
        if (int rc = ps.d_queries.ensure(qbytes)) return rc;
        if (int rc = ps.d_ids.ensure(rn * 4)) return rc;
        if (int rc = ps.d_dists.ensure(rn * 4)) return rc;
        CUDA_OK(cudaMemcpyAsync(ps.d_queries.ptr, queries, qbytes, cudaMemcpyHostToDevice, ps.stream));
        {
            std::lock_guard<std::mutex> lock(h->mu);
            if (int rc = search_device_impl(h, ps.d_queries.ptr, num_queries, k, (int*)ps.d_ids.ptr, (float*)ps.d_dists.ptr, nullptr,
                                            ps.stream))
                return rc;
        }
        CUDA_OK(cudaEventRecord(ps.done, ps.stream));
        lists.ids[i] = (const int*)ps.d_ids.ptr;
        lists.dists[i] = (const float*)ps.d_dists.ptr;
    }
    // gather + merge in one kernel on shard 0's GPU: it reads the other GPUs' lists over NVLink
    sptag_b200_index* h0 = g->shards[0];
    DeviceGuard guard(h0->device);
    if (int rc = g->d_out_ids.ensure(rn * 4)) return rc;
    if (int rc = g->d_out_dists.ensure(rn * 4)) return rc;
    cudaStream_t s0 = g->per[0].stream;
    for (int i = 1; i < ns; ++i) CUDA_OK(cudaStreamWaitEvent(s0, g->per[(size_t)i].done, 0));
    const int threads = 128;
    merge_topk_peer_kernel<<<(num_queries + threads - 1) / threads, threads, 0, s0>>>(lists, ns, num_queries, k, (int*)g->d_out_ids.ptr,
                                                                                       (float*)g->d_out_dists.ptr);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaMemcpyAsync(out_ids, g->d_out_ids.ptr, rn * 4, cudaMemcpyDeviceToHost, s0));
    CUDA_OK(cudaMemcpyAsync(out_dists, g->d_out_dists.ptr, rn * 4, cudaMemcpyDeviceToHost, s0));
    CUDA_OK(cudaStreamSynchronize(s0));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_last_kernel_ms(sptag_b200_handle h, float* ms_out) {
    if (!h || !ms_out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    if (!h->timed) return fail(SPTAG_B200_FAIL, "no search has run on this handle yet");
    DeviceGuard guard(h->device);
    CUDA_OK(cudaEventSynchronize(h->ev_stop));
    CUDA_OK(cudaEventElapsedTime(ms_out, h->ev_start, h->ev_stop));
    return SPTAG_B200_SUCCESS;
}

int32_t sptag_b200_num_vectors(sptag_b200_handle h) { return h ? h->n : 0; }
int32_t sptag_b200_dim(sptag_b200_handle h) { return h ? h->dim : 0; }
int32_t sptag_b200_value_type(sptag_b200_handle h) { return h ? h->value_type : -1; }
int32_t sptag_b200_metric(sptag_b200_handle h) { return h ? h->metric : -1; }
int32_t sptag_b200_algo(sptag_b200_handle h) { return h ? h->algo : -1; }

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Index mutation: AddIndex / DeleteIndex / SaveIndex (BKTIndex.cpp:876-970, KDTIndex.cpp:602-696, VectorIndex.cpp)
// ---------------------------------------------------------------------------------------------------------------
namespace {

// Grow `b` to at least `need` bytes keeping its first `keep` bytes; capacity grows by half at least, so a stream of
// small adds reallocates O(log n) times.  The caller has waited for every launch that reads the buffer.
int grow_keep(DeviceBuffer& b, size_t need, size_t keep) {
    if (need <= b.bytes) return 0;
    size_t cap = std::max(need, b.bytes + b.bytes / 2);
    void* p = nullptr;
    if (cudaMalloc(&p, cap) != cudaSuccess) {
        cudaGetLastError();
        cap = need;
        cudaError_t e = cudaMalloc(&p, cap);
        if (e != cudaSuccess) return fail(SPTAG_B200_MEMORY_OVERFLOW, "cudaMalloc(%zu) failed: %s", cap, cudaGetErrorString(e));
    }
    if (keep && b.ptr) {
        cudaError_t e = cudaMemcpy(p, b.ptr, std::min(keep, b.bytes), cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) {
            cudaFree(p);
            return fail(SPTAG_B200_FAIL, "device copy on growth failed: %s", cudaGetErrorString(e));
        }
    }
    b.release();
    b.ptr = p;
    b.bytes = cap;
    return 0;
}

// A mutation runs under h->mu after every kernel already enqueued on the handle (searches of other threads hold the
// lock only while they enqueue; each records its scratch set's ev_done), so a concurrent search sees all of it or none.
int quiesce(sptag_b200_index* h) {
    for (auto& sc : h->scratch)
        if (sc.used) CUDA_OK(cudaEventSynchronize(sc.ev_done));
    return 0;
}

int check_mutable(const sptag_b200_index* h) {
    if (h->open_iterators > 0)
        return fail(SPTAG_B200_FAIL, "%d iterator(s) of this index are open: their per-query visited sets are sized to the "
                                     "current vector count; close them before changing the index", h->open_iterators);
    return 0;
}

// The tombstone map exists from the first deletion on (sptag_b200_load / _create allocate it only for a non-empty one)
// (sptag_b200_add grows an existing map with the vectors)
int ensure_deleted_map(sptag_b200_index* h) {
    if (h->d_deleted.ptr) return 0;
    if (int rc = h->d_deleted.ensure((size_t)h->n)) return rc;
    CUDA_OK(cudaMemset(h->d_deleted.ptr, 0, (size_t)h->n));
    return 0;
}

int value_base(int vt) {  // COMMON::Utils::GetBase<T> (CommonUtils.h:54-59)
    switch (vt) {
    case SPTAG_B200_VT_INT8: return 127;
    case SPTAG_B200_VT_UINT8: return 255;
    case SPTAG_B200_VT_INT16: return 32767;
    }
    return 1;
}

bool write_all(FILE* f, const void* p, size_t bytes) { return bytes == 0 || std::fwrite(p, 1, bytes, f) == bytes; }

const char* value_type_name(int vt) {
    switch (vt) {
    case SPTAG_B200_VT_INT8: return "Int8";
    case SPTAG_B200_VT_UINT8: return "UInt8";
    case SPTAG_B200_VT_INT16: return "Int16";
    }
    return "Float";
}

}  // namespace

extern "C" {

int sptag_b200_delete(sptag_b200_handle h, const int32_t* ids, int32_t num, int32_t* out_codes) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num < 0 || (num > 0 && !ids)) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (num == 0) return SPTAG_B200_SUCCESS;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    if (int rc = check_mutable(h)) return rc;
    if (int rc = quiesce(h)) return rc;
    if (int rc = ensure_deleted_map(h)) return rc;
    // ids as search returns them: the shard offset comes off first
    std::vector<int32_t> local((size_t)num);
    for (int i = 0; i < num; ++i) {
        const long long v = (long long)ids[i] - h->id_offset;
        local[(size_t)i] = (v < 0 || v >= h->n) ? -1 : (int32_t)v;  // out of range: VectorNotFound
    }
    if (int rc = h->d_mut.ensure((size_t)num * 8 + 16)) return rc;
    if (int rc = h->d_first.ensure((size_t)h->n * 4)) return rc;
    int* d_ids = (int*)h->d_mut.ptr;
    int* d_codes = d_ids + num;
    int* d_count = d_codes + num;
    cudaStream_t stream = nullptr;
    CUDA_OK(cudaMemcpyAsync(d_ids, local.data(), (size_t)num * 4, cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaMemsetAsync(d_count, 0, 4, stream));
    const unsigned blocks = (unsigned)((num + 255) / 256);
    tombstone_reset_kernel<<<blocks, 256, 0, stream>>>(d_ids, num, h->n, (int*)h->d_first.ptr);
    tombstone_order_kernel<<<blocks, 256, 0, stream>>>(d_ids, num, h->n, (int*)h->d_first.ptr);
    tombstone_apply_kernel<<<blocks, 256, 0, stream>>>(d_ids, num, h->n, (const int*)h->d_first.ptr,
                                                       (signed char*)h->d_deleted.ptr, d_codes, d_count);
    g_launches += 3;
    CUDA_OK(cudaGetLastError());
    int added = 0;
    CUDA_OK(cudaMemcpyAsync(&added, d_count, 4, cudaMemcpyDeviceToHost, stream));
    if (out_codes) CUDA_OK(cudaMemcpyAsync(out_codes, d_codes, (size_t)num * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    h->num_deleted += added;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_delete_vectors(sptag_b200_handle h, const void* vectors, int32_t num) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num < 0 || (num > 0 && !vectors)) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (h->q_type != 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "DeleteIndex(vectors) on a quantized index is not built");
    if (num == 0) return SPTAG_B200_SUCCESS;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    if (int rc = check_mutable(h)) return rc;
    const int k = h->cef;
    if (k < 1 || k > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "CEF = %d outside [1, 2048]", k);
    if (int rc = quiesce(h)) return rc;
    if (int rc = ensure_deleted_map(h)) return rc;
    const size_t qb = query_bytes(h);
    const size_t qoff = round_up((size_t)k * 8 + 16, 256);
    if (int rc = h->d_mut.ensure(qoff + (size_t)num * qb)) return rc;
    int* d_ids = (int*)h->d_mut.ptr;
    float* d_dists = (float*)(d_ids + k);
    int* d_count = (int*)(d_dists + k);
    unsigned char* d_q = (unsigned char*)h->d_mut.ptr + qoff;
    cudaStream_t stream = nullptr;
    CUDA_OK(cudaMemcpyAsync(d_q, vectors, (size_t)num * qb, cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaMemsetAsync(d_count, 0, 4, stream));
    // SearchIndex(query) per vector (the index's MaxCheck, searchDeleted = false, K = CEF), then DeleteIndex of every
    // result closer than 1e-6 -- in vector order, each search seeing the tombstones of the ones before it
    CallOpts opts;
    opts.search_deleted = 0;
    opts.tombstones_live = true;
    for (int i = 0; i < num; ++i) {
        if (int rc = search_device_impl(h, d_q + (size_t)i * qb, 1, k, d_ids, d_dists, nullptr, stream, false, opts)) {
            cudaStreamSynchronize(stream);
            return rc;
        }
        tombstone_close_kernel<<<1, 32, 0, stream>>>(d_ids, d_dists, k, h->id_offset, (signed char*)h->d_deleted.ptr, d_count);
        g_launches++;
        CUDA_OK(cudaGetLastError());
    }
    int added = 0;
    CUDA_OK(cudaMemcpyAsync(&added, d_count, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    h->num_deleted += added;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_add(sptag_b200_handle h, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                   int32_t* out_first_id) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!vectors || num <= 0 || dim <= 0) return fail(SPTAG_B200_EMPTY_DATA, "no vectors to add");
    if (dim != h->dim) return fail(SPTAG_B200_DIMENSION_MISMATCH, "vectors have %d dimensions, the index %d", dim, h->dim);
    if (h->q_type != 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "AddIndex on a quantized index is not built");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    if (int rc = check_mutable(h)) return rc;
    const int k = h->add_cef + 1;
    if (k < 1 || k > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "AddCEF = %d outside [0, 2047]", h->add_cef);
    if ((long long)h->n + num > 0x7fffffffLL - 1) return fail(SPTAG_B200_MEMORY_OVERFLOW, "more than 2^31 - 2 vectors");
    if (int rc = quiesce(h)) return rc;
    cudaStream_t stream = nullptr;
    const int old_n = h->n, new_n = h->n + num;
    const size_t rs = h->row_stride, row_bytes = (size_t)h->dim * value_size(h->value_type);
    // Dataset::AddBatch (Dataset.h:127-144): append the rows (plus the spare padded row), new graph rows all -1, new
    // tombstone bytes 0
    if (int rc = grow_keep(h->d_vectors, ((size_t)new_n + 1) * rs, (size_t)old_n * rs)) return rc;
    CUDA_OK(cudaMemsetAsync((unsigned char*)h->d_vectors.ptr + (size_t)old_n * rs, 0, ((size_t)num + 1) * rs, stream));
    CUDA_OK(cudaMemcpy2DAsync((unsigned char*)h->d_vectors.ptr + (size_t)old_n * rs, rs, vectors, row_bytes, row_bytes,
                              (size_t)num, cudaMemcpyHostToDevice, stream));
    const size_t grow_row = (size_t)h->degree * 4;
    if (int rc = grow_keep(h->d_graph, (size_t)new_n * grow_row, (size_t)old_n * grow_row)) return rc;
    CUDA_OK(cudaMemsetAsync((unsigned char*)h->d_graph.ptr + (size_t)old_n * grow_row, 0xff, (size_t)num * grow_row, stream));
    if (h->d_deleted.ptr) {
        if (int rc = grow_keep(h->d_deleted, (size_t)new_n, (size_t)old_n)) return rc;
        CUDA_OK(cudaMemsetAsync((unsigned char*)h->d_deleted.ptr + old_n, 0, (size_t)num, stream));
    }
    unsigned char* dv = (unsigned char*)h->d_vectors.ptr;
    if (h->metric == SPTAG_B200_METRIC_COSINE && !normalized) {
        const unsigned blocks = (unsigned)((num + 127) / 128);
        const int base = value_base(h->value_type);
        with_elem(h, [&](auto el) {
            normalize_rows_kernel<typename decltype(el)::type><<<blocks, 128, 0, stream>>>(dv, rs, old_n, num, h->dim, base);
        });
        g_launches++;
        CUDA_OK(cudaGetLastError());
    }
    h->n = new_n;
    // RefineNode(node, updateNeighbors = true, searchDeleted = true, AddCEF) for node = old_n .. new_n - 1, in order
    // (NeighborhoodGraph.h:535-561): each node's search sees the rows the nodes before it rebuilt and inserted into
    if (int rc = h->d_ids.ensure((size_t)k * 4)) return rc;
    if (int rc = h->d_dists.ensure((size_t)k * 4)) return rc;
    int* d_ids = (int*)h->d_ids.ptr;
    float* d_dists = (float*)h->d_dists.ptr;
    int* graph = (int*)h->d_graph.ptr;
    CallOpts ropts;
    ropts.max_check = h->max_check_refine;  // RefineSearchIndex: workSpace->Reset(MaxCheckForRefineGraph, AddCEF + 1)
    ropts.search_deleted = 1;
    ropts.refine_query_stride = rs;
    const int deg = h->degree;
    const unsigned ins_blocks = (unsigned)((k + 3) / 4);
    for (int node = old_n; node < new_n; ++node) {
        if (int rc = search_device_impl(h, dv + (size_t)node * rs, 1, k, d_ids, d_dists, nullptr, stream, /*refine=*/true, ropts)) {
            cudaStreamSynchronize(stream);
            h->n = node;  // keep the rows that are linked in (no row points to a node that was not inserted)
            return rc;
        }
        int* row = graph + (size_t)node * deg;
        with_metric_elem(h, [&](auto cos, auto el) {
            rebuild_neighbors_kernel<cos, el><<<1, 32, (size_t)deg * 4, stream>>>(dv, rs, h->dim, node, 1, d_ids, d_dists, k,
                                                                                 deg, h->rng_factor, row, h->simd_width);
            insert_neighbors_kernel<cos, el><<<ins_blocks, 128, 0, stream>>>(dv, rs, h->dim, node, d_ids, d_dists, k, graph,
                                                                             deg, h->simd_width);
        });
        g_launches += 2;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) {
            cudaStreamSynchronize(stream);
            h->n = node;
            return fail(SPTAG_B200_FAIL, "AddIndex step of node %d failed: %s", node, cudaGetErrorString(e));
        }
    }
    CUDA_OK(cudaStreamSynchronize(stream));
    if (out_first_id) *out_first_id = old_n + h->id_offset;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_save(sptag_b200_handle h, const char* folder) {
    if (!h) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!folder) return fail(SPTAG_B200_LACK_OF_INPUTS, "null folder");
    if (h->q_type != 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "saving a quantized index is not built (the quantizer blob is not kept)");
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    if (int rc = quiesce(h)) return rc;
    const std::string dir(folder);
    mkdir(dir.c_str(), 0777);  // like SaveIndex, which creates the folder; an existing one is reused
    const size_t n = (size_t)h->n, rs = h->row_stride, row_bytes = (size_t)h->dim * value_size(h->value_type);
    const bool bkt = (h->algo == SPTAG_B200_ALGO_BKT);
    const size_t node_sz = bkt ? 12 : 16;
    std::vector<unsigned char> vec(n * row_bytes), nodes(((size_t)h->node_count + 1) * node_sz), del(n, 0);
    std::vector<int32_t> graph(n * (size_t)h->degree), starts((size_t)h->tree_num);
    CUDA_OK(cudaMemcpy2D(vec.data(), row_bytes, h->d_vectors.ptr, rs, row_bytes, n, cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(graph.data(), h->d_graph.ptr, graph.size() * 4, cudaMemcpyDeviceToHost));
    // the node array on the device ends with the (-1, -1, -1) sentinel LoadTrees appends (BKTree.h:662); the reference
    // saves its loaded array, sentinel included
    CUDA_OK(cudaMemcpy(nodes.data(), h->d_nodes.ptr, nodes.size(), cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(starts.data(), h->d_tree_starts.ptr, starts.size() * 4, cudaMemcpyDeviceToHost));
    if (h->d_deleted.ptr) CUDA_OK(cudaMemcpy(del.data(), h->d_deleted.ptr, n, cudaMemcpyDeviceToHost));
    int32_t node_count = h->node_count;
    if (bkt) {
        int32_t last;
        memcpy(&last, nodes.data() + (size_t)(node_count - 1) * node_sz, 4);
        if (last != -1) node_count++;
    }
    auto open_w = [&](const char* name) { return std::fopen((dir + "/" + name).c_str(), "wb"); };
    bool ok = true;
    // vectors.bin (Dataset.h:146-180), graph.bin (NeighborhoodGraph.h:606-615), tree.bin (BKTree.h:635-645 /
    // KDTree.h:123-133), deletes.bin (Labelset.h:78-83: count, then Dataset<int8> n x 1)
    if (FILE* f = open_w("vectors.bin")) {
        const int32_t hdr[2] = {h->n, h->dim};
        ok = write_all(f, hdr, 8) && write_all(f, vec.data(), vec.size()) && ok;
        ok = std::fclose(f) == 0 && ok;
    } else ok = false;
    if (FILE* f = open_w("graph.bin")) {
        const int32_t hdr[2] = {h->n, h->degree};
        ok = write_all(f, hdr, 8) && write_all(f, graph.data(), graph.size() * 4) && ok;
        ok = std::fclose(f) == 0 && ok;
    } else ok = false;
    if (FILE* f = open_w("tree.bin")) {
        ok = write_all(f, &h->tree_num, 4) && write_all(f, starts.data(), starts.size() * 4) && write_all(f, &node_count, 4) &&
             write_all(f, nodes.data(), (size_t)node_count * node_sz) && ok;
        ok = std::fclose(f) == 0 && ok;
    } else ok = false;
    if (FILE* f = open_w("deletes.bin")) {
        const int32_t hdr[3] = {h->num_deleted, h->n, 1};
        ok = write_all(f, hdr, 12) && write_all(f, del.data(), del.size()) && ok;
        ok = std::fclose(f) == 0 && ok;
    } else ok = false;
    // indexloader.ini as VectorIndex::SaveIndexConfig writes it (VectorIndex.cpp:197-222): [Index] with the algorithm and
    // value type, then the parameters; the reference's LoadIndex and sptag_b200_load both read it
    if (FILE* f = open_w("indexloader.ini")) {
        const char* metric = h->metric == SPTAG_B200_METRIC_L2 ? "L2" : (h->metric == SPTAG_B200_METRIC_COSINE ? "Cosine" : "InnerProduct");
        const int w = std::fprintf(
            f,
            "[Index]\nIndexAlgoType=%s\nValueType=%s\n\nTreeFilePath=tree.bin\nGraphFilePath=graph.bin\nVectorFilePath=vectors.bin\n"
            "DeleteVectorFilePath=deletes.bin\nNeighborhoodSize=%d\nCEF=%d\nAddCEF=%d\nMaxCheckForRefineGraph=%d\nRNGFactor=%f\n"
            "DistCalcMethod=%s\nMaxCheck=%d\nThresholdOfNumberOfContinuousNoBetterPropagation=%d\nNumberOfInitialDynamicPivots=%d\n"
            "NumberOfOtherDynamicPivots=%d\n",
            bkt ? "BKT" : "KDT", value_type_name(h->value_type), h->degree, h->cef, h->add_cef, h->max_check_refine,
            h->rng_factor, metric, h->max_check, h->no_better_threshold, h->initial_pivots, h->other_pivots);
        ok = w > 0 && std::fclose(f) == 0 && ok;
    } else ok = false;
    if (!ok) return fail(SPTAG_B200_FAIL, "cannot write the index files in %s", folder);
    return SPTAG_B200_SUCCESS;
}

int32_t sptag_b200_num_deleted(sptag_b200_handle h) {
    if (!h) return 0;
    std::lock_guard<std::mutex> lock(h->mu);  // written by the delete calls under the same lock
    return h->num_deleted;
}

}  // extern "C"
