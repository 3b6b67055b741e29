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
#include "multi_scan.h"
#include "spann_build.h"
#include "spann_scan.h"

#include <algorithm>
#include <atomic>
#include <cctype>
#include <cerrno>
#include <cfloat>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <cxxabi.h>
#include <deque>
#include <dlfcn.h>
#include <fcntl.h>
#include <fstream>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <strings.h>
#include <sys/stat.h>
#include <sstream>
#include <string>
#include <thread>
#include <type_traits>
#include <unistd.h>
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

// The two staging sets of a handle's host-buffer calls, each with its own lock and stream, so that two callers overlap.
// Buffers: what a set holds besides them.  The streams go with the pool, which its owner destroys with the handle's
// device current.
template <typename Buffers>
struct StagingPool {
    struct Set : Buffers {
        std::mutex mu;
        cudaStream_t stream = nullptr;
    };
    Set sets[2];
    std::atomic<unsigned> rr{0};
    ~StagingPool() {
        for (Set& s : sets)
            if (s.stream) cudaStreamDestroy(s.stream);
    }
    bool create_streams() {
        for (Set& s : sets)
            if (cudaStreamCreate(&s.stream) != cudaSuccess) return false;
        return true;
    }
    // A set of the caller's own for the whole call: the one that is free, else wait for the next in turn
    Set* acquire(std::unique_lock<std::mutex>& lock) {
        for (Set& s : sets) {
            std::unique_lock<std::mutex> l(s.mu, std::try_to_lock);
            if (l.owns_lock()) {
                lock = std::move(l);
                return &s;
            }
        }
        Set* s = &sets[rr.fetch_add(1) & 1u];
        lock = std::unique_lock<std::mutex>(s->mu);
        return s;
    }
};

// One set per query in the hashed visited-set format (vhash_home), grown while its owner runs: the visited sets of
// iterators on hash tables, the SPANN iterators' dedupers and the multi-index scan's seen sets.  The kernels find query
// q's set at d_tables[q] and its size and fill in vbits / vfill of q's IterState in the owner's array.  A set is a table
// of 2^bits[q] entries, or (bits 0) a bitmap of bitmap_words words once a table would be larger.  The sets live in bufs:
// one buffer at open, one per growth round; a buffer is freed when no query's set lives in it any more.
struct QueryTables {
    static constexpr size_t kNoBitmap = 0;  // bitmap_words of sets that stay tables however large they grow
    size_t bitmap_words = kNoBitmap;
    IterState* state = nullptr;  // the owner's per-query IterState array (device)
    std::vector<int> bits, buf;  // per query: log2 of its table's entries (0: a bitmap), the index of its buffer
    std::vector<unsigned int*> set;
    std::vector<DeviceBuffer> bufs;
    std::vector<int> refs;  // per buffer: the queries whose sets live in it
    DeviceBuffer d_tables, d_jobs;

    // nq empty tables of 2^bits0 entries, and st0 with vbits = bits0 written to each of the nq IterStates at st.  Blocks
    // until done.
    int open(size_t nq, int bits0, size_t bitmap_words_, IterState* st, IterState st0 = IterState()) {
        const size_t entries = (size_t)1 << bits0;
        bitmap_words = bitmap_words_;
        state = st;
        bufs.emplace_back();
        refs.push_back((int)nq);
        if (int rc = bufs[0].ensure(nq * entries * 4)) return rc;
        if (int rc = d_tables.ensure(nq * sizeof(unsigned int*))) return rc;
        bits.assign(nq, bits0);
        buf.assign(nq, 0);
        set.resize(nq);
        for (size_t q = 0; q < nq; ++q) set[q] = (unsigned int*)bufs[0].ptr + q * entries;
        st0.vbits = bits0;
        const std::vector<IterState> sts(nq, st0);
        CUDA_OK(cudaMemset(bufs[0].ptr, 0, bufs[0].bytes));
        CUDA_OK(cudaMemcpy(d_tables.ptr, set.data(), nq * sizeof(unsigned int*), cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(state, sts.data(), nq * sizeof(IterState), cudaMemcpyHostToDevice));
        return 0;
    }

    // Move the sets of queries qs[i] to one new, zeroed buffer: tables of 2^new_bits[i] entries, or bitmaps where such a
    // table would be larger than one.  keep: the ids are carried over; otherwise the sets start empty (the query's call
    // runs again from the start).  Blocks until the move is done.
    int grow(const std::vector<unsigned>& qs, const std::vector<int>& new_bits, bool keep, cudaStream_t stream) {
        std::vector<IterGrowJob> jobs(qs.size());
        size_t words = 0;
        for (size_t i = 0; i < qs.size(); ++i) {
            int b = new_bits[i];
            if (b && bitmap_words != kNoBitmap && ((size_t)1 << b) > bitmap_words) b = 0;  // a bitmap, and stays one
            jobs[i].new_bits = b;
            jobs[i].new_set = (unsigned int*)(words * 4);  // offset until the buffer exists
            words += b ? ((size_t)1 << b) : bitmap_words;
        }
        DeviceBuffer nbuf;
        if (int rc = nbuf.ensure(words * 4)) return rc;
        CUDA_OK(cudaMemsetAsync(nbuf.ptr, 0, nbuf.bytes, stream));
        for (size_t i = 0; i < qs.size(); ++i) {
            const unsigned q = qs[i];
            jobs[i].new_set = (unsigned int*)((char*)nbuf.ptr + (size_t)jobs[i].new_set);
            jobs[i].old_set = set[q];
            jobs[i].q = (int)q;
            jobs[i].old_bits = bits[q];
            jobs[i].keep = keep ? 1 : 0;
        }
        if (int rc = d_jobs.ensure(jobs.size() * sizeof(IterGrowJob))) return rc;
        CUDA_OK(cudaMemcpyAsync(d_jobs.ptr, jobs.data(), jobs.size() * sizeof(IterGrowJob), cudaMemcpyHostToDevice, stream));
        iter_grow_kernel<<<(unsigned)jobs.size(), 32, 0, stream>>>((const IterGrowJob*)d_jobs.ptr, (unsigned int**)d_tables.ptr,
                                                                   (int*)state);
        g_launches++;
        CUDA_OK(cudaGetLastError());
        CUDA_OK(cudaStreamSynchronize(stream));
        const int nb = (int)bufs.size();
        for (size_t i = 0; i < qs.size(); ++i) {
            const unsigned q = qs[i];
            if (--refs[buf[q]] == 0) bufs[buf[q]].release();
            buf[q] = nb;
            bits[q] = jobs[i].new_bits;
            set[q] = jobs[i].new_set;
        }
        bufs.push_back(std::move(nbuf));
        refs.push_back((int)qs.size());
        return 0;
    }

    // Read the header of the device list d_list (kIterListHeader layout) into hdr, and double the sets of the hdr[0]
    // queries it lists.  Blocks.
    int double_listed(const unsigned int* d_list, unsigned* hdr, bool keep, cudaStream_t stream) {
        CUDA_OK(cudaMemcpyAsync(hdr, d_list, kIterListHeader * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (hdr[0] == 0) return 0;
        std::vector<unsigned> qs(hdr[0]);
        CUDA_OK(cudaMemcpy(qs.data(), d_list + kIterListHeader, qs.size() * 4, cudaMemcpyDeviceToHost));
        std::vector<int> nb(qs.size());
        for (size_t i = 0; i < qs.size(); ++i) nb[i] = bits[qs[i]] + 1;
        return grow(qs, nb, keep, stream);
    }

    size_t bytes() const {
        size_t b = 0;
        for (const DeviceBuffer& v : bufs) b += v.bytes;
        return b;
    }
};

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
    int bfs = 0;  // EnableBfs (BKT only): != 0 seeds each tree breadth-first (BKTree.h:703-758)
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
    // -1 auto (the bitmap unless its per-slot allocation fails), 0 bitmap, 1 hashed set per slot
    int visited_set = -1;
    int visited_hash_entries = 0;  // table entries per slot, 0 = 2^(bits(max(MaxCheck, MaxCheckForRefineGraph)) + 2)
    // B200.RowSketch: -1 auto (float BKT rows of 2 KB or more, unless the sketches do not fit in HBM), 0 off, 1 on.
    // d_sketch holds the sketches of rows [0, sketch_n) (search_kernels.cuh warp_sketch); it is a function of the rows, so
    // it is rebuilt, never saved.  d_skipped: the candidates whose rows the searches of this handle did not fetch.
    int row_sketch = -1;
    DeviceBuffer d_sketch, d_skipped;
    int sketch_n = 0;
    bool sketch_unfit = false;  // auto: the allocation failed for lack of memory; cleared by setting B200.RowSketch
    std::atomic<int> last_visited_overflows{0};  // queries the hashed set handed to the re-run, last blocking search
    // iterators: -1 auto (the bitmaps unless their allocation fails), 0 bitmap, 1 a growing hash table per query
    int iter_visited_set = -1;
    int iter_hash_entries = 0;  // initial table entries per query, 0 = 2^(bits(max(MaxCheck, MaxCheckForRefineGraph)) + 2)
    int max_dup = -1;           // largest duplicate group of the tree (the tree never changes); -1 = not computed yet
    // the last iterator call: suspensions at a step top / before a SearchTrees pop, tables grown, visited-set bytes held
    long last_iter_susp_step = 0, last_iter_susp_trees = 0, last_iter_growths = 0, last_iter_visited_bytes = 0;
    // host stub of the last search, sketch::, bfs:: or iterator kernel this handle launched (B200.LastSearchKernel)
    const void* last_search_kernel = nullptr;
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
    // Hashed visited set: d_vhash holds the per-slot tables, d_vlog their clear logs, d_overflow the abandoned queries, and
    // d_visited only the bitmaps of the re-run grid.
    struct Scratch {
        DeviceBuffer d_visited, d_ng_spill, d_spt_spill, d_counter, d_vlog, d_topk, d_codes, d_adc, d_vhash, d_overflow;
        bool visited_clean = false;   // the whole d_visited buffer is known to be zero
        // auto visited set: the size of a per-slot bitmap allocation that failed for lack of memory (0 = none).  Launches
        // that need at least as much skip the attempt (set 0 binds the hashed set, set 1 defers to set 0), so the failed
        // cudaMalloc and the free that precedes it are not repeated per call.  Cleared by setting B200.VisitedSet.
        size_t bitmap_unfit = 0;
        cudaEvent_t ev_done = nullptr;  // recorded after every kernel that uses this set; the next launch on it waits
        cudaStream_t last_stream = nullptr;
        bool used = false;
        void release() {  // early free: set 1 did not fit in HBM and the launch falls back to set 0
            d_visited.release(); d_ng_spill.release(); d_spt_spill.release(); d_counter.release(); d_vlog.release();
            d_topk.release(); d_codes.release(); d_adc.release(); d_vhash.release(); d_overflow.release();
        }
        size_t bytes() const {
            return d_visited.bytes + d_ng_spill.bytes + d_spt_spill.bytes + d_counter.bytes + d_vlog.bytes + d_topk.bytes +
                   d_codes.bytes + d_adc.bytes + d_vhash.bytes + d_overflow.bytes;
        }
    } scratch[2];
    DeviceBuffer d_ids, d_dists;                      // refine pass: per-batch result lists
    // Host-buffer entry points: two staging sets, each with its own stream, so that one caller's H2D / D2H overlaps
    // another caller's kernel (the kernels themselves share the per-slot scratch and are ordered by ev_done)
    struct StagingBuffers {
        DeviceBuffer d_queries, d_ids, d_dists, d_stats, d_filter, d_overflows;
    };
    StagingPool<StagingBuffers> staging;
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
    // Hashed visited sets (B200.IteratorVisitedSet): tables that grow, each turning into a bitmap of visited_words words
    // once it would outgrow one
    bool hashed = false;
    int margin = 0;  // degree + largest duplicate group + 1 (IterVisited::margin)
    QueryTables tables;
    DeviceBuffer d_resume, d_susp[2];
    size_t visited_bytes() const { return d_visited.bytes + tables.bytes(); }
};

namespace {

int heap_lastlevel(int size) {
    // Heap::Resize: lastlevel = int(pow(2.0, floor(log2((float)size))))  (Heap.h:24)
    return (int)std::pow(2.0, std::floor(std::log2((float)size)));
}

// EnableBfs is in force: a BKT handle with a non-zero value.  Its searches take the bfs:: kernels.
bool bfs_seeding(const sptag_b200_index* h) { return h->algo == SPTAG_B200_ALGO_BKT && h->bfs != 0; }

template <bool BFS>
SearchKernelFn pick_kernel_seeded(const sptag_b200_index* h, int mres_cap, int slots) {
    const bool kdt = (h->algo == SPTAG_B200_ALGO_KDT);
    const bool cosine = (h->metric != SPTAG_B200_METRIC_L2);
    if (h->q_type != 0) return pick_pq_kernel<BFS>(mres_cap);  // quantized: BKT + L2 only (PQQuantizer.h:130-136)
    if (h->value_type == SPTAG_B200_VT_INT8) return pick_int_kernel<BFS, 1>(cosine, mres_cap, kdt);
    if (h->value_type == SPTAG_B200_VT_UINT8) return pick_int_kernel<BFS, 2>(cosine, mres_cap, kdt);
    if (h->value_type == SPTAG_B200_VT_INT16) return pick_int_kernel<BFS, 3>(cosine, mres_cap, kdt);
    const int kdim = (h->simd_width == 16) ? h->dim : 0;  // the 128- / 768-d specialisations are AVX-512 trees
    return cosine ? pick_float_kernel<BFS, true>(kdim, mres_cap, kdt, slots)
                  : pick_float_kernel<BFS, false>(kdim, mres_cap, kdt, slots);
}

// The kernel instantiation for this index / parameter set (nullptr: unsupported m_Results capacity); the
// instantiations live in kern_*.cu (kernel_select.h)
SearchKernelFn pick_kernel(const sptag_b200_index* h, int mres_cap, int slots = 0, bool sketch = false) {
    if (sketch) {
        const int kdim = (h->simd_width == 16) ? h->dim : 0;
        return h->metric != SPTAG_B200_METRIC_L2 ? pick_sketch_kernel<true>(kdim, mres_cap) : pick_sketch_kernel<false>(kdim, mres_cap);
    }
    return bfs_seeding(h) ? pick_kernel_seeded<true>(h, mres_cap, slots) : pick_kernel_seeded<false>(h, mres_cap, slots);
}

// The ResultIterator::Next (Fn = IterateKernelFn) or SearchIndexIterativeFromNeareast first-call (NearestFirstKernelFn)
// kernel of an iterator step planned with parameters p (nullptr: unsupported m_Results capacity)
template <typename Fn>
Fn pick_iter_step_kernel(const sptag_b200_index* h, const SearchParams& p) {
    const bool cosine = h->metric != SPTAG_B200_METRIC_L2;
    return p.bfs ? pick_iter_kernel<Fn, true>(h->value_type, cosine, p.mres_cap)
                 : pick_iter_kernel<Fn, false>(h->value_type, cosine, p.mres_cap);
}

// The demangled name of a kernel's host launch stub without return type and parameter list, e.g.
// "sptag_b200::search_kernel<128, false, 16, false, false, 0, 20>".  A kernel of internal linkage (the SPANN posting
// kernels) has no exported stub symbol: its device name comes from the runtime instead, e.g.
// "sptag_b200::(anonymous namespace)::spann_scan_kernel<false, 2>".  Empty if neither knows the stub.
std::string kernel_name(const void* stub) {
    if (!stub) return std::string();
    Dl_info info;
    const char* mangled = nullptr;
    if (dladdr(stub, &info) && info.dli_sname && info.dli_saddr == stub)
        mangled = info.dli_sname;
    else if (cudaFuncGetName(&mangled, stub) != cudaSuccess || !mangled) {
        cudaGetLastError();
        return std::string();
    }
    int status = 0;
    char* d = abi::__cxa_demangle(mangled, nullptr, nullptr, &status);
    std::string s = (status == 0 && d) ? d : mangled;
    free(d);
    if (s.compare(0, 5, "void ") == 0) s.erase(0, 5);
    // the parameter list: the (...) that ends the name ("(anonymous namespace)" may come before it; template arguments
    // are integers and booleans only)
    if (!s.empty() && s.back() == ')') {
        size_t i = s.size(), depth = 0;
        while (i-- > 0) {
            if (s[i] == ')') ++depth;
            else if (s[i] == '(' && --depth == 0) break;
        }
        if (i < s.size()) s.erase(i);
    }
    return s;
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
    int* d_overflows = nullptr;  // device int: receives how many queries the hashed set handed to the re-run (bitmap: 0)
    bool sketch = false;         // the handle's row sketches cover every row: take the sketch:: kernel (search_device_impl)
    // device {count, query indices}: search only the listed queries of the batch (their results land at their own rows)
    const unsigned int* d_query_list = nullptr;
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

// log2 of a hashed visited set's entries: `entries` (B200.VisitedHashEntries, B200.IteratorVisitedHashEntries) rounded up
// to a power of two, or when it is 0 the reference's first-block size 2^(bits(max(MaxCheck, MaxCheckForRefineGraph)) +
// HashTableExponent 2) (WorkSpace.h:83-93) for `check` = that maximum.  At least 64 entries: a query stops inserting at
// half the capacity, and the last row chunk may add up to 31 ids past that, which must still find an empty position (the
// probes end only at one).
int vhash_log2_entries(int entries, int check) {
    int bits = 0;
    if (entries > 0) {
        while ((1 << bits) < entries) ++bits;
        return bits;
    }
    for (unsigned s = (unsigned)std::max(check, 1); s != 0; s >>= 1) ++bits;
    return std::min(std::max(bits + 2, 6), 30);
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
    p.bfs = bfs_seeding(h) ? h->bfs : 0;
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
    if (opts.sketch) {  // float rows: the PQ tables' slots are free (SearchParams)
        p.sketch = (const unsigned char*)h->d_sketch.ptr;
        p.rows_skipped = (unsigned long long*)h->d_skipped.ptr;
    }

    // ---- per-slot arena sizes ----
    p.visited_words = round_up(((size_t)h->n + 1 + 31) / 32, 4);
    // (even entry counts keep every slot's arena 16-byte aligned for the paired child loads)
    p.ng_spill_entries = round_up((size_t)std::min<long long>((long long)p.ng_length, (long long)h->n + 2) + 2, 2);
    p.spt_spill_entries = round_up((size_t)std::min<long long>((long long)p.spt_length, (long long)h->node_count + 2) + 2, 2);
    if (p.bfs) p.spt_spill_entries += 2 * kBfsHeapEntries;  // the two BFS heaps (WarpSearch::bfs_heap)
    const bool use_log = h->visited_log < 0 ? (p.visited_words * 4 > 256 * 1024) : (h->visited_log != 0);
    if (use_log) {
        const size_t entries = h->visited_log_entries > 0 ? (size_t)h->visited_log_entries
                                                          : (size_t)std::max(65536, 8 * alloc_check);
        p.vlog_entries = std::min(entries, (size_t)h->n + 2);
    }
    // hashed visited set, bound only by bind_scratch
    const int log2_entries = vhash_log2_entries(h->visited_hash_entries, alloc_check);
    p.vhash_mask = (1u << log2_entries) - 1u;
    p.vhash_shift = 32 - log2_entries;
    p.vhash_limit = INT_MAX;
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
    // must mirror WarpSearch::kFast (BFS seeding runs the generic-dimension kernels)
    const bool sketch = !pq && p.sketch != nullptr;  // the sketch:: kernels have no 128- or 768-d row path of their own
    const bool fast128 = !sketch && !p.bfs && !pq && h->value_type == SPTAG_B200_VT_FLOAT && h->dim == 128 && h->simd_width == 16;
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
    // the sketch pass stages up to 32 sketch rows at a time through the ring (768-d, 2 x 2 rows of 3 136 B: 16 of 784 B)
    if (sketch)
        p.sketch_batch = (int)std::min<size_t>(32, (size_t)stage_rows * stages * p.slot_stride / sketch_stride(h->dim));
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
        const bool query_in_regs_only = !p.bfs && !pq && h->value_type == SPTAG_B200_VT_FLOAT && h->algo == SPTAG_B200_ALGO_BKT &&
                                        h->dim == 768 && h->simd_width == 16;  // must mirror kRegsOnly in search_kernel
        off += query_in_regs_only ? 16 : round_up((size_t)h->dim * 4 + 16, 16);  // float query, or M row offsets for PQ
        if (sketch) {  // the query's sketch elements
            p.off_sketch = (int)off;
            off += sketch_elems(h->dim);
        }
        L.smem = round_up(off, 128);
        if (L.smem > h->smem_optin)
            return fail(SPTAG_B200_MEMORY_OVERFLOW, "shared memory per query slot %zu exceeds %zu", L.smem, h->smem_optin);

        L.kern = pick_kernel(h, p.mres_cap, want_slots, sketch);
        if (!L.kern)
            return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, K) = %d exceeds what this index type supports (2048; quantized: 1024)", p.mres_cap);
        // the opt-in maximum, one value for every call: handles that share an instantiation (a SPANN group's heads)
        // plan their launches on several threads, and a smaller value set between another thread's plan and its launch
        // would fail that launch
        CUDA_OK(cudaFuncSetAttribute((const void*)L.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_optin));
        // resident single-warp CTAs per SM allowed by registers + shared memory for this instantiation
        int fit = 0;
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, (const void*)L.kern, 32, L.smem));
        if (fit < 1) return fail(SPTAG_B200_MEMORY_OVERFLOW, "search kernel does not fit on an SM (smem %zu)", L.smem);
        int per_sm = h->queries_per_sm;
        if (per_sm <= 0) per_sm = fit;  // the kernel is latency-bound per warp: fill the SM
        // 3 KB rows (HBM-bound): 11-12 slots, with larger queue heads, were the fastest of 10-18 on an H100 (DESIGN.md §5);
        // with the sketch pass staged through the ring, 11 slots beat 12 by 2.5 % on C2 (DESIGN.md §5)
        if (h->queries_per_sm <= 0 && big_rows) per_sm = std::min(per_sm, sketch ? 11 : 12);
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
    L.p.nq = nq;
    return lay_out(h, nq, L);
}

// Grid of the launch that re-runs, on the bitmap, the queries a hashed-set launch abandoned: one slot per SM
int rerun_grid(const sptag_b200_index* h, int nq) { return std::max(1, std::min(nq, h->num_sms)); }
constexpr int kRerunCounter = 32;  // the re-run's work counter: word 32 of the set's 256-byte counter block

// Point the launch at scratch set `set`, allocated for every resident slot (grown, never shrunk).  The visited set is
// the bitmap per slot, or the hashed set (B200.VisitedSet = 1, or auto when the bitmaps do not fit in HBM).  L.p is
// changed only on success.  Caller holds h->mu.
int bind_scratch(sptag_b200_index* h, SearchLaunch& L, int set) {
    sptag_b200_index::Scratch& sc = h->scratch[set];
    SearchParams p = L.p;
    const size_t alloc_slots = (size_t)h->num_sms * L.per_sm;
    const size_t bitmap_bytes = alloc_slots * p.visited_words * 4;
    bool hashed = h->visited_set == 1;
    if (!hashed && h->visited_set < 0 && sc.bitmap_unfit != 0 && bitmap_bytes >= sc.bitmap_unfit) {
        // auto, and a bitmap this large did not fit before: set 1 defers to set 0 (search_device_impl), set 0 is hashed
        if (set != 0) return fail(SPTAG_B200_MEMORY_OVERFLOW, "visited bitmaps of %zu bytes do not fit", bitmap_bytes);
        hashed = true;
    } else if (!hashed) {
        const size_t before = sc.d_visited.bytes;
        if (int rc = sc.d_visited.ensure(bitmap_bytes)) {
            if (h->visited_set == 0 || cudaGetLastError() != cudaErrorMemoryAllocation) return rc;
            // auto: the per-slot bitmaps do not fit (the failed cudaMalloc's error is cleared above).  Set 1 lets the launch
            // run behind set 0 as before; set 0 binds the hashed set.
            sc.bitmap_unfit = bitmap_bytes;
            if (set != 0) return rc;
            hashed = true;
        }
        if (sc.d_visited.bytes != before) sc.visited_clean = false;
    }
    if (hashed) {
        const size_t entries = (size_t)p.vhash_mask + 1;
        p.vhash_limit = (int)(entries / 2);
        p.vlog_entries = (size_t)p.vhash_limit + 32;  // a query stops inserting at the limit; one row chunk may cross it
        const size_t before = sc.d_vhash.bytes;
        if (int rc = sc.d_vhash.ensure(alloc_slots * entries * 4)) return rc;
        if (sc.d_vhash.bytes != before) CUDA_OK(cudaMemset(sc.d_vhash.ptr, 0, sc.d_vhash.bytes));  // queries leave it empty
        if (int rc = sc.d_vlog.ensure(alloc_slots * p.vlog_entries * 4)) return rc;
        if (int rc = sc.d_overflow.ensure(((size_t)p.nq + 1) * 4)) return rc;
        if (int rc = sc.d_visited.ensure((size_t)rerun_grid(h, p.nq) * p.visited_words * 4)) return rc;
        sc.visited_clean = false;  // the re-run clears its bitmap per query
        p.vhash = (unsigned int*)sc.d_vhash.ptr;
        p.vlog = (unsigned int*)sc.d_vlog.ptr;
        p.overflow = (unsigned int*)sc.d_overflow.ptr;
    } else if (p.vlog_entries) {
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
    L.p = p;
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

// B200.RowSketch applies to this handle: float rows searched by the BKT kernels without breadth-first seeding
bool sketch_applies(const sptag_b200_index* h) {
    return h->value_type == SPTAG_B200_VT_FLOAT && h->q_type == 0 && h->algo == SPTAG_B200_ALGO_BKT && !bfs_seeding(h);
}
// Whether this handle's searches take the sketch:: kernels, with the sketches of the rows that have none yet (a new
// handle's, or the rows sptag_b200_add appended) built first.  Blocks until they are built: a search on another stream
// may follow.  Auto turns itself off when the array does not fit.  Caller holds h->mu.
int ensure_sketch(sptag_b200_index* h, cudaStream_t stream, bool& on) {
    on = false;
    if (!sketch_applies(h) || h->row_sketch == 0 || (h->row_sketch < 0 && (h->row_stride < 2048 || h->sketch_unfit))) return 0;
    const size_t stride = sketch_stride(h->dim), need = ((size_t)h->n + 1) * stride;
    if (need > h->d_sketch.bytes) {
        h->sketch_n = 0;
        if (int rc = h->d_sketch.ensure(std::max(need, h->d_sketch.bytes + h->d_sketch.bytes / 2))) {
            if (h->row_sketch > 0 || cudaGetLastError() != cudaErrorMemoryAllocation) return rc;
            h->sketch_unfit = true;
            return 0;
        }
    }
    if (!h->d_skipped.ptr) {
        if (int rc = h->d_skipped.ensure(8)) return rc;
        CUDA_OK(cudaMemset(h->d_skipped.ptr, 0, 8));
    }
    h->sketch_n = std::min(h->sketch_n, h->n);
    if (h->sketch_n < h->n) {
        const int num = h->n - h->sketch_n;
        row_sketch_kernel<<<(unsigned)((num + 3) / 4), 128, 0, stream>>>((const unsigned char*)h->d_vectors.ptr, h->row_stride,
                                                                        h->sketch_n, num, h->dim, (unsigned char*)h->d_sketch.ptr);
        g_launches++;
        CUDA_OK(cudaGetLastError());
        CUDA_OK(cudaStreamSynchronize(stream));
        h->sketch_n = h->n;
    }
    on = true;
    return 0;
}

// refine = true: the RefineSearchIndex flavour (BKTIndex.cpp:698-711) -- queries are base rows of the index itself
// (stride = the padded row stride), duplicate groups are not expanded, ids come back local (no shard offset); the
// caller passes MaxCheckForRefineGraph as opts.max_check.  Caller holds h->mu.
int search_device_impl(sptag_b200_index* h, const void* d_queries, int nq, int k, int* d_ids, float* d_dists,
                       int* d_stats, cudaStream_t stream, bool refine = false, CallOpts opts = CallOpts()) {
    if (nq <= 0) return SPTAG_B200_SUCCESS;
    int set = refine ? 0 : pick_scratch(h, stream);
    if (int rc = ensure_sketch(h, stream, opts.sketch)) return rc;
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
    p.rerun = opts.d_query_list;
    p.out_ids = d_ids;
    p.out_dists = d_dists;
    p.out_stats = d_stats;
    CUDA_OK(cudaMemsetAsync(p.work_counter, 0, 4, stream));
    if (p.vhash) {
        CUDA_OK(cudaMemsetAsync(p.work_counter + kRerunCounter, 0, 4, stream));
        CUDA_OK(cudaMemsetAsync(p.overflow, 0, 4, stream));
    }
    CUDA_OK(cudaEventRecord(h->ev_start, stream));
    L.kern<<<L.grid, 32, L.smem, stream>>>(p);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    h->last_search_kernel = (const void*)L.kern;
    if (p.vhash) {
        // the queries that filled their table run again on the bitmap: same stream, no host synchronisation; the count
        // is read on the device, so an empty list costs one near-empty launch
        SearchParams r = p;
        r.vhash = nullptr;
        r.vhash_limit = INT_MAX;
        r.vlog = nullptr;  // clear the bitmap per query
        r.vlog_entries = 0;
        r.overflow = nullptr;
        r.rerun = p.overflow;
        r.work_counter = p.work_counter + kRerunCounter;
        L.kern<<<rerun_grid(h, nq), 32, L.smem, stream>>>(r);
        g_launches++;
        CUDA_OK(cudaGetLastError());
    }
    CUDA_OK(cudaEventRecord(h->ev_stop, stream));
    if (opts.d_overflows) {
        if (p.vhash)
            CUDA_OK(cudaMemcpyAsync(opts.d_overflows, p.overflow, 4, cudaMemcpyDeviceToDevice, stream));
        else
            CUDA_OK(cudaMemsetAsync(opts.d_overflows, 0, 4, stream));
    }
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

// Before an iterator's first call, whose seeding cannot suspend: every hashed table of fewer than 2^need entries is
// replaced by an empty one of 2^need (the tables are still empty: nothing has run), or by a bitmap where such a table
// would be larger.  Caller holds h->mu.
int fit_iter_tables(sptag_b200_iterator* it, int need) {
    std::vector<unsigned> qs;
    std::vector<int> bits;
    for (int q = 0; q < it->nq; ++q)
        if (it->tables.bits[q] != 0 && it->tables.bits[q] < need) {
            qs.push_back((unsigned)q);
            bits.push_back(need);
        }
    return qs.empty() ? 0 : it->tables.grow(qs, bits, false, nullptr);
}

// The first Next of an iterator on hash tables with EnableBfs = bfs > 0: the breadth-first seeding inserts at most
// MaxBFSNodes centres per level and tree.  Caller holds h->mu.
int fit_bfs_seeding(sptag_b200_iterator* it, int bfs) {
    const long long seeds = std::min<long long>((long long)kBfsMaxNodes * bfs * it->h->tree_num, (long long)it->h->n + 1);
    int need = 6;
    while (need < 31 && ((long long)1 << (need - 1)) < seeds) ++need;
    return fit_iter_tables(it, need);
}

// Run one iterator step planned by plan_iterator_step.  The iterator's queue lengths and per-query arenas replace the
// per-slot scratch of a search; of scratch set 0 only the work counter is used, with the same ordering as a search.
// The grid stays the search kernel's.  launch(p, grid, smem, stream, iv) enqueues the iterate or nearest-first kernel;
// `what` names k in the refusal.  On hashed visited sets the kernel leaves the queries that reached their table's limit
// on a list: their tables grow (restart: they are replaced by empty ones) and the kernel runs again over that list,
// until the list is empty.  d_list (device, kIterListHeader layout, or nullptr for every query): the queries of the
// first launch.  out_ids nullptr: the results stay in it->d_ids and the call returns without waiting for the last
// launch.  Caller holds h->mu.
template <typename LaunchFn>
int run_iterator_step(sptag_b200_iterator* it, int k, const char* what, SearchLaunch& L, int32_t* out_ids,
                      float* out_dists, int32_t* out_counts, uint8_t* out_relaxed_mono, bool restart, LaunchFn&& launch,
                      const unsigned int* d_list = nullptr) {
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
    IterVisited iv = {};
    iv.margin = it->margin;
    iv.list = d_list;
    if (it->hashed) {
        iv.tables = (unsigned int* const*)it->tables.d_tables.ptr;
        iv.resume = (float*)it->d_resume.ptr;
        iv.suspended = (unsigned int*)it->d_susp[0].ptr;
    }
    if (int rc = scratch_acquire(h, stream)) return rc;
    CUDA_OK(cudaMemsetAsync(p.work_counter, 0, 4, stream));
    if (it->hashed) CUDA_OK(cudaMemsetAsync(iv.suspended, 0, kIterListHeader * 4, stream));
    CUDA_OK(cudaEventRecord(h->ev_start, stream));
    if (int rc = launch(p, L.grid, smem, stream, iv)) return rc;
    g_launches++;
    CUDA_OK(cudaGetLastError());
    long susp_step = 0, susp_trees = 0, growths = 0;
    for (int cur = 0; it->hashed; cur ^= 1) {  // at most ~log2(n) rounds: every round doubles the listed tables
        unsigned hdr[kIterListHeader];
        if (int rc = it->tables.double_listed((const unsigned int*)it->d_susp[cur].ptr, hdr, !restart, stream)) return rc;
        susp_step += hdr[1];
        susp_trees += hdr[2];
        if (hdr[0] == 0) break;
        growths += (long)hdr[0];
        iv.list = (const unsigned int*)it->d_susp[cur].ptr;
        iv.suspended = (unsigned int*)it->d_susp[cur ^ 1].ptr;
        CUDA_OK(cudaMemsetAsync(p.work_counter, 0, 4, stream));
        CUDA_OK(cudaMemsetAsync(iv.suspended, 0, kIterListHeader * 4, stream));
        if (int rc = launch(p, std::min(L.grid, (int)hdr[0]), smem, stream, iv)) return rc;
        g_launches++;
        CUDA_OK(cudaGetLastError());
    }
    h->last_iter_susp_step = susp_step;
    h->last_iter_susp_trees = susp_trees;
    h->last_iter_growths = growths;
    h->last_iter_visited_bytes = (long)it->visited_bytes();
    CUDA_OK(cudaEventRecord(h->ev_stop, stream));
    h->timed = true;
    if (int rc = scratch_release(h, stream)) return rc;
    it->stepped = true;
    if (!out_ids) return SPTAG_B200_SUCCESS;
    CUDA_OK(cudaMemcpyAsync(out_ids, it->d_ids.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_dists, it->d_dists.ptr, rn * 4, cudaMemcpyDeviceToHost, stream));
    if (out_counts) CUDA_OK(cudaMemcpyAsync(out_counts, it->d_counts.ptr, (size_t)it->nq * 4, cudaMemcpyDeviceToHost, stream));
    if (out_relaxed_mono)
        CUDA_OK(cudaMemcpyAsync(out_relaxed_mono, it->d_relaxed.ptr, (size_t)it->nq, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
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

// The handle's metric flag (true for every metric but L2) and element code, as the posting kernels' launchers take them
struct MetricElem {
    bool cosine;
    int elem;
};
MetricElem metric_elem(const sptag_b200_index* h) {
    MetricElem m = {h->metric != SPTAG_B200_METRIC_L2, 0};
    with_elem(h, [&](auto el) { m.elem = el; });
    return m;
}

// Writes nq queries (host or device memory) to dst as rows of the handle's row stride, zero padded, as the posting and
// cross-distance kernels read them
int upload_query_rows(const sptag_b200_index* h, void* dst, const void* queries, size_t nq, cudaStream_t stream) {
    const size_t qrow = (size_t)h->dim * value_size(h->value_type);
    CUDA_OK(cudaMemsetAsync(dst, 0, nq * h->row_stride, stream));
    CUDA_OK(cudaMemcpy2DAsync(dst, h->row_stride, queries, qrow, qrow, nq, cudaMemcpyDefault, stream));
    return 0;
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
        !h->staging.create_streams())
        return destroy_on_fail(fail(SPTAG_B200_FAIL, "cudaEventCreate / cudaStreamCreate failed"));
    cudaStream_t up = h->staging.sets[0].stream;
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

// indexloader.ini as Helper::IniReader reads it (SimpleIniReader.cpp:40-135): [Section] headers and Name=Value lines,
// section and parameter names trimmed and lower-cased; values trimmed here too
typedef std::map<std::string, std::map<std::string, std::string>> IniSections;
std::string trim(const std::string& v) {
    const size_t a = v.find_first_not_of(" \t\r");
    if (a == std::string::npos) return std::string();
    return v.substr(a, v.find_last_not_of(" \t\r") + 1 - a);
}
std::string lower(std::string v) {
    for (char& c : v) c = (char)std::tolower((unsigned char)c);
    return v;
}
bool read_ini(const std::string& path, IniSections& out) {
    std::ifstream ini(path);
    if (!ini) return false;
    std::string line, section;
    while (std::getline(ini, line)) {
        line = trim(line);
        if (line.empty() || line[0] == ';' || line[0] == '#') continue;
        if (line[0] == '[') {
            const size_t close = line.find(']');
            section = lower(trim(line.substr(1, close == std::string::npos ? std::string::npos : close - 1)));
            continue;
        }
        const size_t eq = line.find('=');
        if (eq != std::string::npos) out[section][lower(trim(line.substr(0, eq)))] = trim(line.substr(eq + 1));
    }
    return true;
}
std::string ini_get(const IniSections& ini, const char* section, const char* name, const std::string& def) {
    auto s = ini.find(lower(section));
    if (s == ini.end()) return def;
    auto it = s->second.find(lower(name));
    return it == s->second.end() ? def : it->second;
}

bool ini_true(const std::string& v) { return lower(v) == "true" || v == "1"; }

// The names of IndexAlgoType, VectorValueType and DistCalcMethod in an ini (DefinitionList.h), matched exactly
struct EnumName {
    int value;
    const char* name;
};
const EnumName kIndexAlgoTypes[] = {{SPTAG_B200_ALGO_BKT, "BKT"}, {SPTAG_B200_ALGO_KDT, "KDT"}};
const EnumName kValueTypes[] = {{SPTAG_B200_VT_INT8, "Int8"}, {SPTAG_B200_VT_UINT8, "UInt8"},
                                {SPTAG_B200_VT_INT16, "Int16"}, {SPTAG_B200_VT_FLOAT, "Float"}};
const EnumName kDistCalcMethods[] = {{SPTAG_B200_METRIC_L2, "L2"}, {SPTAG_B200_METRIC_COSINE, "Cosine"},
                                     {SPTAG_B200_METRIC_INNERPRODUCT, "InnerProduct"}};
template <size_t N>
int enum_value(const EnumName (&names)[N], const std::string& name) {  // -1: not a name of the table
    for (const EnumName& e : names)
        if (name == e.name) return e.value;
    return -1;
}
template <size_t N>
const char* enum_name(const EnumName (&names)[N], int value) {
    for (const EnumName& e : names)
        if (value == e.value) return e.name;
    return "Undefined";
}

// The parameters of a handle type H, one table per type as the reference's ParameterDefinitionList.h keeps them:
// set_param, get_param and the ini loaders all read the table.  Names match case-insensitively (StrEqualIgnoreCase,
// BKTIndex.cpp:980-1025).
enum : unsigned {
    kRefKey = 1,   // a key of the reference's ini: read from [Index] by sptag_b200_load, from [BuildHead] for a SPANN head
    kBktOnly = 2,  // BKT handles only: ParamNotFound on KDT
    kBool = 4,     // stored as v != 0
    kPow2 = 8,     // accepted: 0 or a power of two in [64, 2^30]
    kHead = 16,    // SPANN: the head handle's parameter, set and read there
};
template <typename H>
struct Param {
    const char* name;
    unsigned flags = 0;
    int H::*i = nullptr;                      // an int value (strtol, base 10)
    float H::*f = nullptr;                    // a float value (strtof)
    long lo = LONG_MIN, hi = LONG_MAX;        // the int values accepted
    int (*set)(H*, long) = nullptr;           // stores an accepted int value in place of i, with the side effects
    int (*get)(H*, char*, size_t) = nullptr;  // prints a read-only value
    Param(const char* n, int H::*m, unsigned fl = 0, long l = LONG_MIN, long u = LONG_MAX, int (*s)(H*, long) = nullptr)
        : name(n), flags(fl), i(m), lo(l), hi(u), set(s) {}
    Param(const char* n, float H::*m, unsigned fl = 0) : name(n), flags(fl), f(m) {}
    Param(const char* n, int (*g)(H*, char*, size_t)) : name(n), get(g) {}
    Param(const char* n, unsigned fl) : name(n), flags(fl) {}
};

template <typename H, size_t N>
const Param<H>* find_param(const Param<H> (&table)[N], const char* name, bool bkt = true) {
    for (const Param<H>& p : table)
        if (strcasecmp(p.name, name) == 0) return (p.flags & kBktOnly) && !bkt ? nullptr : &p;
    return nullptr;
}

// p: find_param's result for name.  The caller holds the lock of h's parameters.
template <typename H>
int set_param(H* h, const Param<H>* p, const char* name, const char* value) {
    if (!p) return fail(SPTAG_B200_PARAM_NOT_FOUND, "unknown parameter %s", name);
    if (p->get) return fail(SPTAG_B200_LACK_OF_INPUTS, "%s is read-only", p->name);
    char* end = nullptr;
    const float x = p->f ? strtof(value, &end) : 0.0f;
    const long v = p->f ? 0 : strtol(value, &end, 10);
    if (end == value) return fail(SPTAG_B200_FAILED_PARSE_VALUE, "cannot parse '%s' for %s", value, p->name);
    if (p->f) {
        h->*p->f = x;
        return SPTAG_B200_SUCCESS;
    }
    if ((p->flags & kPow2) && v != 0 && (v < 64 || v > (1l << 30) || (v & (v - 1)) != 0))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "%s %ld: 0 or a power of two in [64, 2^30]", p->name, v);
    if (v < p->lo || v > p->hi) return fail(SPTAG_B200_LACK_OF_INPUTS, "%s %ld outside [%ld, %ld]", p->name, v, p->lo, p->hi);
    if (p->set) return p->set(h, v);
    h->*p->i = (p->flags & kBool) ? (v != 0) : (int)v;
    return SPTAG_B200_SUCCESS;
}

int put(char* out, size_t capacity, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(out, capacity, fmt, ap);
    va_end(ap);
    return SPTAG_B200_SUCCESS;
}

template <typename H>
int get_param(H* h, const Param<H>* p, const char* name, char* out, size_t capacity) {
    if (!p) return fail(SPTAG_B200_PARAM_NOT_FOUND, "unknown parameter %s", name);
    if (p->get) return p->get(h, out, capacity);
    return p->f ? put(out, capacity, "%f", h->*p->f) : put(out, capacity, "%d", h->*p->i);  // %f: as ConvertToString
}

using Index = sptag_b200_index;
const Param<Index> kIndexParams[] = {
    {"MaxCheck", &Index::max_check, kRefKey},  // search: BKT/ParameterDefinitionList.h:44-49
    {"MaxCheckForRefineGraph", &Index::max_check_refine, kRefKey},
    {"NumberOfInitialDynamicPivots", &Index::initial_pivots, kRefKey},
    {"NumberOfOtherDynamicPivots", &Index::other_pivots, kRefKey},
    {"ThresholdOfNumberOfContinuousNoBetterPropagation", &Index::no_better_threshold, kRefKey},
    {"EnableBfs", &Index::bfs, kRefKey | kBktOnly},  // any int, like BKTree::m_bfs
    {"AddCEF", &Index::add_cef, kRefKey},  // graph updates: BKT/ParameterDefinitionList.h:28-31
    {"CEF", &Index::cef, kRefKey},
    {"RNGFactor", &Index::rng_factor, kRefKey},
    {"SearchDeleted", &Index::search_deleted, kBool},
    {"EnableADC", &Index::q_adc, kBool},  // VectorIndex::SetQuantizerADC (VectorIndex.h:136-138)
    {"B200.QueriesPerSM", &Index::queries_per_sm},
    {"B200.StageRows", &Index::stage_rows},
    {"B200.Stages", &Index::stages, 0, LONG_MIN, LONG_MAX,
     [](Index* h, long v) { h->stages = (int)v; h->stages_set = true; return SPTAG_B200_SUCCESS; }},
    {"B200.NGCacheEntries", &Index::h_ng},
    {"B200.SPTCacheEntries", &Index::h_spt},
    {"B200.SimdWidth", &Index::simd_width},
    {"B200.SlotScheme", &Index::slot_scheme},
    {"B200.VisitedLog", &Index::visited_log},
    {"B200.VisitedLogEntries", &Index::visited_log_entries},
    {"B200.VisitedSet", &Index::visited_set, 0, -1, 1, [](Index* h, long v) {
         h->visited_set = (int)v;
         for (auto& sc : h->scratch) sc.bitmap_unfit = 0;  // auto tries the bitmap again
         return SPTAG_B200_SUCCESS;
     }},
    {"B200.VisitedHashEntries", &Index::visited_hash_entries, kPow2},
    {"B200.IteratorVisitedSet", &Index::iter_visited_set, 0, -1, 1},  // taken by iterators opened afterwards
    {"B200.IteratorVisitedHashEntries", &Index::iter_hash_entries, kPow2},
    {"B200.RowSketch", &Index::row_sketch, 0, -1, 1, [](Index* h, long v) {
         if (v == 1 && !(h->value_type == SPTAG_B200_VT_FLOAT && h->q_type == 0 && h->algo == SPTAG_B200_ALGO_BKT))
             return fail(SPTAG_B200_LACK_OF_INPUTS, "B200.RowSketch 1: row sketches exist for float BKT indexes only");
         h->row_sketch = (int)v;
         h->sketch_unfit = false;  // auto tries the allocation again
         if (v == 0) { h->d_sketch.release(); h->sketch_n = 0; }
         return SPTAG_B200_SUCCESS;
     }},
    {"B200.RowsSkipped", [](Index* h, char* o, size_t n) {  // since the handle was made, over the searches that have finished
         unsigned long long c = 0;
         if (h->d_skipped.ptr) {
             DeviceGuard guard(h->device);
             CUDA_OK(cudaDeviceSynchronize());
             CUDA_OK(cudaMemcpy(&c, h->d_skipped.ptr, 8, cudaMemcpyDeviceToHost));
         }
         return put(o, n, "%ld", (long)c);
     }},
    {"B200.LastSearchKernel", [](Index* h, char* o, size_t n) { return put(o, n, "%s", kernel_name(h->last_search_kernel).c_str()); }},
    {"B200.LastVisitedOverflows", [](Index* h, char* o, size_t n) { return put(o, n, "%d", h->last_visited_overflows.load()); }},
    {"B200.ScratchBytes", [](Index* h, char* o, size_t n) { return put(o, n, "%zu", h->scratch[0].bytes() + h->scratch[1].bytes()); }},
    {"B200.LastIteratorSuspensions",  // "step,trees" of the last iterator call
     [](Index* h, char* o, size_t n) { return put(o, n, "%ld,%ld", h->last_iter_susp_step, h->last_iter_susp_trees); }},
    {"B200.LastIteratorGrowths", [](Index* h, char* o, size_t n) { return put(o, n, "%ld", h->last_iter_growths); }},
    {"B200.LastIteratorVisitedBytes", [](Index* h, char* o, size_t n) { return put(o, n, "%ld", h->last_iter_visited_bytes); }},
    // device time of the last refine pass
    {"B200.LastRefineSearchUs", [](Index* h, char* o, size_t n) { return put(o, n, "%ld", (long)(h->refine_search_ms * 1e3)); }},
    {"B200.LastRefineRebuildUs", [](Index* h, char* o, size_t n) { return put(o, n, "%ld", (long)(h->refine_rebuild_ms * 1e3)); }},
};

// The reference keys of kIndexParams present in ini's section, set on h.  Values set_param refuses are ignored, as
// LoadIndex ignores a failed ConvertStringTo.
void load_ref_keys(sptag_b200_index* h, const IniSections& ini, const char* section) {
    for (const Param<Index>& p : kIndexParams) {
        const std::string v = (p.flags & kRefKey) ? ini_get(ini, section, p.name, "") : "";
        if (!v.empty()) sptag_b200_set_param(h, p.name, v.c_str());
    }
}

}  // namespace

extern "C" {

const char* sptag_b200_last_error(void) { return g_last_error.c_str(); }

int64_t sptag_b200_launch_count(void) { return (int64_t)g_launches.load(); }

int sptag_b200_debug_kernel_for(int32_t value_type, int32_t metric, int32_t algo, int32_t dim, int32_t simd_width,
                                int32_t enable_bfs, int32_t row_sketch, int32_t quantized, int32_t mres_cap, int32_t slots,
                                int32_t family, char* name_out, int32_t capacity) {
    if (!name_out || capacity < 1) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    // the fields the selectors read, on a handle that owns nothing
    sptag_b200_index h;
    h.algo = algo;
    h.metric = metric;
    h.value_type = value_type;
    h.q_type = quantized ? 1 : 0;
    h.dim = dim;
    h.simd_width = simd_width;
    h.bfs = enable_bfs;
    const void* stub = nullptr;
    if (family == 0) {
        stub = (const void*)pick_kernel(&h, mres_cap, slots, row_sketch != 0 && sketch_applies(&h));
    } else if (family == 1 || family == 2) {
        SearchParams p;
        memset(&p, 0, sizeof(p));
        p.bfs = bfs_seeding(&h) ? h.bfs : 0;
        p.mres_cap = mres_cap;
        stub = family == 1 ? (const void*)pick_iter_step_kernel<IterateKernelFn>(&h, p)
                           : (const void*)pick_iter_step_kernel<NearestFirstKernelFn>(&h, p);
    } else {
        return fail(SPTAG_B200_LACK_OF_INPUTS, "family %d is not 0 (search), 1 (iterator) or 2 (nearest first)", family);
    }
    if (!stub) return fail(SPTAG_B200_LACK_OF_INPUTS, "no kernel for m_Results capacity %d", mres_cap);
    const std::string name = kernel_name(stub);
    if (name.empty()) return fail(SPTAG_B200_FAIL, "the kernel's launch stub has no exported symbol");
    snprintf(name_out, (size_t)capacity, "%s", name.c_str());
    return SPTAG_B200_SUCCESS;
}

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
    // indexloader.ini as VectorIndex::LoadIndex reads it (VectorIndex.cpp:617-681): the index's parameters and files
    // from [Index] (BKTIndex.cpp:21-31), its quantizer from [Quantizer] (VectorIndex.cpp:188-192)
    IniSections ini;
    if (!read_ini(dir + "/indexloader.ini", ini)) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot open %s/indexloader.ini", folder);
    auto get = [&](const char* name, const char* def) { return ini_get(ini, "Index", name, def); };
    IndexShape sh;
    sh.device = device;
    sh.id_offset = id_offset;
    const std::string algo = get("IndexAlgoType", "BKT");
    sh.algo = enum_value(kIndexAlgoTypes, algo);
    if (sh.algo < 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported IndexAlgoType %s", algo.c_str());
    const std::string vt = get("ValueType", "Float");
    sh.value_type = enum_value(kValueTypes, vt);
    if (sh.value_type < 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported ValueType %s", vt.c_str());
    const int metric = enum_value(kDistCalcMethods, get("DistCalcMethod", "Cosine"));  // reference default is Cosine
    sh.metric = metric < 0 ? SPTAG_B200_METRIC_COSINE : metric;
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
    const std::string qpath = ini_get(ini, "Quantizer", "QuantizerFilePath", "");
    if (!qpath.empty()) {
        std::vector<char> qb;
        if (!read_file(dir + "/" + qpath, qb)) {
            sptag_b200_destroy(h);
            return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read quantizer file %s", qpath.c_str());
        }
        if (int rc = sptag_b200_set_quantizer(h, qb.data(), (int64_t)qb.size())) {
            sptag_b200_destroy(h);
            return rc;
        }
    }
    load_ref_keys(h, ini, "Index");  // (EnableBfs is BKT-only: the KDT loader ignores the key)
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
    std::lock_guard<std::mutex> lock(h->mu);
    return set_param(h, find_param(kIndexParams, name, h->algo == SPTAG_B200_ALGO_BKT), name, value);
}

int sptag_b200_get_param(sptag_b200_handle h, const char* name, char* value_out, int32_t capacity) {
    if (!h || !name || !value_out || capacity <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    std::lock_guard<std::mutex> lock(h->mu);
    return get_param(h, find_param(kIndexParams, name, h->algo == SPTAG_B200_ALGO_BKT), name, value_out, (size_t)capacity);
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
    std::unique_lock<std::mutex> slock;
    auto* st = h->staging.acquire(slock);
    DeviceGuard guard(h->device);
    const size_t qbytes = (size_t)num_queries * query_bytes(h);
    const size_t rn = (size_t)num_queries * k;
    if (int rc = st->d_queries.ensure(qbytes)) return rc;
    if (int rc = st->d_ids.ensure(rn * 4)) return rc;
    if (int rc = st->d_dists.ensure(rn * 4)) return rc;
    if (out_stats)
        if (int rc = st->d_stats.ensure((size_t)num_queries * kStatsPerQuery * 4)) return rc;
    if (int rc = st->d_overflows.ensure(4)) return rc;
    opts.d_overflows = (int*)st->d_overflows.ptr;
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
    int overflows = 0;
    CUDA_OK(cudaMemcpyAsync(&overflows, st->d_overflows.ptr, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    h->last_visited_overflows = overflows;
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
    // (with room for the two BFS heaps whatever EnableBfs is now: the value in force at the first Next decides)
    it->spt_entries = p.spt_spill_entries + (p.bfs ? 0 : 2 * kBfsHeapEntries);
    const size_t qbytes = (size_t)num_queries * query_bytes(h);
    int rc = 0;
    if ((rc = it->d_queries.ensure(qbytes)) || (rc = it->d_ng.ensure((size_t)num_queries * it->ng_entries * 8)) ||
        (rc = it->d_spt.ensure((size_t)num_queries * it->spt_entries * 8)) ||
        (rc = it->d_state.ensure((size_t)num_queries * sizeof(IterState))) ||
        (rc = it->d_counts.ensure((size_t)num_queries * 4)) || (rc = it->d_relaxed.ensure((size_t)num_queries))) {
        delete it;
        return rc;
    }
    // The visited sets: a bitmap per query, or (B200.IteratorVisitedSet = 1, or auto when the bitmaps do not fit) a
    // hash table per query that grows while the iterator runs
    it->hashed = h->iter_visited_set == 1;
    if (!it->hashed && (rc = it->d_visited.ensure((size_t)num_queries * it->visited_words * 4))) {
        if (h->iter_visited_set == 0 || cudaGetLastError() != cudaErrorMemoryAllocation) {
            delete it;
            return rc;
        }
        it->hashed = true;  // auto: the bitmaps do not fit (the failed cudaMalloc's error is cleared above)
    }
    IterState st0 = {};
    st0.first = 1;   // first call: InitSearchTrees + SearchTrees
    st0.slots = -1;  // no QueryResult yet: the first Next sets the slot count
    if (it->hashed) {
        if (h->max_dup < 0) {  // computed once per handle: the tree does not change
            int* d_max = (int*)h->scratch[0].d_counter.ptr + 16;
            int m = 0;
            cudaError_t e = cudaMemset(d_max, 0, 4);
            max_dup_group_kernel<<<(h->node_count + 255) / 256, 256>>>((const int*)h->d_nodes.ptr, h->node_count, d_max);
            g_launches++;
            if (e == cudaSuccess) e = cudaMemcpy(&m, d_max, 4, cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) {
                delete it;
                return fail(SPTAG_B200_FAIL, "iterator set-up failed: %s", cudaGetErrorString(e));
            }
            h->max_dup = m;
        }
        it->margin = h->degree + h->max_dup + 1;
        // initial entries: B200.IteratorVisitedHashEntries, or the reference's first-block size as for search; raised
        // until one step fits below the limit, so that doubling a table always makes room for the step that suspended
        int bits = vhash_log2_entries(h->iter_hash_entries, std::max(h->max_check, h->max_check_refine));
        while (bits < 30 && (1 << (bits - 1)) < it->margin) ++bits;
        if ((rc = it->d_resume.ensure((size_t)num_queries * kIterResumeWords * 4)) ||
            (rc = it->d_susp[0].ensure((size_t)(kIterListHeader + num_queries) * 4)) ||
            (rc = it->d_susp[1].ensure((size_t)(kIterListHeader + num_queries) * 4)) ||
            (rc = it->tables.open((size_t)num_queries, bits, it->visited_words, (IterState*)it->d_state.ptr, st0))) {
            delete it;
            return rc;
        }
    }
    cudaError_t e = cudaMemcpy(it->d_queries.ptr, queries, qbytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !it->hashed) {  // (the tables' open wrote the states of hashed sets)
        const std::vector<IterState> st(num_queries, st0);
        e = cudaMemset(it->d_visited.ptr, 0, it->d_visited.bytes);
        if (e == cudaSuccess) e = cudaMemcpy(it->d_state.ptr, st.data(), st.size() * sizeof(IterState), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
        delete it;
        return fail(SPTAG_B200_FAIL, "iterator set-up failed: %s", cudaGetErrorString(e));
    }
    h->open_iterators++;  // sptag_b200_iterator_close gives it back
    *out = it;
    return SPTAG_B200_SUCCESS;
}

}  // extern "C"

namespace {

// ResultIterator::Next(batch) for the queries on d_list (nullptr: every query); batch is checked by the caller.
// out_ids nullptr: the results stay in it->d_ids / d_dists / d_counts, and the call does not wait for the last launch.
int next_step(sptag_b200_iterator* it, int batch, int32_t* out_ids, float* out_dists, int32_t* out_counts,
              uint8_t* out_relaxed_mono, const unsigned int* d_list) {
    sptag_b200_index* h = it->h;
    std::lock_guard<std::mutex> lock(h->mu);
    DeviceGuard guard(h->device);
    SearchLaunch L;
    if (int rc = plan_iterator_step(it, batch, L)) return rc;
    IterateKernelFn kern = pick_iter_step_kernel<IterateKernelFn>(h, L.p);
    if (!kern) return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, batch) = %d exceeds the supported 1024", L.p.mres_cap);
    if (!it->stepped && it->nearest_k == 0 && it->hashed && L.p.bfs > 0)
        if (int rc = fit_bfs_seeding(it, L.p.bfs)) return rc;
    return run_iterator_step(it, batch, "batch", L, out_ids, out_dists, out_counts, out_relaxed_mono, false,
                             [&](const SearchParams& p, int grid, size_t smem, cudaStream_t stream, const IterVisited& iv) {
                                 CUDA_OK(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                                 kern<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr, (int*)it->d_counts.ptr,
                                                                  (unsigned char*)it->d_relaxed.ptr, iv);
                                 h->last_search_kernel = (const void*)kern;
                                 return 0;
                             },
                             d_list);
}

}  // namespace

extern "C" {

int sptag_b200_iterator_next(sptag_b200_iter it, int32_t batch, int32_t* out_ids, float* out_dists, int32_t* out_counts,
                             uint8_t* out_relaxed_mono) {
    if (!it || !it->h) return fail(SPTAG_B200_EMPTY_INDEX, "null iterator");
    if (!out_ids || !out_dists) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (batch < 1 || batch > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "batch = %d outside [1, 1024]", batch);
    return next_step(it, batch, out_ids, out_dists, out_counts, out_relaxed_mono, nullptr);
}

}  // extern "C"

namespace {

// SearchIndexIterativeFromNeareast at k for the queries on d_list (nullptr: every query); k is checked by the caller.
// The results are copied to out_ids / out_dists, or (nullptr) stay in it->d_ids / it->d_dists.
int nearest_step(sptag_b200_iterator* it, int k, int32_t* out_ids, float* out_dists, const unsigned int* d_list) {
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
    NearestFirstKernelFn kfirst = pick_iter_step_kernel<NearestFirstKernelFn>(h, L.p);
    IterateKernelFn knext = pick_iter_step_kernel<IterateKernelFn>(h, L.p);
    if (!kfirst || !knext)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "max(MaxCheck/16, k) = %d exceeds the supported 1024", L.p.mres_cap);
    if (first && it->hashed) {
        // the seeding from the k results inserts at most k x (degree + 1) ids after nodeCheckStatus.clear(): every table
        // holds that below its limit (the tables are still empty)
        int need = 6;
        while (((size_t)1 << (need - 1)) < (size_t)k * (h->degree + 1)) ++need;
        if (int rc = fit_iter_tables(it, need)) return rc;
    }
    bool reset_slots = !first;
    const int rc = run_iterator_step(
        it, k, "k", L, out_ids, out_dists, nullptr, nullptr, first,
        [&](const SearchParams& p, int grid, size_t smem, cudaStream_t stream, const IterVisited& iv) {
            if (first) {
                CUDA_OK(cudaFuncSetAttribute((const void*)kfirst, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                kfirst<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr, iv);
                h->last_search_kernel = (const void*)kfirst;
            } else {
                // the caller Reset()s a QueryResult that keeps its k slots (SPANNIndex.cpp:284): no cap from the previous
                // count (once per call: a resume launch must not undo what its completed queries set).  Every query's
                // cap is reset, listed or not: each of these calls resets it before the kernel reads it.
                if (reset_slots)
                    CUDA_OK(cudaMemset2DAsync((char*)it->d_state.ptr + offsetof(IterState, slots), sizeof(IterState), 0xFF,
                                              sizeof(int), (size_t)it->nq, stream));
                reset_slots = false;
                CUDA_OK(cudaFuncSetAttribute((const void*)knext, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                knext<<<grid, 32, smem, stream>>>(p, (int*)it->d_state.ptr, (int*)it->d_counts.ptr, (unsigned char*)it->d_relaxed.ptr, iv);
                h->last_search_kernel = (const void*)knext;
            }
            return 0;
        },
        d_list);
    if (rc) return rc;
    it->nearest_k = k;
    return SPTAG_B200_SUCCESS;
}

}  // namespace

extern "C" {

int sptag_b200_iterator_next_from_nearest(sptag_b200_iter it, int32_t k, int32_t* out_ids, float* out_dists,
                                          uint8_t* out_found) {
    if (!it || !it->h) return fail(SPTAG_B200_EMPTY_INDEX, "null iterator");
    if (!out_ids || !out_dists) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (k < 1 || k > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside [1, 1024]", k);
    if (int rc = nearest_step(it, k, out_ids, out_dists, nullptr)) return rc;
    if (out_found)  // the reference's return value: is the first result slot a real vector
        for (int q = 0; q < it->nq; ++q) out_found[q] = out_ids[(size_t)q * k] >= 0 ? 1 : 0;
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
        const int w = std::fprintf(
            f,
            "[Index]\nIndexAlgoType=%s\nValueType=%s\n\nTreeFilePath=tree.bin\nGraphFilePath=graph.bin\nVectorFilePath=vectors.bin\n"
            "DeleteVectorFilePath=deletes.bin\nNeighborhoodSize=%d\nCEF=%d\nAddCEF=%d\nMaxCheckForRefineGraph=%d\nRNGFactor=%f\n"
            "DistCalcMethod=%s\nMaxCheck=%d\nThresholdOfNumberOfContinuousNoBetterPropagation=%d\nNumberOfInitialDynamicPivots=%d\n"
            "NumberOfOtherDynamicPivots=%d\n",
            enum_name(kIndexAlgoTypes, h->algo), enum_name(kValueTypes, h->value_type), h->degree, h->cef, h->add_cef,
            h->max_check_refine, h->rng_factor, enum_name(kDistCalcMethods, h->metric), h->max_check,
            h->no_better_threshold, h->initial_pivots, h->other_pivots);
        // written only when set, so that the folders of handles without it stay as they were
        const int wb = (bkt && h->bfs != 0) ? std::fprintf(f, "EnableBfs=%d\n", h->bfs) : 1;
        ok = w > 0 && wb > 0 && std::fclose(f) == 0 && ok;
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

// ---------------------------------------------------------------------------------------------------------------
// SPANN with its posting lists in HBM (SPANN::Index<T>, SPANNIndex.cpp; ExtraFullGraphSearcher.h).  The head is an
// ordinary handle loaded by sptag_b200_load; the lists are packed into one id array and one array of rows padded to the
// head's row stride, with one element offset per list.  The search runs the head search kernels at width W, then the
// posting scan kernel (kern_spann.cu; kern_spann_pq.cu on a quantized index, whose head and lists hold M-byte code
// rows: ExtraFullGraphSearcher<std::uint8_t>, SPANNIndex.cpp:93-99).
// ---------------------------------------------------------------------------------------------------------------
namespace {

// The threads a FILE-placed handle reads its posting files on.  run(n, fn) calls fn(0) .. fn(n - 1) on them and returns
// when every call has returned; two callers' batches share the threads, in turn.  The destructor joins them.
class ReadPool {
  public:
    explicit ReadPool(unsigned threads) {
        for (unsigned i = 0; i < threads; ++i) workers_.emplace_back([this] { work(); });
    }
    ~ReadPool() {
        {
            std::lock_guard<std::mutex> lock(mu_);
            stop_ = true;
        }
        more_.notify_all();
        for (std::thread& t : workers_) t.join();
    }
    void run(size_t n, const std::function<void(size_t)>& fn) {
        if (n == 0) return;
        Batch b{&fn, n};
        std::unique_lock<std::mutex> lock(mu_);
        queue_.push_back(&b);
        more_.notify_all();
        done_.wait(lock, [&] { return b.done == n; });
    }

  private:
    struct Batch {
        const std::function<void(size_t)>* fn;
        size_t n, next = 0, done = 0;
    };
    void work() {
        std::unique_lock<std::mutex> lock(mu_);
        for (;;) {
            more_.wait(lock, [&] { return stop_ || !queue_.empty(); });
            if (queue_.empty()) return;  // stop_: no caller is waiting (the handle is being destroyed)
            Batch* b = queue_.front();
            const size_t i = b->next++;
            if (b->next == b->n) queue_.pop_front();
            lock.unlock();
            (*b->fn)(i);
            lock.lock();
            if (++b->done == b->n) done_.notify_all();
        }
    }
    std::mutex mu_;
    std::condition_variable more_, done_;
    std::deque<Batch*> queue_;
    bool stop_ = false;
    std::vector<std::thread> workers_;
};

// A FILE-placed handle's posting files: each one's path and descriptor (O_RDONLY, open for the handle's life)
struct PostingFileSet {
    std::vector<std::string> paths;
    std::vector<int> fds;
    ~PostingFileSet() {
        for (int fd : fds) close(fd);
    }
};

// A staging set's windows for the FILE placement: two pinned, mapped windows of `bytes` the posting files are read into,
// each followed by its piece table, and per window the event recorded behind the last unpack kernel that read it
constexpr size_t kFileWindow = 64ull << 20;
constexpr int kPieceLists = 4096;
struct FileWindows {
    unsigned char* host = nullptr;  // 2 x (bytes + kPieceLists FilePieceLists)
    unsigned char* dev = nullptr;   // its device (mapped) address
    size_t bytes = 0;
    cudaEvent_t read[2] = {nullptr, nullptr};
    DeviceBuffer d_tables;  // 2 x kPieceLists FilePieceLists
    FileWindows() = default;
    FileWindows(const FileWindows&) = delete;
    FileWindows& operator=(const FileWindows&) = delete;
    ~FileWindows() {
        if (host) cudaFreeHost(host);
        for (cudaEvent_t e : read)
            if (e) cudaEventDestroy(e);
    }
    size_t span() const { return bytes + kPieceLists * sizeof(FilePieceList); }
    unsigned char* window(int w) const { return host + w * span(); }
    FilePieceList* table(int w) const { return reinterpret_cast<FilePieceList*>(window(w) + bytes); }
};

}  // namespace

struct sptag_b200_spann {
    sptag_b200_index* head = nullptr;
    bool quantized = false;  // [Base] QuantizerFilePath: the head's quantizer scores the postings too
    int vis = 0;          // m_vectorInfoSize: dim * sizeof(T) + sizeof(int) (quantized: M code bytes + sizeof(int))
    int rearranged = 0;   // EnablePostingListRearrange
    int num_lists = 0;
    std::vector<int> cnt, pages;  // per list: full element count, page count (host copies for the table size)
    // search parameters (SPANN/ParameterDefinitionList.h:110-117)
    int internal = 64;
    float max_dist_ratio = 10000.0f;
    int page_limit = 3;       // SearchPostingPageLimit as set
    int vector_limit_pages = 0;  // ceil(PostingVectorLimit * vis / PageSize): the least page limit in force
    int longest = 0;          // spann_update_shape
    bool truncated = false;
    // iterators: IterativeSearchHeadBatch (ParameterDefinitionList.h:125), the first dedup table size (0 = from the
    // lists), and what the last Next on this handle did
    int head_batch = 32;
    int dedup_entries = 0;
    long last_iter_rounds = 0, last_iter_dedup_bytes = 0;
    // host stub of the last posting-scan or posting-step kernel this handle launched (B200.LastPostingKernel)
    const void* last_posting_kernel = nullptr;
    DeviceBuffer d_translate, d_off, d_cnt, d_pages, d_ids, d_rows;
    // Host placement (sptag_b200_spann_load_ex): the rows, then the ids, in one pinned mapped allocation, and the HBM stage
    // of each staging set (B200.PostingStageBytes); what the last search or iterator step on this handle gathered
    bool host_postings = false;
    void* h_postings = nullptr;
    size_t h_posting_bytes = 0;
    const unsigned char* h_rows = nullptr;  // device (mapped) pointers into h_postings
    const int* h_ids = nullptr;
    int stage_bytes = 256 << 20;
    long last_gather_bytes = 0, last_gather_rounds = 0;
    // Host placement's HBM cache of lists (sptag_b200_spann_cache_lists): one allocation of cache_pool elements (the cached
    // lists, whole, in the order given) then cache_stage elements per staging set, their rows at the head's row stride,
    // then their ids; d_resident: per list, its first element in the pool or -1.  Replaced with both staging sets held;
    // cache_stage never shrinks, so that a stage a caller fitted before taking its set is still there.  The sizes are
    // also written under mu, for the parameters.
    DeviceBuffer d_cache, d_resident;
    std::vector<int> cache_lists;
    long long cache_pool = 0, cache_stage = 0, cache_bytes = 0;
    // File placement (host_postings is set too: the lists are staged as the host placement's are): the lists stay in
    // their posting files and each call reads its union from there (spann_stage); per list its file and first byte.
    // last_read_bytes: the file bytes the last search, iterator step or cache install on this handle read.
    bool file_postings = false;
    PostingFileSet post_files;
    std::vector<int> list_file;
    std::vector<long long> list_start;
    std::unique_ptr<ReadPool> readers;
    long last_read_bytes = 0;
    // Host-buffer calls run on one of two staging sets, each with its own stream, head results, dedup tables and outputs,
    // so that two callers overlap; the head search kernels are ordered by the head handle (search_device_impl)
    struct StagingBuffers {
        DeviceBuffer d_q, d_qpad, d_hids, d_hdists, d_ids, d_dists, d_stats, d_tables;
        DeviceBuffer d_codes, d_adc;  // quantized: the queries' codes (SDC) or rotated vectors (ADC); ADC tables per block
        // host placement: the chosen lists per item, the union (PostingGather), an iterator launch's sub-list, the stage
        DeviceBuffer d_chosen, d_nchosen, d_flags, d_len, d_stage_off, d_union, d_nunion, d_cub, d_sub, d_stage;
        DeviceBuffer d_view_off;  // with a cache: the view's list offsets
        DeviceBuffer d_peer_elems;  // a group member's: the elements a call copied from peers
        FileWindows windows;        // file placement
    };
    StagingPool<StagingBuffers> staging;
    std::mutex mu;  // the search parameters
    // A member of a SPANN group (sptag_b200_spann_group_load): the group owns the handle and the pinned allocation
    // (h_postings stays null here).  Its peer table (spann_group_peer_tables, rebuilt with every member's staging sets
    // held, so that a call holding one set sees a fixed table): per list the member that caches it and its first element
    // there, per member the pool's rows and ids; peers.first is null when no reachable peer caches a list.
    sptag_b200_spann_group* group = nullptr;
    DeviceBuffer d_peer_first, d_peer_owner;
    PostingPeers peers = {};
    long peer_lists = 0;
    long last_peer_gather_bytes = 0;
};

// A SPANN group: members on one or more devices that share one pinned copy of the posting lists, and whose HBM caches
// hold each list at most once.  reach[i][o]: member i reads member o's pool (the same device, or peer access enabled).
struct sptag_b200_spann_group {
    std::vector<sptag_b200_spann*> members;
    std::vector<std::vector<char>> reach;
    void* h_postings = nullptr;
    std::mutex install;  // taken by every install on a member, before every member's staging sets (GroupSets)
    std::mutex params;   // sptag_b200_spann_group_set_param
};

namespace {

// The page limit a search uses: LoadIndex raises SearchPostingPageLimit to the pages of PostingVectorLimit vectors
// (ExtraFullGraphSearcher.h:167)
int spann_page_limit(const sptag_b200_spann* s) { return std::max(s->page_limit, s->vector_limit_pages); }

// HBM that AUTO placement and cache_warm's default budget leave for the searches' buffers (head results, dedup tables,
// outputs, stages)
constexpr long long kPostingReserve = 1ll << 30;

// The parameters a SPANN search or iterator step runs with, read together under s->mu
struct SpannSnapshot {
    int internal, page_limit, longest, stage_bytes;
    float max_dist_ratio;
};
// Takes the snapshot, and refuses a page limit that truncates lists of the rearranged layout: the reference reads a
// truncated list's ids from an offset computed with the truncated count (ExtraFullGraphSearcher.h:1186-1190), and its
// results on such lists are not reproduced
int spann_snapshot(sptag_b200_spann* s, SpannSnapshot& out) {
    bool truncated = false;
    {
        std::lock_guard<std::mutex> lock(s->mu);
        out.internal = s->internal;
        out.max_dist_ratio = s->max_dist_ratio;
        out.page_limit = spann_page_limit(s);
        out.longest = s->longest;
        out.stage_bytes = s->stage_bytes;
        truncated = s->truncated;
    }
    if (truncated && s->rearranged)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "SearchPostingPageLimit %d truncates posting lists of the rearranged layout",
                    out.page_limit);
    return 0;
}

// The posting lists of the index as the posting kernels read them at page limit page_limit (host placement: the ids and
// rows in mapped host memory, which gather_rounds stages)
PostingLists posting_lists(const sptag_b200_spann* s, int page_limit) {
    const int* ids = s->host_postings ? s->h_ids : (const int*)s->d_ids.ptr;
    const unsigned char* rows = s->host_postings ? s->h_rows : (const unsigned char*)s->d_rows.ptr;
    return {(const long long*)s->d_off.ptr, (const int*)s->d_cnt.ptr, (const int*)s->d_pages.ptr, ids, rows,
            s->head->row_stride, s->vis, page_limit};
}

// The elements of a stage: B200.PostingStageBytes, or one query's worst case if larger
long long stage_elems(const sptag_b200_spann* s, const SpannSnapshot& sp) {
    const long long elem_bytes = (long long)s->head->row_stride + 4;
    const long long cap = std::max<long long>(sp.stage_bytes, (long long)std::max(sp.internal, 0) * sp.longest * elem_bytes);
    return cap / elem_bytes;
}

// File placement: the window of a staging set, grown to `bytes` (its events and tables made on first use).  Caller holds
// the set; the set's earlier unpack kernels have completed or are waited for here.
int spann_file_windows(FileWindows& fw, size_t bytes) {
    for (cudaEvent_t& e : fw.read)
        if (!e) CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    if (int rc = fw.d_tables.ensure(2 * kPieceLists * sizeof(FilePieceList))) return rc;
    if (fw.bytes >= bytes) return 0;
    for (cudaEvent_t e : fw.read) CUDA_OK(cudaEventSynchronize(e));
    if (fw.host) cudaFreeHost(fw.host);
    fw.host = fw.dev = nullptr;
    fw.bytes = bytes;
    if (cudaHostAlloc((void**)&fw.host, 2 * fw.span(), cudaHostAllocMapped) != cudaSuccess) {
        fw.host = nullptr;
        fw.bytes = 0;
        cudaGetLastError();
        return fail(SPTAG_B200_MEMORY_OVERFLOW, "cudaHostAlloc(%zu) of the posting-file windows failed",
                    2 * (bytes + kPieceLists * sizeof(FilePieceList)));
    }
    CUDA_OK(cudaHostGetDevicePointer((void**)&fw.dev, fw.host, 0));
    return 0;
}

// File placement: every posting file is still the one the handle opened at its path (a file moved away or replaced
// since the load fails the call, which would otherwise read the old file's bytes)
int spann_files_in_place(const sptag_b200_spann* s) {
    const PostingFileSet& pf = s->post_files;
    for (size_t i = 0; i < pf.fds.size(); ++i) {
        struct stat at, open_st;
        if (stat(pf.paths[i].c_str(), &at) != 0 || fstat(pf.fds[i], &open_st) != 0 || at.st_dev != open_st.st_dev ||
            at.st_ino != open_st.st_ino)
            return fail(SPTAG_B200_FAIL, "posting file %s is no longer the file the index loaded (moved or replaced)",
                        pf.paths[i].c_str());
    }
    return 0;
}

// Where a union's lists come from, for the gather rounds and the cache installs: copies g.len[l] elements of every list
// l of g.lists (*g.nlists of them) to element g.stage_off[l] of g's stage.  whole: g.len holds every element of each
// list (a cache install), else the searched prefix at g.host.page_limit.
//   HOST (and a group member): from mapped host memory or a peer's pool, with the gather kernel.
//   FILE: the union, in order, is cut into pieces that fit a window of kFileWindow bytes (or of the largest list's raw
//   bytes), each list's raw bytes at a 16-byte-aligned offset: plain, its len x vis searched bytes; rearranged, the
//   whole list.  The read pool preads piece p into one of the set's two windows while the unpack kernel of piece p - 1
//   cuts the other into the stage; a window is refilled once the event behind its last kernel has completed.
//   read_bytes += the file bytes read.  A failed or short read fails the call, naming the file, the list and the
//   offset, with the stream synchronised.
int spann_stage(sptag_b200_spann* s, sptag_b200_spann::StagingBuffers& set, const PostingGather& g, bool whole,
                cudaStream_t stream, long& read_bytes) {
    if (!s->file_postings) {
        CUDA_OK(launch_spann_gather(g, s->head->num_sms * 4, stream));
        g_launches++;
        return 0;
    }
    if (int rc = spann_files_in_place(s)) return rc;
    int n = 0;
    CUDA_OK(cudaMemcpyAsync(&n, g.nlists, 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    std::vector<int> lists((size_t)n);
    if (n > 0) {
        CUDA_OK(cudaMemcpyAsync(lists.data(), g.lists, (size_t)n * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
    }
    // each list's raw bytes: the host's own count of what g.len holds
    std::vector<long long> raw((size_t)n);
    long long largest = 0, total = 0;
    for (int u = 0; u < n; ++u) {
        const int l = lists[u];
        const long long len = whole ? s->cnt[l] : posting_searched(s->cnt[l], s->pages[l], g.host.page_limit, s->vis);
        raw[u] = len == 0 ? 0 : (s->rearranged ? (long long)s->cnt[l] : len) * s->vis;
        largest = std::max(largest, raw[u]);
        total += raw[u];
    }
    FileWindows& fw = set.windows;
    if (int rc = spann_file_windows(fw, std::max<size_t>(kFileWindow, round_up((size_t)largest, 16)))) return rc;
    // a piece's reads, split into jobs of about kReadJob bytes so that a large list keeps several threads busy
    constexpr long long kReadJob = 1ll << 20;
    struct Read {
        int file, list;
        long long offset, bytes;
        unsigned char* dst;
    };
    std::vector<Read> reads;
    std::vector<size_t> jobs;  // the first read of each job, then reads.size()
    std::mutex err_mu;
    std::string err;
    auto do_job = [&](size_t j) {
        for (size_t r = jobs[j]; r < jobs[j + 1]; ++r) {
            const Read& rd = reads[r];
            long long got = 0;
            while (got < rd.bytes) {
                const ssize_t k = pread(s->post_files.fds[rd.file], rd.dst + got, (size_t)(rd.bytes - got), rd.offset + got);
                if (k < 0 && errno == EINTR) continue;
                if (k <= 0) {
                    char msg[512];
                    snprintf(msg, sizeof(msg), "posting file %s: list %d: read at offset %lld %s",
                             s->post_files.paths[rd.file].c_str(), rd.list, rd.offset + got,
                             k < 0 ? strerror(errno) : "ends before the list does");
                    std::lock_guard<std::mutex> lock(err_mu);
                    if (err.empty()) err = msg;
                    return;
                }
                got += k;
            }
        }
    };
    const std::function<void(size_t)> job_fn = do_job;
    int piece = 0;
    for (int u0 = 0; u0 < n; ++piece) {
        const int w = piece & 1;
        CUDA_OK(cudaEventSynchronize(fw.read[w]));  // the kernel that last read this window
        unsigned char* win = fw.window(w);
        FilePieceList* table = fw.table(w);
        reads.clear();
        jobs.assign(1, 0);
        long long at = 0, job_bytes = 0;
        int u = u0;
        for (; u < n && u - u0 < kPieceLists; ++u) {
            const long long off = (long long)round_up((size_t)at, 16);
            if (u > u0 && off + raw[u] > (long long)fw.bytes) break;
            const int l = lists[u];
            table[u - u0] = {off, l, 0};
            for (long long b = 0; b < raw[u]; b += kReadJob) {
                reads.push_back({s->list_file[l], l, s->list_start[l] + b, std::min(kReadJob, raw[u] - b), win + off + b});
                job_bytes += reads.back().bytes;
                if (job_bytes >= kReadJob) {
                    jobs.push_back(reads.size());
                    job_bytes = 0;
                }
            }
            at = off + raw[u];
        }
        if (jobs.back() != reads.size()) jobs.push_back(reads.size());
        s->readers->run(jobs.size() - 1, job_fn);
        if (!err.empty()) {
            cudaStreamSynchronize(stream);
            return fail(SPTAG_B200_FAIL, "%s", err.c_str());
        }
        FilePieceList* d_table = (FilePieceList*)fw.d_tables.ptr + w * kPieceLists;
        CUDA_OK(cudaMemcpyAsync(d_table, table, (size_t)(u - u0) * sizeof(FilePieceList), cudaMemcpyHostToDevice, stream));
        CUDA_OK(launch_spann_file_unpack(g, d_table, u - u0, fw.dev + (win - fw.host), s->rearranged != 0, stream));
        g_launches++;
        CUDA_OK(cudaEventRecord(fw.read[w], stream));
        u0 = u;
    }
    read_bytes += (long)total;
    return 0;
}

// Host placement: runs the n items of a call (the queries of a search, or of an iterator's posting-step launch) in
// gather rounds on staging set sb.  A round takes the next m items, m starting at n and halved (rounded up) until the
// union of their lists fits the stage (never below one item), gathers that union into the stage and runs them on it;
// the next round starts from the same m.  choose(b, e, chosen, nchosen) points chosen / nchosen at the lists items
// [b, e) read (stride apart), enqueued on stream; run(b, e, view) runs items [b, e) on the staged view.  The stage holds
// the larger of B200.PostingStageBytes and one query's worst case.  Adds the bytes gathered and the rounds to bytes and
// rounds, the part of those bytes a group member copied from peers' pools to peer_bytes, and the file bytes a
// FILE-placed handle read to read_bytes.
template <typename Buffers, typename Choose, typename Run>
int gather_rounds(sptag_b200_spann* s, Buffers& sb, const SpannSnapshot& sp, int n, int stride, cudaStream_t stream,
                  Choose&& choose, Run&& run, long& bytes, long& rounds, long& peer_bytes, long& read_bytes) {
    const PostingLists host = posting_lists(s, sp.page_limit);
    const long long elem_bytes = (long long)host.row_stride + 4;
    const long long cap_elems = stage_elems(s, sp);
    const size_t nl = (size_t)s->num_lists;
    // the cache cannot change while this caller holds a staging set (spann_cache_install holds both), and
    // spann_acquire_fitted took the set with a cache stage of at least cap_elems
    const bool cached = s->d_cache.ptr != nullptr;
    if (cached && cap_elems > s->cache_stage)
        return fail(SPTAG_B200_FAIL, "the cache's stage of %lld elements is smaller than the %lld needed", s->cache_stage,
                    cap_elems);
    const size_t temp = spann_union_temp_bytes(s->num_lists);
    if (temp == 0) return fail(SPTAG_B200_FAIL, "the posting-list union's scratch size query failed");
    if (int rc = sb.d_flags.ensure(nl)) return rc;
    if (int rc = sb.d_len.ensure((nl + 1) * 8)) return rc;
    if (int rc = sb.d_stage_off.ensure((nl + 1) * 8)) return rc;
    if (int rc = sb.d_union.ensure(nl * 4 + 4)) return rc;
    if (int rc = sb.d_nunion.ensure(4)) return rc;
    if (int rc = sb.d_cub.ensure(temp)) return rc;
    if (cached) {
        if (int rc = sb.d_view_off.ensure(nl * 8)) return rc;
    } else if (int rc = sb.d_stage.ensure((size_t)std::max(cap_elems, 1ll) * elem_bytes)) {
        return rc;
    }
    PostingGather g;
    memset(&g, 0, sizeof(g));
    g.host = host;
    g.num_lists = s->num_lists;
    g.flags = (unsigned char*)sb.d_flags.ptr;
    g.len = (long long*)sb.d_len.ptr;
    g.stage_off = (long long*)sb.d_stage_off.ptr;
    g.lists = (int*)sb.d_union.ptr;
    g.nlists = (int*)sb.d_nunion.ptr;
    g.temp = sb.d_cub.ptr;
    g.temp_bytes = sb.d_cub.bytes;
    g.stage_rows = (unsigned char*)sb.d_stage.ptr;
    g.stage_ids = (int*)(g.stage_rows + (size_t)std::max(cap_elems, 1ll) * host.row_stride);
    PostingLists view = host;
    view.off = g.stage_off;
    view.ids = g.stage_ids;
    view.rows = g.stage_rows;
    if (cached) {  // the pool, then the stage of each staging set, in one element space
        const long long all = s->cache_pool + 2 * s->cache_stage;
        unsigned char* rows = (unsigned char*)s->d_cache.ptr;
        int* ids = (int*)(rows + (size_t)all * host.row_stride);
        g.resident = (const long long*)s->d_resident.ptr;
        g.stage_base = s->cache_pool + (long long)(&sb - s->staging.sets) * s->cache_stage;
        g.view_off = (long long*)sb.d_view_off.ptr;
        g.stage_rows = rows + (size_t)g.stage_base * host.row_stride;
        g.stage_ids = ids + g.stage_base;
        view.off = g.view_off;
        view.ids = ids;
        view.rows = rows;
    }
    // the peer table is rebuilt only while every staging set of every member is held, so it is fixed during the call
    if (s->peers.first) {
        if (int rc = sb.d_peer_elems.ensure(8)) return rc;
        g.peers = s->peers;
        g.peers.elems = (unsigned long long*)sb.d_peer_elems.ptr;
        CUDA_OK(cudaMemsetAsync(g.peers.elems, 0, 8, stream));
    }
    for (int b = 0, m = n; b < n; b += m) {
        m = std::min(m, n - b);
        long long elems = 0;
        for (;;) {
            const int* chosen = nullptr;
            const int* nchosen = nullptr;
            if (int rc = choose(b, b + m, chosen, nchosen)) return rc;
            CUDA_OK(launch_spann_union(g, chosen, nchosen, stride, m, stream));
            CUDA_OK(cudaMemcpyAsync(&elems, g.stage_off + nl, 8, cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            if (elems <= cap_elems || m == 1) break;
            m = (m + 1) / 2;
        }
        if (elems > cap_elems)  // one query reads at most SearchInternalResultNum lists of at most `longest` elements
            return fail(SPTAG_B200_FAIL, "one query's %lld posting elements exceed the stage's %lld", elems, cap_elems);
        if (int rc = spann_stage(s, sb, g, false, stream, read_bytes)) return rc;
        if (int rc = run(b, b + m, view)) return rc;
        bytes += (long)(elems * elem_bytes);
        ++rounds;
    }
    if (g.peers.first) {
        unsigned long long from_peers = 0;
        CUDA_OK(cudaMemcpyAsync(&from_peers, g.peers.elems, 8, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        peer_bytes += (long)((long long)from_peers * elem_bytes);
    }
    return 0;
}

// The longest list a search reads at the page limit in force, and whether that limit truncates any list (recomputed when
// the limit changes).  Caller holds s->mu.
void spann_update_shape(sptag_b200_spann* s) {
    const int limit = spann_page_limit(s);
    s->longest = 0;
    s->truncated = false;
    for (int l = 0; l < s->num_lists; ++l) {
        const int tc = posting_searched(s->cnt[l], s->pages[l], limit, s->vis);
        s->longest = std::max(s->longest, tc);
        s->truncated = s->truncated || tc < s->cnt[l];
    }
}

// Host placement: both staging sets, so that no search or iterator step runs while the cache changes (in set order, as
// nothing else holds more than one)
struct BothSets {
    std::unique_lock<std::mutex> a, b;
    explicit BothSets(sptag_b200_spann* s) : a(s->staging.sets[0].mu), b(s->staging.sets[1].mu) {}
};

// Releases the cache, and the stages of the uncached path (HBM the cache's own stages replace).  Caller holds BothSets.
void spann_cache_release(sptag_b200_spann* s) {
    s->d_cache.release();
    for (auto& set : s->staging.sets) set.d_stage.release();
    std::lock_guard<std::mutex> lock(s->mu);
    s->cache_lists.clear();
    s->cache_pool = s->cache_bytes = 0;
}

// The copy of spann_cache_install, on the handle's device (the lists' source: spann_stage, on staging set 0)
int spann_cache_copy(sptag_b200_spann* s, const std::vector<int>& lists, long long stage) {
    const size_t nl = (size_t)s->num_lists, rs = s->head->row_stride;
    stage = std::max({stage, s->cache_stage, 1ll});
    std::vector<long long> resident(nl, -1), len(nl, 0);
    long long pool = 0;
    for (int l : lists) {
        resident[l] = pool;
        len[l] = s->cnt[l];
        pool += s->cnt[l];
    }
    const long long all = pool + 2 * stage;
    if (int rc = s->d_cache.ensure((size_t)all * (rs + 4))) return rc;
    // the copy's inputs: the lists, their count, each one's length
    DeviceBuffer d_in;
    if (int rc = s->d_resident.ensure(nl * 8)) return rc;
    if (int rc = d_in.ensure(nl * 8 + lists.size() * 4 + 4)) return rc;
    long long* d_len = (long long*)d_in.ptr;
    int* d_lists = (int*)(d_len + nl);
    int* d_n = d_lists + lists.size();
    const int n = (int)lists.size();
    CUDA_OK(cudaMemcpy(s->d_resident.ptr, resident.data(), nl * 8, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_len, len.data(), nl * 8, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_lists, lists.data(), lists.size() * 4, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_n, &n, 4, cudaMemcpyHostToDevice));
    PostingGather g;
    memset(&g, 0, sizeof(g));
    g.host = posting_lists(s, 0);
    g.num_lists = s->num_lists;
    g.len = d_len;
    g.stage_off = (long long*)s->d_resident.ptr;
    g.lists = d_lists;
    g.nlists = d_n;
    g.stage_rows = (unsigned char*)s->d_cache.ptr;
    g.stage_ids = (int*)(g.stage_rows + (size_t)all * rs);
    cudaStream_t stream = s->staging.sets[0].stream;
    long read_bytes = 0;
    if (int rc = spann_stage(s, s->staging.sets[0], g, true, stream, read_bytes)) return rc;
    CUDA_OK(cudaStreamSynchronize(stream));
    std::lock_guard<std::mutex> lock(s->mu);
    s->last_read_bytes = read_bytes;
    s->cache_lists = lists;
    s->cache_pool = pool;
    s->cache_stage = stage;
    s->cache_bytes = pool * (long long)(rs + 4);
    return 0;
}

// Installs the cache of `lists` (valid, distinct) with stages of at least `stage` elements: releases the old one, then
// copies every element of each list from mapped host memory into the pool with the gather kernel.  MemoryOverFlow when
// the allocation fails; the handle is then uncached.  Caller holds BothSets.
int spann_cache_install(sptag_b200_spann* s, const std::vector<int>& lists, long long stage) {
    DeviceGuard guard(s->head->device);
    spann_cache_release(s);
    if (lists.empty()) return 0;
    const int rc = spann_cache_copy(s, lists, stage);
    if (rc) s->d_cache.release();
    return rc;
}

// Every member's two staging sets, in member order then set order, under the group's install mutex: what an install on
// a group member holds, since its peers read its pool.  A search or iterator step holds one set of one member at a
// time and takes no other lock while it does, so this order cannot deadlock.
struct GroupSets {
    std::unique_lock<std::mutex> install;
    std::vector<std::unique_lock<std::mutex>> sets;
    explicit GroupSets(sptag_b200_spann_group* g) : install(g->install) {
        for (sptag_b200_spann* m : g->members)
            for (auto& set : m->staging.sets) sets.emplace_back(set.mu);
    }
};

// Rebuilds every member's peer table from the members' caches (spann_cache_copy's pool layout: the lists whole, in
// cache_lists order).  A member whose table cannot be uploaded reads every list it does not cache from host memory.
// Caller holds GroupSets.
int spann_group_peer_tables(sptag_b200_spann_group* g) {
    const size_t n = g->members.size(), nl = (size_t)g->members[0]->num_lists;
    std::vector<int> owner(nl, -1);
    std::vector<long long> first(nl, -1);
    PostingPeers pools = {};
    for (size_t o = 0; o < n; ++o) {
        const sptag_b200_spann* m = g->members[o];
        if (!m->d_cache.ptr) continue;
        long long pos = 0;
        for (int l : m->cache_lists) {
            owner[l] = (int)o;
            first[l] = pos;
            pos += m->cnt[l];
        }
        pools.rows[o] = (const unsigned char*)m->d_cache.ptr;
        pools.ids[o] = (const int*)(pools.rows[o] + (size_t)(m->cache_pool + 2 * m->cache_stage) * m->head->row_stride);
    }
    int rc = 0;
    for (size_t i = 0; i < n; ++i) {
        sptag_b200_spann* s = g->members[i];
        std::vector<long long> from(nl, -1);
        std::vector<int> by(nl, 0);
        long count = 0;
        for (size_t l = 0; l < nl; ++l) {
            if (owner[l] < 0 || owner[l] == (int)i || !g->reach[i][(size_t)owner[l]]) continue;
            from[l] = first[l];
            by[l] = owner[l];
            ++count;
        }
        PostingPeers p = pools;
        p.first = nullptr;
        p.owner = nullptr;
        int r = 0;
        if (count > 0) {
            DeviceGuard guard(s->head->device);
            if (!(r = s->d_peer_first.ensure(nl * 8)) && !(r = s->d_peer_owner.ensure(nl * 4))) {
                cudaError_t e = cudaMemcpy(s->d_peer_first.ptr, from.data(), nl * 8, cudaMemcpyHostToDevice);
                if (e == cudaSuccess) e = cudaMemcpy(s->d_peer_owner.ptr, by.data(), nl * 4, cudaMemcpyHostToDevice);
                if (e != cudaSuccess) r = fail(SPTAG_B200_FAIL, "peer table upload failed: %s", cudaGetErrorString(e));
            }
            if (!r) {
                p.first = (const long long*)s->d_peer_first.ptr;
                p.owner = (const int*)s->d_peer_owner.ptr;
            }
        }
        if (r && !rc) rc = r;
        std::lock_guard<std::mutex> lock(s->mu);
        s->peers = p;
        s->peer_lists = p.first ? count : 0;
    }
    return rc;
}

// Before a host-placed call takes its staging set: a cache whose stages are smaller than the call's (the stage
// parameters grew since the install) is re-installed with the call's.  Locks: the handle's two staging sets; on a group
// member the group's install mutex and every member's sets (GroupSets), and every peer table is rebuilt before they
// are released, since the member's pool moved.
int spann_cache_fit(sptag_b200_spann* s, const SpannSnapshot& sp) {
    const long long need = stage_elems(s, sp);
    {
        std::lock_guard<std::mutex> lock(s->mu);
        if (s->cache_lists.empty() || s->cache_stage >= need) return 0;
    }
    std::unique_ptr<GroupSets> all;
    std::unique_ptr<BothSets> both;
    if (s->group)
        all.reset(new GroupSets(s->group));
    else
        both.reset(new BothSets(s));
    std::vector<int> lists;
    {
        std::lock_guard<std::mutex> lock(s->mu);
        if (s->cache_lists.empty() || s->cache_stage >= need) return 0;
        lists = s->cache_lists;
    }
    const int rc = spann_cache_install(s, lists, need);
    if (!s->group) return rc;
    const int prc = spann_group_peer_tables(s->group);
    return rc ? rc : prc;
}

// A host-placed call's staging set, with a cache (if any) whose stages hold the call's stage: the cache is fitted, the
// set taken, and both again if an install from smaller stage parameters came in between (a cache's stage only grows,
// so the second fit holds).  The fit takes its locks (spann_cache_fit) and releases them before the set is taken.
template <typename Set>
int spann_acquire_fitted(sptag_b200_spann* s, const SpannSnapshot& sp, std::unique_lock<std::mutex>& slock, Set*& set) {
    for (;;) {
        if (int rc = spann_cache_fit(s, sp)) return rc;
        set = s->staging.acquire(slock);
        if (!s->d_cache.ptr || s->cache_stage >= stage_elems(s, sp)) return 0;  // held set: the cache cannot change
        slock.unlock();
    }
}

// Search parameters (SPANN/ParameterDefinitionList.h:110-125), under s->mu; the kHead ones are set and read on the head
// (SPANNIndex.cpp:901) without it
using Spann = sptag_b200_spann;
const Param<Spann> kSpannParams[] = {
    {"MaxCheck", kHead},
    {"B200.IteratorVisitedSet", kHead},  // with the next: the visited sets of the head iterators SPANN iterators open
    {"B200.IteratorVisitedHashEntries", kHead},
    // the one quantizer of the head and the postings (VectorIndex::SetQuantizerADC, VectorIndex.h:136-138)
    {"EnableADC", kHead},
    {"SearchInternalResultNum", &Spann::internal, 0, 0, 2048,
     [](Spann* s, long v) { s->internal = (int)v; spann_update_shape(s); return SPTAG_B200_SUCCESS; }},
    {"SearchPostingPageLimit", &Spann::page_limit, 0, 0, 2048,
     [](Spann* s, long v) { s->page_limit = (int)v; spann_update_shape(s); return SPTAG_B200_SUCCESS; }},
    {"MaxDistRatio", &Spann::max_dist_ratio},
    {"IterativeSearchHeadBatch", &Spann::head_batch, 0, 1, 1024},
    {"B200.SpannDedupEntries", &Spann::dedup_entries, kPow2},
    {"PostingBytes", [](Spann* s, char* o, size_t n) {
         return put(o, n, "%zu", s->d_translate.bytes + s->d_off.bytes + s->d_cnt.bytes + s->d_pages.bytes + s->d_ids.bytes + s->d_rows.bytes);
     }},
    // host placement (sptag_b200_spann_load_ex): the HBM stage per staging set, and what the placement holds and gathered
    {"B200.PostingStageBytes", &Spann::stage_bytes, 0, 0, INT_MAX},
    {"B200.PostingPlacement", [](Spann* s, char* o, size_t n) {
         return put(o, n, "%s", s->file_postings ? "file" : s->host_postings ? "host" : "device");
     }},
    {"B200.PostingHostBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%zu", s->h_posting_bytes); }},
    {"B200.LastGatherBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_gather_bytes); }},
    {"B200.LastGatherRounds", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_gather_rounds); }},
    // file placement: the posting-file bytes the last search, iterator step or cache install read
    {"B200.LastReadBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_read_bytes); }},
    // the HBM cache of lists (sptag_b200_spann_cache_lists): its lists and the pool's bytes
    {"B200.PostingCacheLists", [](Spann* s, char* o, size_t n) { return put(o, n, "%zu", s->cache_lists.size()); }},
    {"B200.PostingCacheBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%lld", s->cache_bytes); }},
    // a group member's (sptag_b200_spann_group_load): lists it reads from a peer's cache, and the part of
    // B200.LastGatherBytes its last search or iterator step copied from peers
    {"B200.PostingPeerLists", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->peer_lists); }},
    {"B200.LastPeerGatherBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_peer_gather_bytes); }},
    {"B200.LastIteratorRounds", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_iter_rounds); }},
    {"B200.LastIteratorDedupBytes", [](Spann* s, char* o, size_t n) { return put(o, n, "%ld", s->last_iter_dedup_bytes); }},
    {"B200.LastPostingKernel", [](Spann* s, char* o, size_t n) { return put(o, n, "%s", kernel_name(s->last_posting_kernel).c_str()); }},
};

// One posting file (OutputSSDIndexFile, ExtraFullGraphSearcher.h:1292-1420; read as LoadingHeadInfo does, :1030-1120):
// int32 listCount, totalDocCount, dim, listPageOffset; per list int32 pageNum, uint16 pageOffset, int32 listEleCount,
// uint16 listPageCount; list l's bytes start at ((listPageOffset + pageNum) << 12) + pageOffset
struct PostingFile {
    FILE* f = nullptr;
    int lists = 0, dim = 0;
    std::vector<long long> start;
    std::vector<int> cnt, pages;
};
int read_posting_header(FILE* f, PostingFile& pf, const char* name) {
    int32_t hdr[4];
    if (std::fread(hdr, 4, 4, f) != 4) return fail(SPTAG_B200_FAIL, "posting file %s: truncated header", name);
    pf.f = f;
    pf.lists = hdr[0];
    pf.dim = hdr[2];
    if (pf.lists < 0) return fail(SPTAG_B200_FAIL, "posting file %s: bad list count %d", name, pf.lists);
    const long long fsz = file_size(f);
    fseeko(f, 16, SEEK_SET);
    pf.start.resize((size_t)pf.lists);
    pf.cnt.resize((size_t)pf.lists);
    pf.pages.resize((size_t)pf.lists);
    for (int i = 0; i < pf.lists; ++i) {
        unsigned char b[12];
        if (std::fread(b, 1, 12, f) != 12) return fail(SPTAG_B200_FAIL, "posting file %s: truncated list infos", name);
        int32_t page_num, ele;
        uint16_t page_off, page_cnt;
        memcpy(&page_num, b, 4);
        memcpy(&page_off, b + 4, 2);
        memcpy(&ele, b + 6, 4);
        memcpy(&page_cnt, b + 10, 2);
        if (ele < 0) return fail(SPTAG_B200_FAIL, "posting file %s: list %d has %d elements", name, i, ele);
        pf.start[i] = (((long long)hdr[3] + page_num) << 12) + page_off;
        pf.cnt[i] = ele;
        pf.pages[i] = page_cnt;
        if (pf.start[i] < 0 || pf.start[i] > fsz) return fail(SPTAG_B200_FAIL, "posting file %s: list %d outside the file", name, i);
    }
    return 0;
}


// spann_fill's placement for a group's first member: HOST, in an allocation every device maps (cudaHostAllocPortable)
constexpr int kPostingsPortable = -1;

// Everything sptag_b200_spann_load reads after the head: the head's [BuildHead] parameters, the search parameters, the
// translate map and the posting files, with the lists' rows and ids placed as `placement` says (SPTAG_B200_POSTINGS_*,
// or kPostingsPortable; FILE reads only the files' headers).  With `shared` (a group's later members: the portable allocation of shared_bytes its first
// member filled from the same folder) the lists' bodies are not read again: the handle maps that allocation, which it
// does not own.  The caller destroys s on failure.
int spann_fill(sptag_b200_spann* s, const std::string& dir, const IniSections& ini, int placement, void* shared = nullptr,
               size_t shared_bytes = 0) {
    auto get = [&](const char* section, const char* name, const char* def) { return ini_get(ini, section, name, def); };
    sptag_b200_handle head = s->head;
    // SPANN::Index::LoadConfig hands every [BuildHead] entry to the head (SPANNIndex.cpp:59-71, :1033-1038)
    load_ref_keys(head, ini, "BuildHead");
    s->vis = head->dim * (int)value_size(head->value_type) + 4;
    s->rearranged = ini_true(get("BuildSSDIndex", "EnablePostingListRearrange", "false")) ? 1 : 0;
    s->internal = atoi(get("BuildSSDIndex", "SearchInternalResultNum", "64").c_str());
    s->max_dist_ratio = strtof(get("BuildSSDIndex", "MaxDistRatio", "10000").c_str(), nullptr);
    s->page_limit = atoi(get("BuildSSDIndex", "SearchPostingPageLimit", "3").c_str());
    s->head_batch = atoi(get("BuildSSDIndex", "IterativeSearchHeadBatch", "32").c_str());
    const long long vector_limit = atoll(get("BuildSSDIndex", "PostingVectorLimit", "118").c_str());
    s->vector_limit_pages = (int)((vector_limit * s->vis + 4095) / 4096);
    DeviceGuard guard(head->device);
    if (!s->staging.create_streams()) return fail(SPTAG_B200_FAIL, "cudaStreamCreate failed");
    cudaStream_t up = s->staging.sets[0].stream;
    // m_vectorTranslateMap: one uint64 per head (SPANNIndex.cpp:133-134), kept as the SizeType the search casts it to
    {
        FileCloser fc;
        const std::string path = dir + "/" + get("Base", "HeadVectorIDs", "SPTAGHeadVectorIDs.bin");
        FILE* f = fc.open(path);
        if (!f) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read %s", path.c_str());
        std::vector<uint64_t> map((size_t)head->n);
        if (std::fread(map.data(), 8, map.size(), f) != map.size())
            return fail(SPTAG_B200_FAIL, "%s holds fewer than %d ids", path.c_str(), head->n);
        std::vector<int32_t> tr(map.size());
        for (size_t i = 0; i < map.size(); ++i) tr[i] = (int32_t)(uint32_t)map[i];
        if (int rc = s->d_translate.ensure(tr.size() * 4)) return rc;
        CUDA_OK(cudaMemcpy(s->d_translate.ptr, tr.data(), tr.size() * 4, cudaMemcpyHostToDevice));
    }
    // the posting files: SSDIndex, SSDIndex_1, ... while they exist (ExtraFullGraphSearcher.h:165-206)
    FileCloser fc;
    std::vector<PostingFile> files;
    std::vector<std::string> paths;
    const std::string base = dir + "/" + get("BuildSSDIndex", "SSDIndex", get("Base", "SSDIndex", "SPTAGFullList.bin").c_str());
    for (std::string cur = base;; cur = base + "_" + std::to_string(files.size())) {
        FILE* f = fc.open(cur);
        if (!f) break;
        files.emplace_back();
        paths.push_back(cur);
        if (int rc = read_posting_header(f, files.back(), cur.c_str())) return rc;
        if (files.back().dim != head->dim)
            return fail(SPTAG_B200_DIMENSION_MISMATCH, "%s: dimension %d, head index %d", cur.c_str(), files.back().dim, head->dim);
    }
    if (files.empty()) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read %s", base.c_str());
    long long total = 0;
    for (const PostingFile& pf : files) {
        for (int i = 0; i < pf.lists; ++i) {
            s->cnt.push_back(pf.cnt[i]);
            s->pages.push_back(pf.pages[i]);
            total += pf.cnt[i];
        }
    }
    s->num_lists = (int)s->cnt.size();
    if (s->num_lists < head->n) return fail(SPTAG_B200_FAIL, "%d posting lists for %d heads", s->num_lists, head->n);
    const size_t rs = head->row_stride, row_bytes = (size_t)s->vis - 4;
    std::vector<long long> off(s->cnt.size());
    for (size_t l = 0, acc = 0; l < off.size(); acc += (size_t)s->cnt[l], ++l) off[l] = (long long)acc;
    if (int rc = s->d_off.ensure(off.size() * 8)) return rc;
    if (int rc = s->d_cnt.ensure(off.size() * 4)) return rc;
    if (int rc = s->d_pages.ensure(off.size() * 4)) return rc;
    const size_t rows_bytes = ((size_t)total + 1) * rs, ids_bytes = ((size_t)total + 1) * 4;
    if (placement == SPTAG_B200_POSTINGS_AUTO) {
        // HBM when the lists fit beside a reserve for the searches' buffers (head results, dedup tables, outputs)
        size_t free_bytes = 0, total_bytes = 0;
        CUDA_OK(cudaMemGetInfo(&free_bytes, &total_bytes));
        placement = free_bytes >= rows_bytes + ids_bytes + kPostingReserve ? SPTAG_B200_POSTINGS_DEVICE : SPTAG_B200_POSTINGS_HOST;
    }
    unsigned char* rows_base = nullptr;
    int32_t* ids_base = nullptr;
    if (shared && shared_bytes != rows_bytes + ids_bytes)
        return fail(SPTAG_B200_FAIL, "the posting lists take %zu bytes, the group's first member loaded %zu",
                    rows_bytes + ids_bytes, shared_bytes);
    if (placement == SPTAG_B200_POSTINGS_HOST || placement == kPostingsPortable) {
        // the rows, then the ids (rows_bytes is a multiple of 16), in the layout they have in HBM
        const unsigned flags = placement == kPostingsPortable ? cudaHostAllocMapped | cudaHostAllocPortable : cudaHostAllocMapped;
        if (!shared && cudaHostAlloc(&s->h_postings, rows_bytes + ids_bytes, flags) != cudaSuccess) {
            s->h_postings = nullptr;
            cudaGetLastError();
            return fail(SPTAG_B200_MEMORY_OVERFLOW, "cudaHostAlloc(%zu) of the posting lists failed", rows_bytes + ids_bytes);
        }
        s->host_postings = true;
        s->h_posting_bytes = rows_bytes + ids_bytes;
        if (!shared) memset(s->h_postings, 0, rows_bytes);
        void* dev = nullptr;
        CUDA_OK(cudaHostGetDevicePointer(&dev, shared ? shared : s->h_postings, 0));
        rows_base = (unsigned char*)dev;
        ids_base = (int32_t*)(rows_base + rows_bytes);
        s->h_rows = rows_base;
        s->h_ids = ids_base;
    } else if (placement != SPTAG_B200_POSTINGS_FILE) {
        if (int rc = s->d_ids.ensure(ids_bytes)) return rc;
        if (int rc = s->d_rows.ensure(rows_bytes)) return rc;
        CUDA_OK(cudaMemset(s->d_rows.ptr, 0, s->d_rows.bytes));
        rows_base = (unsigned char*)s->d_rows.ptr;
        ids_base = (int32_t*)s->d_ids.ptr;
    }
    const cudaMemcpyKind to = s->host_postings ? cudaMemcpyDefault : cudaMemcpyDeviceToDevice;  // UVA: to mapped host memory
    CUDA_OK(cudaMemcpy(s->d_off.ptr, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(s->d_cnt.ptr, s->cnt.data(), off.size() * 4, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(s->d_pages.ptr, s->pages.data(), off.size() * 4, cudaMemcpyHostToDevice));
    if (placement == SPTAG_B200_POSTINGS_FILE) {
        // The lists stay in their files, whose descriptors the handle keeps (dups of the ones the headers were read
        // from).  Nothing is read before the first search, so every list's extent is checked here.
        size_t first_list = 0;
        for (size_t fi = 0; fi < files.size(); ++fi) {
            const PostingFile& pf = files[fi];
            const long long fsz = file_size(pf.f);
            for (int i = 0; i < pf.lists; ++i) {
                if (pf.cnt[i] > 0 && pf.start[i] + (long long)pf.cnt[i] * s->vis > fsz)
                    return fail(SPTAG_B200_FAIL, "posting list %zu runs past the end of its file %s", first_list + i,
                                paths[fi].c_str());
                s->list_file.push_back((int)fi);
                s->list_start.push_back(pf.start[i]);
            }
            first_list += (size_t)pf.lists;
            const int fd = fcntl(fileno(pf.f), F_DUPFD_CLOEXEC, 0);
            if (fd < 0) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot keep %s open: %s", paths[fi].c_str(), strerror(errno));
            s->post_files.fds.push_back(fd);
            s->post_files.paths.push_back(paths[fi]);
        }
        s->host_postings = s->file_postings = true;
        s->readers.reset(new ReadPool(std::min(16u, std::max(1u, std::thread::hardware_concurrency()))));
    }
    if (shared || s->file_postings) {
        std::lock_guard<std::mutex> lock(s->mu);
        spann_update_shape(s);
        return 0;
    }
    // The lists of a file are read in file order, in runs of consecutive lists of at most kRun bytes (a longer list is a
    // run of its own), each run streamed through upload_rows' pinned chunks into one device staging buffer and split
    // there: ParsePostingList lays an element out as int32 id + row, ParsePostingListRearrange as every row of the list,
    // then every id (ExtraFullGraphSearcher.h:1186-1196).  HBM beyond the packed lists: the largest run.
    const long long kRun = 64ll << 20;
    DeviceBuffer stage;
    size_t first_list = 0;
    for (const PostingFile& pf : files) {
        const long long fsz = file_size(pf.f);
        std::vector<int> order;
        for (int i = 0; i < pf.lists; ++i) {
            if (pf.cnt[i] == 0) continue;
            if (pf.start[i] + (long long)pf.cnt[i] * s->vis > fsz)
                return fail(SPTAG_B200_FAIL, "posting list %zu runs past the end of its file", first_list + i);
            order.push_back(i);
        }
        std::sort(order.begin(), order.end(), [&](int x, int y) { return pf.start[x] < pf.start[y]; });
        for (size_t r0 = 0; r0 < order.size();) {
            const long long begin = pf.start[order[r0]];
            long long end = begin + (long long)pf.cnt[order[r0]] * s->vis;
            size_t r1 = r0 + 1;
            for (; r1 < order.size(); ++r1) {
                const long long e = std::max(end, pf.start[order[r1]] + (long long)pf.cnt[order[r1]] * s->vis);
                if (e - begin > kRun) break;
                end = e;
            }
            const size_t bytes = (size_t)(end - begin);
            if (int rc = stage.ensure(bytes)) return rc;
            ArraySource src;
            src.file = pf.f;
            src.offset = begin;
            const size_t pages = bytes >> 12, tail = bytes & 4095;
            if (int rc = upload_rows(src, stage.ptr, pages, 4096, 4096, up)) return rc;
            src.offset = begin + (long long)(pages << 12);
            if (int rc = upload_rows(src, (unsigned char*)stage.ptr + (pages << 12), 1, tail, tail, up)) return rc;
            for (size_t r = r0; r < r1; ++r) {
                const int i = order[r];
                const size_t c = (size_t)pf.cnt[i], l = first_list + (size_t)i;
                const unsigned char* src_list = (const unsigned char*)stage.ptr + (pf.start[i] - begin);
                unsigned char* drow = rows_base + (size_t)off[l] * rs;
                int32_t* did = ids_base + off[l];
                if (s->rearranged) {
                    CUDA_OK(cudaMemcpy2DAsync(drow, rs, src_list, row_bytes, row_bytes, c, to, up));
                    CUDA_OK(cudaMemcpyAsync(did, src_list + c * row_bytes, c * 4, to, up));
                } else {
                    CUDA_OK(cudaMemcpy2DAsync(did, 4, src_list, (size_t)s->vis, 4, c, to, up));
                    CUDA_OK(cudaMemcpy2DAsync(drow, rs, src_list + 4, (size_t)s->vis, row_bytes, c, to, up));
                }
            }
            CUDA_OK(cudaStreamSynchronize(up));  // the next run reuses the staging buffer
            r0 = r1;
        }
        first_list += (size_t)pf.lists;
    }
    std::lock_guard<std::mutex> lock(s->mu);
    spann_update_shape(s);
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// SPANN posting-list build (the SSD stage of SPANN::Index<T>::BuildIndexInternal, SPANNIndex.cpp:889-951, with
// ExtraFullGraphSearcher::BuildIndex, ExtraFullGraphSearcher.h:587-922) from a head that is already built
// ---------------------------------------------------------------------------------------------------------------

// SelectPostingOffset (ExtraFullGraphSearcher.h:1206-1290): lists are placed greedily, each time the one with the largest
// bytes % PageSize that still fits in the current page (the lower id among equals); a page that nothing fits is left
// with its rest as padding.  page_num / page_off: where list i starts in the list area; order: the placement order.
void select_posting_offset(const std::vector<long long>& bytes, std::vector<int>& page_num, std::vector<int>& page_off,
                           std::vector<int>& order) {
    page_num.assign(bytes.size(), 0);
    page_off.assign(bytes.size(), 0);
    order.clear();
    std::set<std::pair<int, int>> rest;  // (-(bytes % 4096), id): largest rest first, then the lower id
    for (size_t i = 0; i < bytes.size(); ++i)
        if (bytes[i] != 0) rest.insert({-(int)(bytes[i] % 4096), (int)i});
    int page = 0, off = 0;
    while (!rest.empty()) {
        const int room = 4096 - off;
        auto it = rest.lower_bound({-room, -1});
        if (it == rest.end() || (room != 4096 && it->first == 0)) {
            ++page;
            off = 0;
            continue;
        }
        const int id = it->second;
        page_num[id] = page;
        page_off[id] = off;
        order.push_back(id);
        off -= it->first;
        if (off == 4096) {
            ++page;
            off = 0;
        }
        page += (int)(bytes[id] / 4096);
        rest.erase(it);
    }
}

// One posting file (OutputSSDIndexFile, ExtraFullGraphSearcher.h:1292-1568) of lists [first, first + nl): the header on
// the host, the list area from the device in windows of kWindow bytes, each copied into one of two pinned buffers so
// that the fwrite of one window overlaps the image and copy of the next.
struct SpannBuildFile {
    const int* d_tonode;          // the sorted edges' tonode
    const unsigned char* d_rows;  // the full rows, row_bytes apart
    int row_bytes, rearranged, num_vectors, dim;
    const std::vector<long long>* edge_off;  // per list: its first sorted edge
    const std::vector<int>* count;           // per list: its elements after the cut
    const std::vector<long long>* row_off;   // nullptr, or per list: its first row of d_rows (gathered rows)
};

// A file's placement: its lists in placement order (file-local ids), where each starts in the list area, the area's
// size (the last list's end, padded to a page) and the header
struct SpannFileLayout {
    std::vector<int> order;
    std::vector<long long> start, bytes;
    std::vector<unsigned char> hdr;
    long long area = 0;
};
void spann_file_layout(const SpannBuildFile& b, int first, int nl, SpannFileLayout& L) {
    const long long vis = b.row_bytes + 4;
    L.bytes.assign((size_t)nl, 0);
    for (int i = 0; i < nl; ++i) L.bytes[i] = (long long)(*b.count)[first + i] * vis;
    std::vector<int> page_num, page_off;
    select_posting_offset(L.bytes, page_num, page_off, L.order);
    // header: list count, vector count, dimension, the list area's first page; per list page, offset, count, pages
    const size_t meta = 16 + 12 * (size_t)nl;
    L.hdr.assign(round_up(meta, 4096), 0);
    const int32_t h4[4] = {nl, b.num_vectors, b.dim, (int32_t)(L.hdr.size() / 4096)};
    memcpy(L.hdr.data(), h4, 16);
    for (int i = 0; i < nl; ++i) {
        unsigned char* e = L.hdr.data() + 16 + 12 * (size_t)i;
        const int32_t pn = L.bytes[i] ? page_num[i] : 0, ele = (*b.count)[first + i];
        const uint16_t po = L.bytes[i] ? (uint16_t)page_off[i] : 0, pc = (uint16_t)((L.bytes[i] + 4095) / 4096);
        memcpy(e, &pn, 4);
        memcpy(e + 4, &po, 2);
        memcpy(e + 6, &ele, 4);
        memcpy(e + 10, &pc, 2);
    }
    L.start.clear();
    for (int id : L.order) L.start.push_back((long long)page_num[id] * 4096 + page_off[id]);
    L.area = L.order.empty() ? 0 : (long long)round_up((size_t)(L.start.back() + L.bytes[L.order.back()]), 4096);
}

// Writes one file: open() writes the header and uploads the placed lists' start, edge offset, count (and row offset);
// write() images and writes the list area's bytes [begin, end) in windows of at most kWindow bytes from the sorted
// edges and rows given; finish() writes the last window.  The areas of successive write() calls follow each other.
struct SpannFileWriter {
    static constexpr long long kWindow = 64ll << 20;
    const SpannBuildFile* b = nullptr;
    const SpannFileLayout* L = nullptr;
    std::string path;
    cudaStream_t stream = nullptr;
    std::unique_ptr<FILE, int (*)(FILE*)> f{nullptr, std::fclose};
    std::vector<int> cnt;  // per placed list
    DeviceBuffer d_start, d_eoff, d_cnt, d_roff, d_win;
    void* pin[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    SpannImageParams p;
    size_t lo = 0;           // the first list that ends after the window's start
    long long next = 0;      // the next window's number (its buffer: number & 1)
    long long pending = -1;  // the window waiting for its fwrite
    long long pending_bytes = 0;
    ~SpannFileWriter() {
        for (int i = 0; i < 2; ++i) {
            if (pin[i]) cudaFreeHost(pin[i]);
            if (ev[i]) cudaEventDestroy(ev[i]);
        }
    }
    // the window size: an upper bound of the device bytes the writer allocates besides the per-list arrays
    static long long window_bytes(long long area) { return std::min(kWindow, area); }
    int open(const SpannBuildFile& bf, const SpannFileLayout& lay, const std::string& file_path, int first, cudaStream_t s) {
        b = &bf;
        L = &lay;
        path = file_path;
        stream = s;
        FILE* fp = std::fopen(path.c_str(), "wb");
        if (!fp) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot write %s", path.c_str());
        f.reset(fp);
        if (std::fwrite(L->hdr.data(), 1, L->hdr.size(), fp) != L->hdr.size())
            return fail(SPTAG_B200_FAIL, "writing %s failed", path.c_str());
        if (L->area == 0) return 0;
        std::vector<long long> eoff, roff;
        for (int id : L->order) {
            eoff.push_back((*b->edge_off)[first + id]);
            cnt.push_back((*b->count)[first + id]);
            if (b->row_off) roff.push_back((*b->row_off)[first + id]);
        }
        const size_t win = (size_t)window_bytes(L->area);
        if (int rc = d_start.ensure(L->start.size() * 8)) return rc;
        if (int rc = d_eoff.ensure(eoff.size() * 8)) return rc;
        if (int rc = d_cnt.ensure(cnt.size() * 4)) return rc;
        if (b->row_off)
            if (int rc = d_roff.ensure(roff.size() * 8)) return rc;
        if (int rc = d_win.ensure(win)) return rc;
        CUDA_OK(cudaMemcpyAsync(d_start.ptr, L->start.data(), L->start.size() * 8, cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(d_eoff.ptr, eoff.data(), eoff.size() * 8, cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(d_cnt.ptr, cnt.data(), cnt.size() * 4, cudaMemcpyHostToDevice, stream));
        if (b->row_off) CUDA_OK(cudaMemcpyAsync(d_roff.ptr, roff.data(), roff.size() * 8, cudaMemcpyHostToDevice, stream));
        for (int i = 0; i < 2; ++i) {
            if (cudaMallocHost(&pin[i], win) != cudaSuccess)
                return fail(SPTAG_B200_MEMORY_OVERFLOW, "pinned window buffer (%zu bytes) failed", win);
            CUDA_OK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
        }
        memset(&p, 0, sizeof(p));
        p.start = (const long long*)d_start.ptr;
        p.edge_off = (const long long*)d_eoff.ptr;
        p.count = (const int*)d_cnt.ptr;
        p.row_off = b->row_off ? (const long long*)d_roff.ptr : nullptr;
        p.row_bytes = b->row_bytes;
        p.rearranged = b->rearranged;
        p.out = (unsigned char*)d_win.ptr;
        // the first stream work on the uploads' host vectors must end before they go out of scope
        CUDA_OK(cudaStreamSynchronize(stream));
        return 0;
    }
    int write(long long begin, long long end, const int* d_tonode, const unsigned char* d_rows) {
        const long long vis = b->row_bytes + 4;
        p.tonode = d_tonode;
        p.rows = d_rows;
        for (long long wb = begin; wb < end; wb += kWindow) {
            p.win_begin = wb;
            p.win_end = std::min(end, wb + kWindow);
            while (lo < L->start.size() && L->start[lo] + (long long)cnt[lo] * vis <= p.win_begin) ++lo;
            size_t hi = lo;
            while (hi < L->start.size() && L->start[hi] < p.win_end) ++hi;
            p.first_list = (int)lo;
            p.num_lists = (int)(hi - lo);
            const long long w = next++;
            CUDA_OK(cudaMemsetAsync(d_win.ptr, 0, (size_t)(p.win_end - p.win_begin), stream));
            CUDA_OK(launch_spann_posting_image(p, stream));
            g_launches++;
            CUDA_OK(cudaMemcpyAsync(pin[w & 1], d_win.ptr, (size_t)(p.win_end - p.win_begin), cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaEventRecord(ev[w & 1], stream));
            if (int rc = write_pending()) return rc;
            pending = w;
            pending_bytes = p.win_end - p.win_begin;
        }
        return 0;
    }
    int write_pending() {
        if (pending < 0) return 0;
        const int i = (int)(pending & 1);
        pending = -1;
        CUDA_OK(cudaEventSynchronize(ev[i]));
        const size_t n = (size_t)pending_bytes;
        if (std::fwrite(pin[i], 1, n, f.get()) != n) return fail(SPTAG_B200_FAIL, "writing %s failed", path.c_str());
        return 0;
    }
    int finish() {
        if (int rc = write_pending()) return rc;
        if (std::fflush(f.get()) != 0) return fail(SPTAG_B200_FAIL, "writing %s failed", path.c_str());
        return 0;
    }
};

int write_posting_file(const SpannBuildFile& b, const std::string& path, int first, int nl, cudaStream_t stream) {
    SpannFileLayout L;
    spann_file_layout(b, first, nl, L);
    SpannFileWriter w;
    if (int rc = w.open(b, L, path, first, stream)) return rc;
    if (L.area == 0) return 0;
    if (int rc = w.write(0, L.area, b.d_tonode, b.d_rows)) return rc;
    return w.finish();
}

// Owns what one sptag_b200_spann_build call allocates on the device, in pinned host memory and its streams; frees them
// (and unregisters the caller's rows) with the device current
struct SpannBuildState {
    sptag_b200_handle head = nullptr;
    cudaStream_t stream = nullptr, copy = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr}, copied[2] = {nullptr, nullptr};
    DeviceBuffer d_rows, d_head, d_list, d_ids, d_dists, d_keys[2], d_tonode[2], d_size, d_counters, d_temp;
    DeviceBuffer d_brows[2], d_flags, d_group_of, d_arena;  // the streamed path's
    void* h_store = nullptr;            // the streamed path's pinned edge store
    const void* registered = nullptr;   // the caller's rows, registered by this call
    ~SpannBuildState() {
        if (head) {
            DeviceGuard guard(head->device);
            for (cudaStream_t s : {stream, copy})
                if (s) cudaStreamSynchronize(s);
            for (cudaEvent_t e : {ev[0], ev[1], copied[0], copied[1]})
                if (e) cudaEventDestroy(e);
            for (cudaStream_t s : {stream, copy})
                if (s) cudaStreamDestroy(s);
            for (DeviceBuffer* b : {&d_rows, &d_head, &d_list, &d_ids, &d_dists, &d_keys[0], &d_keys[1], &d_tonode[0],
                                    &d_tonode[1], &d_size, &d_counters, &d_temp, &d_brows[0], &d_brows[1], &d_flags,
                                    &d_group_of, &d_arena})
                b->release();
            if (h_store) cudaFreeHost(h_store);
            if (registered) cudaHostUnregister((void*)registered);
        }
        sptag_b200_destroy(head);
    }
    // device milliseconds between ev[0] and ev[1], recorded around work on the stream
    int elapsed(float& acc) {
        CUDA_OK(cudaEventSynchronize(ev[1]));
        float ms = 0;
        CUDA_OK(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        acc += ms;
        return 0;
    }
};

// What both build paths read from the folder and the call
struct SpannBuildConfig {
    std::string dir, out;  // out: the first posting file's path
    int value_type = 0, metric = 0, num = 0, dim = 0, normalized = 0, num_heads = 0;
    int replicas = 0, k = 0, rearranged = 0, file_num = 0;
    float rng_factor = 0;
    long long limit = INT_MAX;  // elements a list keeps after the cut
    size_t row_bytes = 0;
    std::vector<unsigned char> is_head;
    long long searched = 0;     // vectors that are not heads
};

// The ini, the refusals, the head (loaded into st.head with [BuildSSDIndex] MaxCheck) and the head-id file (rewritten
// first with ExcludeHead false)
int spann_build_prepare(const char* folder, const void* vectors, int32_t num, int32_t dim, int32_t normalized, int32_t device,
                        SpannBuildState& st, SpannBuildConfig& c) {
    if (!folder || !vectors || num <= 0) return fail(SPTAG_B200_EMPTY_DATA, "no vectors to build from");
    c.dir = folder;
    IniSections ini;
    if (!read_ini(c.dir + "/indexloader.ini", ini)) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot open %s/indexloader.ini", folder);
    auto get = [&](const char* section, const char* name, const char* def) { return ini_get(ini, section, name, def); };
    // Refusals: what the device does not reproduce (SPANN/ParameterDefinitionList.h:34, :80-92)
    if (!get("Base", "QuantizerFilePath", "").empty())
        return fail(SPTAG_B200_LACK_OF_INPUTS, "posting lists of quantized SPANN indexes are not built on the device");
    for (const char* key : {"EnableDataCompression", "EnableDeltaEncoding", "OutputEmptyReplicaID"})
        if (ini_true(get("BuildSSDIndex", key, "false")))
            return fail(SPTAG_B200_LACK_OF_INPUTS, "%s is not supported by the device build", key);
    c.value_type = enum_value(kValueTypes, get("Base", "ValueType", "Undefined"));
    c.metric = enum_value(kDistCalcMethods, get("Base", "DistCalcMethod", "Undefined"));
    if (c.value_type < 0 || c.metric < 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported ValueType or DistCalcMethod");
    const int ini_dim = atoi(get("Base", "Dim", "-1").c_str());
    if (dim <= 0 || (ini_dim != -1 && ini_dim != dim))
        return fail(SPTAG_B200_DIMENSION_MISMATCH, "vectors have %d dimensions, the folder %d", dim, ini_dim);
    c.replicas = atoi(get("BuildSSDIndex", "ReplicaCount", "8").c_str());
    c.k = atoi(get("BuildSSDIndex", "InternalResultNum", "64").c_str());
    c.rng_factor = strtof(get("BuildSSDIndex", "RNGFactor", "1.0").c_str(), nullptr);
    int page_limit = atoi(get("BuildSSDIndex", "PostingPageLimit", "3").c_str());
    const long long vector_limit = atoll(get("BuildSSDIndex", "PostingVectorLimit", "118").c_str());
    const bool exclude_head = ini_true(get("BuildSSDIndex", "ExcludeHead", "true"));
    c.rearranged = ini_true(get("BuildSSDIndex", "EnablePostingListRearrange", "false")) ? 1 : 0;
    const std::string max_check = get("BuildSSDIndex", "MaxCheck", "4096");
    c.file_num = atoi(get("Base", "SSDIndexFileNum", "1").c_str());
    if (c.replicas < 1 || c.replicas > kSpannBuildMaxReplicas || c.k < 1 || c.k > 2048 || c.file_num < 1 ||
        !std::isfinite(c.rng_factor))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "ReplicaCount %d (1..%d), InternalResultNum %d (1..2048) or SSDIndexFileNum %d",
                    c.replicas, kSpannBuildMaxReplicas, c.k, c.file_num);

    const std::string head_dir = c.dir + "/" + get("Base", "HeadIndexFolder", "HeadIndex");
    if (int rc = sptag_b200_load(head_dir.c_str(), device, 0, &st.head)) return rc;
    sptag_b200_handle h = st.head;
    if (h->q_type != 0 || h->value_type != c.value_type || h->metric != c.metric)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "the head index's value type or distance does not match the folder's");
    if (h->dim != dim) return fail(SPTAG_B200_DIMENSION_MISMATCH, "vectors have %d dimensions, the head index %d", dim, h->dim);
    // SPANNIndex.cpp:901: the head searches with [BuildSSDIndex] MaxCheck
    if (int rc = sptag_b200_set_param(h, "MaxCheck", max_check.c_str())) return rc;
    c.num_heads = h->n;
    // SPANNIndex.cpp:914-925: with ExcludeHead false every head id becomes MaxSize, so that no vector is skipped
    const std::string id_path = c.dir + "/" + get("Base", "HeadVectorIDs", "SPTAGHeadVectorIDs.bin");
    if (!exclude_head) {
        FILE* f = std::fopen(id_path.c_str(), "wb");
        if (!f) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot write %s", id_path.c_str());
        const std::vector<uint64_t> ids((size_t)c.num_heads, (uint64_t)INT_MAX);
        const bool ok = std::fwrite(ids.data(), 8, ids.size(), f) == ids.size();
        if (std::fclose(f) != 0 || !ok) return fail(SPTAG_B200_FAIL, "writing %s failed", id_path.c_str());
    }
    // the head-id set: every uint64 of the file cast to SizeType (ExtraFullGraphSearcher.h:604-616)
    c.is_head.assign((size_t)num, 0);
    {
        std::vector<char> blob;
        if (!read_file(id_path, blob)) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read %s", id_path.c_str());
        for (size_t i = 0; i + 8 <= blob.size(); i += 8) {
            uint64_t v;
            memcpy(&v, blob.data() + i, 8);
            const int32_t id = (int32_t)(uint32_t)v;
            if (id >= 0 && id < num) c.is_head[(size_t)id] = 1;
        }
    }
    c.searched = 0;
    for (unsigned char x : c.is_head) c.searched += !x;
    c.num = num;
    c.dim = dim;
    c.normalized = normalized;
    c.row_bytes = (size_t)dim * value_size(c.value_type);
    // the posting cut (ExtraFullGraphSearcher.h:722-760): PostingPageLimit is first raised to the pages of
    // PostingVectorLimit elements; each list keeps its first limit elements
    const int vis = (int)c.row_bytes + 4;
    c.limit = INT_MAX;
    if (page_limit > 0) {
        page_limit = std::max(page_limit, (int)((vector_limit * vis + 4095) / 4096));
        c.limit = (long long)page_limit * 4096 / vis;
    }
    c.out = c.dir + "/" + get("Base", "SSDIndex", "SPTAGFullList.bin");
    // SSDIndexFileNum files of ceil(lists / files) lists each (ExtraFullGraphSearcher.h:796-802)
    const int per_file = (c.num_heads + c.file_num - 1) / c.file_num;
    if ((long long)(c.file_num - 1) * per_file > c.num_heads)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "SSDIndexFileNum %d leaves a file without lists", c.file_num);
    return 0;
}

// Lists [first, first + nl) of posting file i
void spann_file_lists(const SpannBuildConfig& c, int i, int& first, int& nl) {
    const int per_file = (c.num_heads + c.file_num - 1) / c.file_num;
    first = i * per_file;
    nl = std::min(c.num_heads, first + per_file) - first;
}
std::string spann_file_path(const SpannBuildConfig& c, int i) { return i == 0 ? c.out : c.out + "_" + std::to_string(i); }

// The sort's scratch bytes for n edges
size_t spann_sort_scratch(long long n, int end_bit, cudaStream_t stream) {
    size_t t = 0;
    if (spann_sort_edges(nullptr, &t, nullptr, nullptr, nullptr, nullptr, (int)n, end_bit, stream) != cudaSuccess) return SIZE_MAX / 4;
    return t;
}
size_t spann_select_scratch(int n, cudaStream_t stream) {
    size_t t = 0;
    if (spann_select_edges(nullptr, &t, nullptr, nullptr, n, 0, 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr, stream) !=
        cudaSuccess)
        return SIZE_MAX / 4;
    return t;
}
// SortSelections: node, then distance, then tonode; unfilled edges (node = num_heads) last
int spann_end_bit(int num_heads) {
    int end_bit = 32;
    while (end_bit < 64 && ((unsigned long long)num_heads >> (end_bit - 32)) != 0) ++end_bit;
    return end_bit;
}

// The resident path: the rows and every edge in HBM (sptag_b200_spann_build)
int spann_build_resident(SpannBuildConfig& c, SpannBuildState& st, const void* vectors, int64_t* stats) {
    sptag_b200_handle h = st.head;
    const int num = c.num, dim = c.dim, k = c.k, num_heads = c.num_heads;
    const size_t row_bytes = c.row_bytes, edges = (size_t)num * c.replicas;
    const std::vector<unsigned char>& is_head = c.is_head;
    DeviceGuard guard(h->device);
    CUDA_OK(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : st.ev) CUDA_OK(cudaEventCreate(&e));
    cudaStream_t stream = st.stream;
    const int kBatch = 1 << 16;
    const int batch = std::min(num, kBatch);
    if (int rc = st.d_rows.ensure((size_t)num * row_bytes)) return rc;
    for (int i = 0; i < 2; ++i) {
        if (int rc = st.d_keys[i].ensure(edges * 8)) return rc;
        if (int rc = st.d_tonode[i].ensure(edges * 4)) return rc;
    }
    if (int rc = st.d_head.ensure((size_t)num)) return rc;
    if (int rc = st.d_list.ensure(((size_t)batch + 1) * 4)) return rc;
    if (int rc = st.d_ids.ensure((size_t)batch * k * 4)) return rc;
    if (int rc = st.d_dists.ensure((size_t)batch * k * 4)) return rc;
    if (int rc = st.d_size.ensure((size_t)num_heads * 4 + 4)) return rc;
    if (int rc = st.d_counters.ensure(16)) return rc;  // rejections (uint64), the non-finite flag
    unsigned long long* d_rejected = (unsigned long long*)st.d_counters.ptr;
    int* d_bad = (int*)((unsigned char*)st.d_counters.ptr + 8);
    CUDA_OK(cudaMemsetAsync(st.d_counters.ptr, 0, 16, stream));
    CUDA_OK(cudaMemsetAsync(st.d_size.ptr, 0, (size_t)num_heads * 4, stream));
    CUDA_OK(cudaMemcpyAsync(st.d_head.ptr, is_head.data(), (size_t)num, cudaMemcpyHostToDevice, stream));
    ArraySource src;
    src.ptr = vectors;
    if (int rc = upload_rows(src, st.d_rows.ptr, (size_t)num, row_bytes, row_bytes, stream)) return rc;
    unsigned char* rows = (unsigned char*)st.d_rows.ptr;
    // sort and NaN have no order (std::sort under NaN is undefined): rows must be finite
    if (c.value_type == SPTAG_B200_VT_FLOAT) {
        CUDA_OK(launch_spann_nonfinite_check((const float*)rows, (size_t)num * dim, d_bad, stream));
        int bad = 0;
        CUDA_OK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (bad) return fail(SPTAG_B200_LACK_OF_INPUTS, "a row holds a NaN or an infinity");
    }
    // ExtraFullGraphSearcher.h:650: Cosine rows are normalised unless the caller says they are
    if (c.metric == SPTAG_B200_METRIC_COSINE && !c.normalized) {
        const int base = value_base(c.value_type);
        with_elem(h, [&](auto el) {
            normalize_rows_kernel<typename decltype(el)::type><<<(unsigned)((num + 127) / 128), 128, 0, stream>>>(
                rows, row_bytes, 0, num, dim, base);
        });
        g_launches++;
        CUDA_OK(cudaGetLastError());
    }
    // ApproximateRNG in batches of rows: the head search at K = InternalResultNum for the batch's non-head rows (queries
    // read in place through the query list), then the RNG selection of the whole batch
    const MetricElem me = metric_elem(h);
    float ms_search = 0, ms_rng = 0, ms_sort = 0;
    long long searched = 0;
    std::vector<unsigned int> list((size_t)batch + 1);
    SpannRngParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.res_ids = (const int*)st.d_ids.ptr;
    rp.res_dists = (const float*)st.d_dists.ptr;
    rp.k = k;
    rp.head = (const unsigned char*)st.d_head.ptr;
    rp.rows = (const unsigned char*)h->d_vectors.ptr;
    rp.row_stride = h->row_stride;
    rp.dim = dim;
    rp.simd_width = h->simd_width;
    rp.replicas = c.replicas;
    rp.num_heads = num_heads;
    rp.rng_factor = c.rng_factor;
    rp.keys = (unsigned long long*)st.d_keys[0].ptr;
    rp.tonode = (int*)st.d_tonode[0].ptr;
    rp.list_size = (int*)st.d_size.ptr;
    rp.rejected = d_rejected;
    rp.bad = d_bad;
    for (int b0 = 0; b0 < num; b0 += batch) {
        const int nb = std::min(batch, num - b0);
        unsigned int cq = 0;
        for (int i = 0; i < nb; ++i)
            if (!is_head[(size_t)b0 + i]) list[1 + cq++] = (unsigned int)i;
        list[0] = cq;
        searched += cq;
        CUDA_OK(cudaMemcpyAsync(st.d_list.ptr, list.data(), ((size_t)cq + 1) * 4, cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaEventRecord(st.ev[0], stream));
        if (cq > 0) {
            CallOpts opts;
            opts.search_deleted = 0;
            opts.d_query_list = (const unsigned int*)st.d_list.ptr;
            std::lock_guard<std::mutex> lock(h->mu);
            if (int rc = search_device_impl(h, rows + (size_t)b0 * row_bytes, nb, k, (int*)st.d_ids.ptr,
                                            (float*)st.d_dists.ptr, nullptr, stream, false, opts))
                return rc;
        }
        CUDA_OK(cudaEventRecord(st.ev[1], stream));
        if (int rc = st.elapsed(ms_search)) return rc;  // also frees `list` for the next batch
        rp.first = b0;
        rp.num = nb;
        CUDA_OK(cudaEventRecord(st.ev[0], stream));
        CUDA_OK(launch_spann_rng_select(rp, me.cosine, me.elem, stream));
        g_launches++;
        CUDA_OK(cudaEventRecord(st.ev[1], stream));
        if (int rc = st.elapsed(ms_rng)) return rc;
    }
    int bad = 0;
    unsigned long long rejected = 0;
    CUDA_OK(cudaMemcpy(&bad, d_bad, 4, cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(&rejected, d_rejected, 8, cudaMemcpyDeviceToHost));
    if (bad) return fail(SPTAG_B200_LACK_OF_INPUTS, "a distance is not finite");
    const int end_bit = spann_end_bit(num_heads);
    size_t temp_bytes = 0;
    CUDA_OK(spann_sort_edges(nullptr, &temp_bytes, nullptr, nullptr, nullptr, nullptr, (int)edges, end_bit, stream));
    if (int rc = st.d_temp.ensure(std::max<size_t>(temp_bytes, 1))) return rc;
    CUDA_OK(cudaEventRecord(st.ev[0], stream));
    CUDA_OK(spann_sort_edges(st.d_temp.ptr, &temp_bytes, (const unsigned long long*)st.d_keys[0].ptr,
                             (unsigned long long*)st.d_keys[1].ptr, (const int*)st.d_tonode[0].ptr, (int*)st.d_tonode[1].ptr,
                             (int)edges, end_bit, stream));
    g_launches++;
    CUDA_OK(cudaEventRecord(st.ev[1], stream));
    if (int rc = st.elapsed(ms_sort)) return rc;
    st.d_keys[0].release();
    st.d_tonode[0].release();
    st.d_temp.release();
    std::vector<int> size((size_t)num_heads);
    CUDA_OK(cudaMemcpy(size.data(), st.d_size.ptr, (size_t)num_heads * 4, cudaMemcpyDeviceToHost));
    std::vector<long long> edge_off((size_t)num_heads);
    std::vector<int> count((size_t)num_heads);
    long long before = 0, after = 0;
    for (int l = 0; l < num_heads; ++l) {
        edge_off[l] = before;
        before += size[l];
        count[l] = (int)std::min<long long>(size[l], c.limit);
        after += count[l];
    }
    const auto t0 = std::chrono::steady_clock::now();
    SpannBuildFile bf;
    bf.d_tonode = (const int*)st.d_tonode[1].ptr;
    bf.d_rows = rows;
    bf.row_bytes = (int)row_bytes;
    bf.rearranged = c.rearranged;
    bf.num_vectors = num;
    bf.dim = dim;
    bf.edge_off = &edge_off;
    bf.count = &count;
    bf.row_off = nullptr;
    for (int i = 0; i < c.file_num; ++i) {
        int first, nl;
        spann_file_lists(c, i, first, nl);
        if (int rc = write_posting_file(bf, spann_file_path(c, i), first, nl, stream)) return rc;
    }
    const double ms_write = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const int64_t out[8] = {searched, (int64_t)rejected, before, after, (int64_t)(ms_search * 1000.0),
                            (int64_t)(ms_rng * 1000.0), (int64_t)(ms_sort * 1000.0), (int64_t)(ms_write * 1000.0)};
    memcpy(stats, out, sizeof(out));
    return SPTAG_B200_SUCCESS;
}

// The resident path's device bytes (sptag_b200.h): the rows, 24 B per edge, the sort's scratch, one search batch of
// results and the 64 MB window
long long spann_resident_bytes(const SpannBuildConfig& c, cudaStream_t stream) {
    const long long edges = (long long)c.num * c.replicas;
    return (long long)c.num * (long long)c.row_bytes + 24 * edges +
           (long long)spann_sort_scratch(std::min<long long>(edges, INT_MAX), spann_end_bit(c.num_heads), stream) +
           (long long)std::min(c.num, 1 << 16) * c.k * 8 + SpannFileWriter::kWindow;
}

// The streamed path's pass 1 for batches of B rows (sptag_b200.h)
long long spann_pass1_bytes(const SpannBuildConfig& c, long long B, cudaStream_t stream) {
    const long long per_row = 2 * (long long)c.row_bytes + 1 + 4 + 8ll * c.k + 25ll * c.replicas;
    return B * per_row + 4 + (long long)spann_select_scratch((int)(B * c.replicas), stream) + 32 + 4ll * c.num_heads + 4;
}

// The streamed path: the rows stay in the caller's (mapped) buffer, the edges in a pinned host store, and the posting
// files are written in groups of lists whose edges and rows fit the budget
int spann_build_streamed(SpannBuildConfig& c, SpannBuildState& st, const void* vectors, long long budget, int64_t* stats) {
    sptag_b200_handle h = st.head;
    const int num = c.num, dim = c.dim, k = c.k, num_heads = c.num_heads, R = c.replicas;
    const size_t row_bytes = c.row_bytes;
    const std::vector<unsigned char>& is_head = c.is_head;
    DeviceGuard guard(h->device);
    CUDA_OK(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&st.copy, cudaStreamNonBlocking));
    for (cudaEvent_t& e : st.ev) CUDA_OK(cudaEventCreate(&e));
    for (cudaEvent_t& e : st.copied) CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    cudaStream_t stream = st.stream;
    // pass 1's batch: 65536 rows, halved until its buffers fit
    long long B = std::min(num, 1 << 16);
    while (B > 1 && spann_pass1_bytes(c, B, stream) > budget) B = (B + 1) / 2;
    if (spann_pass1_bytes(c, B, stream) > budget)
        return fail(SPTAG_B200_MEMORY_OVERFLOW, "a device budget of %lld bytes is below the %lld bytes of a one-row batch",
                    budget, spann_pass1_bytes(c, 1, stream));
    // the pinned edge store: every filled edge, 12 B (key, vector id)
    const long long per_vector = std::min({R, k, num_heads});
    const long long store_cap = c.searched * per_vector;
    if (store_cap > 0 && cudaHostAlloc(&st.h_store, (size_t)store_cap * 12, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        st.h_store = nullptr;
        return fail(SPTAG_B200_MEMORY_OVERFLOW, "the pinned edge store (%lld bytes) cannot be allocated", store_cap * 12);
    }
    unsigned long long* h_keys = (unsigned long long*)st.h_store;
    int* h_tonode = (int*)((unsigned char*)st.h_store + (size_t)store_cap * 8);
    // the caller's rows, mapped; a buffer registered before is used as it is
    const size_t all_rows = (size_t)num * row_bytes;
    cudaError_t re = cudaHostRegister((void*)vectors, all_rows, cudaHostRegisterMapped);
    if (re == cudaSuccess) {
        st.registered = vectors;
    } else if (re == cudaErrorHostMemoryAlreadyRegistered) {
        cudaGetLastError();
    } else {
        cudaGetLastError();
        return fail(SPTAG_B200_FAIL, "cudaHostRegister of the rows failed: %s", cudaGetErrorString(re));
    }
    void* d_src = nullptr;
    CUDA_OK(cudaHostGetDevicePointer(&d_src, (void*)vectors, 0));
    const unsigned char* src_rows = (const unsigned char*)vectors;

    // pass 1: search, RNG selection and the filled edges appended to the store, batch by batch
    const long long BR = B * R;
    for (int i = 0; i < 2; ++i)
        if (int rc = st.d_brows[i].ensure((size_t)B * row_bytes)) return rc;
    if (int rc = st.d_head.ensure((size_t)B)) return rc;
    if (int rc = st.d_list.ensure(((size_t)B + 1) * 4)) return rc;
    if (int rc = st.d_ids.ensure((size_t)B * k * 4)) return rc;
    if (int rc = st.d_dists.ensure((size_t)B * k * 4)) return rc;
    for (int i = 0; i < 2; ++i) {
        if (int rc = st.d_keys[i].ensure((size_t)BR * 8)) return rc;
        if (int rc = st.d_tonode[i].ensure((size_t)BR * 4)) return rc;
    }
    if (int rc = st.d_flags.ensure((size_t)BR)) return rc;
    size_t sel_bytes = spann_select_scratch((int)BR, stream);
    if (int rc = st.d_temp.ensure(std::max<size_t>(sel_bytes, 1))) return rc;
    if (int rc = st.d_counters.ensure(32)) return rc;  // rejections (uint64), the two non-finite flags, the selected count
    if (int rc = st.d_size.ensure((size_t)num_heads * 4 + 4)) return rc;
    unsigned long long* d_rejected = (unsigned long long*)st.d_counters.ptr;
    int* d_bad = (int*)((unsigned char*)st.d_counters.ptr + 8);
    int* d_row_bad = d_bad + 1;
    int* d_nsel = d_bad + 2;
    CUDA_OK(cudaMemsetAsync(st.d_counters.ptr, 0, 32, stream));
    CUDA_OK(cudaMemsetAsync(st.d_size.ptr, 0, (size_t)num_heads * 4, stream));
    const MetricElem me = metric_elem(h);
    const bool normalize = c.metric == SPTAG_B200_METRIC_COSINE && !c.normalized;
    const int base = value_base(c.value_type);
    float ms_search = 0, ms_rng = 0, ms_sort = 0;
    long long searched = 0, batches = 0, h2d = 0, stored = 0;
    std::vector<unsigned int> list((size_t)B + 1);
    SpannRngParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.res_ids = (const int*)st.d_ids.ptr;
    rp.res_dists = (const float*)st.d_dists.ptr;
    rp.k = k;
    rp.first = 0;  // batch-local vector ids; the selection adds the batch's first id
    rp.head = (const unsigned char*)st.d_head.ptr;
    rp.rows = (const unsigned char*)h->d_vectors.ptr;
    rp.row_stride = h->row_stride;
    rp.dim = dim;
    rp.simd_width = h->simd_width;
    rp.replicas = R;
    rp.num_heads = num_heads;
    rp.rng_factor = c.rng_factor;
    rp.keys = (unsigned long long*)st.d_keys[0].ptr;
    rp.tonode = (int*)st.d_tonode[0].ptr;
    rp.list_size = (int*)st.d_size.ptr;
    rp.rejected = d_rejected;
    rp.bad = d_bad;
    // batch i's rows go to d_brows[i & 1] on the copy stream while batch i - 1 is searched
    auto copy_batch = [&](int b0) -> int {
        const int nb = std::min<long long>(B, num - b0);
        const int slot = (int)((b0 / B) & 1);
        CUDA_OK(cudaMemcpyAsync(st.d_brows[slot].ptr, src_rows + (size_t)b0 * row_bytes, (size_t)nb * row_bytes,
                                cudaMemcpyHostToDevice, st.copy));
        CUDA_OK(cudaEventRecord(st.copied[slot], st.copy));
        h2d += (long long)nb * (long long)row_bytes;
        return 0;
    };
    if (int rc = copy_batch(0)) return rc;
    for (int b0 = 0; b0 < num; b0 += (int)B) {
        const int nb = (int)std::min<long long>(B, num - b0);
        const int slot = (int)((b0 / B) & 1);
        unsigned char* rows = (unsigned char*)st.d_brows[slot].ptr;
        // the other buffer was last read by the previous batch's search, which the host has waited for
        if (b0 + B < num)
            if (int rc = copy_batch((int)(b0 + B))) return rc;
        CUDA_OK(cudaStreamWaitEvent(stream, st.copied[slot], 0));
        ++batches;
        if (c.value_type == SPTAG_B200_VT_FLOAT)
            CUDA_OK(launch_spann_nonfinite_check((const float*)rows, (size_t)nb * dim, d_row_bad, stream));
        if (normalize) {
            with_elem(h, [&](auto el) {
                normalize_rows_kernel<typename decltype(el)::type><<<(unsigned)((nb + 127) / 128), 128, 0, stream>>>(
                    rows, row_bytes, 0, nb, dim, base);
            });
            g_launches++;
            CUDA_OK(cudaGetLastError());
        }
        unsigned int cq = 0;
        for (int i = 0; i < nb; ++i)
            if (!is_head[(size_t)b0 + i]) list[1 + cq++] = (unsigned int)i;
        list[0] = cq;
        searched += cq;
        CUDA_OK(cudaMemcpyAsync(st.d_list.ptr, list.data(), ((size_t)cq + 1) * 4, cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(st.d_head.ptr, is_head.data() + b0, (size_t)nb, cudaMemcpyHostToDevice, stream));
        int row_bad = 0;
        CUDA_OK(cudaMemcpyAsync(&row_bad, d_row_bad, 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (row_bad) return fail(SPTAG_B200_LACK_OF_INPUTS, "a row holds a NaN or an infinity");
        CUDA_OK(cudaEventRecord(st.ev[0], stream));
        if (cq > 0) {
            CallOpts opts;
            opts.search_deleted = 0;
            opts.d_query_list = (const unsigned int*)st.d_list.ptr;
            std::lock_guard<std::mutex> lock(h->mu);
            if (int rc = search_device_impl(h, rows, nb, k, (int*)st.d_ids.ptr, (float*)st.d_dists.ptr, nullptr, stream,
                                            false, opts))
                return rc;
        }
        CUDA_OK(cudaEventRecord(st.ev[1], stream));
        if (int rc = st.elapsed(ms_search)) return rc;  // also frees `list` and this batch's rows
        rp.num = nb;
        CUDA_OK(cudaEventRecord(st.ev[0], stream));
        CUDA_OK(launch_spann_rng_select(rp, me.cosine, me.elem, stream));
        g_launches++;
        // the filled edges, in vector-id order, with global vector ids
        CUDA_OK(spann_select_edges(st.d_temp.ptr, &sel_bytes, (const unsigned long long*)st.d_keys[0].ptr,
                                   (int*)st.d_tonode[0].ptr, (int)(nb * R), b0, num_heads, nullptr, 0,
                                   (unsigned char*)st.d_flags.ptr, (unsigned long long*)st.d_keys[1].ptr,
                                   (int*)st.d_tonode[1].ptr, d_nsel, stream));
        g_launches += 3;
        CUDA_OK(cudaEventRecord(st.ev[1], stream));
        if (int rc = st.elapsed(ms_rng)) return rc;
        int nsel = 0;
        CUDA_OK(cudaMemcpy(&nsel, d_nsel, 4, cudaMemcpyDeviceToHost));
        if (stored + nsel > store_cap) return fail(SPTAG_B200_FAIL, "the edge store overflowed");
        CUDA_OK(cudaMemcpyAsync(h_keys + stored, st.d_keys[1].ptr, (size_t)nsel * 8, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(h_tonode + stored, st.d_tonode[1].ptr, (size_t)nsel * 4, cudaMemcpyDeviceToHost, stream));
        stored += nsel;
    }
    CUDA_OK(cudaStreamSynchronize(stream));
    int bad = 0;
    unsigned long long rejected = 0;
    CUDA_OK(cudaMemcpy(&bad, d_bad, 4, cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(&rejected, d_rejected, 8, cudaMemcpyDeviceToHost));
    if (bad) return fail(SPTAG_B200_LACK_OF_INPUTS, "a distance is not finite");
    std::vector<int> size((size_t)num_heads);
    CUDA_OK(cudaMemcpy(size.data(), st.d_size.ptr, (size_t)num_heads * 4, cudaMemcpyDeviceToHost));
    for (DeviceBuffer* b : {&st.d_brows[0], &st.d_brows[1], &st.d_head, &st.d_list, &st.d_ids, &st.d_dists, &st.d_keys[0],
                            &st.d_keys[1], &st.d_tonode[0], &st.d_tonode[1], &st.d_flags, &st.d_temp, &st.d_size})
        b->release();
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<int> count((size_t)num_heads);
    long long before = 0, after = 0, largest = -1;
    for (int l = 0; l < num_heads; ++l) {
        before += size[l];
        count[l] = (int)std::min<long long>(size[l], c.limit);
        after += count[l];
        if (count[l] > 0 && (largest < 0 || size[l] > size[largest])) largest = l;
    }
    if (before != stored) return fail(SPTAG_B200_FAIL, "%lld edges stored, %lld counted", stored, before);

    // placement, and the groups: runs of placed lists whose edges, sort buffers and gathered rows fit
    SpannBuildFile bf;
    std::vector<long long> edge_off((size_t)num_heads, 0), row_off((size_t)num_heads, 0);
    bf.d_tonode = nullptr;
    bf.d_rows = nullptr;
    bf.row_bytes = (int)row_bytes;
    bf.rearranged = c.rearranged;
    bf.num_vectors = num;
    bf.dim = dim;
    bf.edge_off = &edge_off;
    bf.count = &count;
    bf.row_off = &row_off;
    std::vector<SpannFileLayout> layouts((size_t)c.file_num);
    long long max_lists = 0, max_window = 0;
    for (int i = 0; i < c.file_num; ++i) {
        int first, nl;
        spann_file_lists(c, i, first, nl);
        spann_file_layout(bf, first, nl, layouts[i]);
        max_lists = std::max<long long>(max_lists, (long long)layouts[i].order.size());
        max_window = std::max(max_window, SpannFileWriter::window_bytes(layouts[i].area));
    }
    const int end_bit = spann_end_bit(num_heads);
    auto a256 = [](long long x) { return (long long)round_up((size_t)x, 256); };
    // a group of E edges (before the cut) and C gathered rows: keys and vector ids twice, the sort's scratch, the rows
    auto group_bytes = [&](long long E, long long C) {
        return 2 * a256(8 * E) + 2 * a256(4 * E) + a256((long long)spann_sort_scratch(E, end_bit, stream)) +
               a256(C * (long long)row_bytes);
    };
    // pass 2's fixed buffers for chunks of C edges: two chunks of keys and vector ids, their flags, the selection's
    // scratch and counters, the list-to-group map, one file's per-list arrays and its window
    auto fixed_bytes = [&](long long C) {
        return 25 * C + (long long)spann_select_scratch((int)C, stream) + 32 + 4ll * num_heads + 28 * max_lists + max_window;
    };
    const long long min_chunk = std::min<long long>(std::max<long long>(stored, 1), 4096);
    const long long largest_group = largest < 0 ? 0 : group_bytes(size[largest], count[largest]);
    const long long minimum = std::max(spann_pass1_bytes(c, 1, stream), fixed_bytes(min_chunk) + largest_group);
    if (budget < minimum)
        return fail(SPTAG_B200_MEMORY_OVERFLOW, "a device budget of %lld bytes: the streamed build needs at least %lld bytes",
                    budget, minimum);
    long long chunk = std::min<long long>(std::max<long long>(stored, 1), 1 << 22);
    while (chunk > min_chunk && fixed_bytes(chunk) + largest_group > budget) chunk = std::max(min_chunk, (chunk + 1) / 2);
    const long long cap = budget - fixed_bytes(chunk);
    struct Group {
        int file, first, end;  // placed lists [first, end) of the file
        long long edges, rows, begin, stop;  // the list area's bytes [begin, stop)
    };
    std::vector<Group> groups;
    std::vector<int> group_of((size_t)num_heads, -1);
    long long max_group = 0;
    for (int i = 0; i < c.file_num; ++i) {
        int first, nl;
        spann_file_lists(c, i, first, nl);
        const SpannFileLayout& L = layouts[i];
        const int n_placed = (int)L.order.size();
        for (int a = 0; a < n_placed;) {
            long long E = 0, C = 0;
            int e = a;
            while (e < n_placed) {
                const int l = first + L.order[e];
                const long long E2 = E + size[l], C2 = C + count[l];
                if (e > a && (E2 > INT_MAX || group_bytes(E2, C2) > cap)) break;
                E = E2;
                C = C2;
                ++e;
            }
            Group g{i, a, e, E, C, L.start[a], e < n_placed ? L.start[e] : L.area};
            // group-local offsets: the sorted edges in list-id order, the gathered rows in placement order
            std::vector<int> ids;
            for (int j = a; j < e; ++j) ids.push_back(first + L.order[j]);
            long long r = 0;
            for (int l : ids) {
                row_off[l] = r;
                r += count[l];
                group_of[l] = (int)groups.size();
            }
            std::sort(ids.begin(), ids.end());
            long long eo = 0;
            for (int l : ids) {
                edge_off[l] = eo;
                eo += size[l];
            }
            max_group = std::max(max_group, group_bytes(E, C));
            groups.push_back(g);
            a = e;
        }
    }

    // pass 2, per group: the group's edges kept from the store, sorted, their rows gathered, its windows written
    if (int rc = st.d_group_of.ensure((size_t)num_heads * 4 + 4)) return rc;
    CUDA_OK(cudaMemcpy(st.d_group_of.ptr, group_of.data(), (size_t)num_heads * 4, cudaMemcpyHostToDevice));
    for (int i = 0; i < 2; ++i) {
        if (int rc = st.d_keys[i].ensure((size_t)chunk * 8)) return rc;
        if (int rc = st.d_tonode[i].ensure((size_t)chunk * 4)) return rc;
    }
    if (int rc = st.d_flags.ensure((size_t)chunk)) return rc;
    sel_bytes = spann_select_scratch((int)chunk, stream);
    if (int rc = st.d_temp.ensure(std::max<size_t>(sel_bytes, 1))) return rc;
    if (int rc = st.d_arena.ensure((size_t)std::max<long long>(max_group, 256))) return rc;
    unsigned char* arena = (unsigned char*)st.d_arena.ptr;
    const unsigned char* d_src_rows = (const unsigned char*)d_src;
    long long gathered = 0;
    for (int i = 0, gi = 0; i < c.file_num; ++i) {
        int first, nl;
        spann_file_lists(c, i, first, nl);
        SpannFileWriter w;
        if (int rc = w.open(bf, layouts[i], spann_file_path(c, i), first, stream)) return rc;
        for (; gi < (int)groups.size() && groups[gi].file == i; ++gi) {
            const Group& g = groups[gi];
            const long long E = g.edges;
            unsigned long long* g_keys[2] = {(unsigned long long*)arena, (unsigned long long*)(arena + a256(8 * E))};
            int* g_ton[2] = {(int*)(arena + 2 * a256(8 * E)), (int*)(arena + 2 * a256(8 * E) + a256(4 * E))};
            unsigned char* g_temp = arena + 2 * a256(8 * E) + 2 * a256(4 * E);
            size_t sort_bytes = spann_sort_scratch(E, end_bit, stream);
            unsigned char* g_rows = g_temp + a256((long long)sort_bytes);
            // the edge pass: the store through two chunk buffers; the copy of chunk j + 1 overlaps chunk j's selection
            long long kept = 0;
            auto copy_chunk = [&](long long c0) -> int {
                const long long n = std::min(chunk, stored - c0);
                const int slot = (int)((c0 / chunk) & 1);
                CUDA_OK(cudaMemcpyAsync(st.d_keys[slot].ptr, h_keys + c0, (size_t)n * 8, cudaMemcpyHostToDevice, st.copy));
                CUDA_OK(cudaMemcpyAsync(st.d_tonode[slot].ptr, h_tonode + c0, (size_t)n * 4, cudaMemcpyHostToDevice, st.copy));
                CUDA_OK(cudaEventRecord(st.copied[slot], st.copy));
                h2d += n * 12;
                return 0;
            };
            if (stored > 0)
                if (int rc = copy_chunk(0)) return rc;
            for (long long c0 = 0; c0 < stored; c0 += chunk) {
                const long long n = std::min(chunk, stored - c0);
                const int slot = (int)((c0 / chunk) & 1);
                // the other chunk buffer was last read by the previous chunk's selection, which the host has waited for
                if (c0 + chunk < stored)
                    if (int rc = copy_chunk(c0 + chunk)) return rc;
                CUDA_OK(cudaStreamWaitEvent(stream, st.copied[slot], 0));
                CUDA_OK(spann_select_edges(st.d_temp.ptr, &sel_bytes, (const unsigned long long*)st.d_keys[slot].ptr,
                                           (int*)st.d_tonode[slot].ptr, (int)n, 0, num_heads, (const int*)st.d_group_of.ptr,
                                           gi, (unsigned char*)st.d_flags.ptr, g_keys[0] + kept, g_ton[0] + kept, d_nsel,
                                           stream));
                g_launches += 3;
                int nsel = 0;
                CUDA_OK(cudaMemcpyAsync(&nsel, d_nsel, 4, cudaMemcpyDeviceToHost, stream));
                CUDA_OK(cudaStreamSynchronize(stream));
                kept += nsel;
            }
            if (kept != E) return fail(SPTAG_B200_FAIL, "group %d: %lld edges kept, %lld expected", gi, kept, E);
            // the edges entered in ascending vector id: the stable sort gives EdgeCompare's order
            CUDA_OK(cudaEventRecord(st.ev[0], stream));
            CUDA_OK(spann_sort_edges(g_temp, &sort_bytes, g_keys[0], g_keys[1], g_ton[0], g_ton[1], (int)E, end_bit, stream));
            g_launches++;
            CUDA_OK(cudaEventRecord(st.ev[1], stream));
            if (int rc = st.elapsed(ms_sort)) return rc;
            // the kept edges' rows, from the caller's buffer
            SpannGatherParams gp;
            memset(&gp, 0, sizeof(gp));
            gp.edge_off = (const long long*)w.d_eoff.ptr;
            gp.row_off = (const long long*)w.d_roff.ptr;
            gp.count = (const int*)w.d_cnt.ptr;
            gp.first_list = g.first;
            gp.num_lists = g.end - g.first;
            gp.tonode = g_ton[1];
            gp.src = d_src_rows;
            gp.row_bytes = (int)row_bytes;
            gp.dst = g_rows;
            CUDA_OK(launch_spann_row_gather(gp, stream));
            g_launches++;
            gathered += g.rows * (long long)row_bytes;
            if (normalize && g.rows > 0) {
                with_elem(h, [&](auto el) {
                    normalize_rows_kernel<typename decltype(el)::type><<<(unsigned)((g.rows + 127) / 128), 128, 0, stream>>>(
                        g_rows, row_bytes, 0, (int)g.rows, dim, base);
                });
                g_launches++;
                CUDA_OK(cudaGetLastError());
            }
            if (int rc = w.write(g.begin, g.stop, g_ton[1], g_rows)) return rc;
        }
        if (layouts[i].area > 0)
            if (int rc = w.finish()) return rc;
    }
    h2d += gathered;
    const double ms_pass2 = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const int64_t out[12] = {searched, (int64_t)rejected, before, after, (int64_t)(ms_search * 1000.0),
                             (int64_t)(ms_rng * 1000.0), (int64_t)(ms_sort * 1000.0),
                             (int64_t)((ms_pass2 - ms_sort) * 1000.0), 1, batches, (int64_t)groups.size(), h2d};
    memcpy(stats, out, sizeof(out));
    return SPTAG_B200_SUCCESS;
}

// sptag_b200_spann_load_ex after its options: the folder's refusals, the head and spann_fill (shared, shared_bytes: a
// group member's, as spann_fill takes them)
int spann_open(const char* folder, int32_t device, int placement, void* shared, size_t shared_bytes,
               sptag_b200_spann_handle* out) {
    *out = nullptr;
    const std::string dir(folder);
    IniSections ini;
    if (!read_ini(dir + "/indexloader.ini", ini)) return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot open %s/indexloader.ini", folder);
    auto get = [&](const char* section, const char* name, const char* def) { return ini_get(ini, section, name, def); };
    if (get("Index", "IndexAlgoType", "SPANN") != "SPANN") return fail(SPTAG_B200_LACK_OF_INPUTS, "%s is not a SPANN index", folder);
    // Refusals: what the device does not hold or decode (SPANN/ParameterDefinitionList.h:34, :79-81)
    const bool quantized = !get("Base", "QuantizerFilePath", "").empty();
    if (quantized && get("Base", "DistCalcMethod", "Cosine") != "L2")  // PQQuantizer::CosineDistance is an error stub
        return fail(SPTAG_B200_LACK_OF_INPUTS, "quantized SPANN indexes are searched with L2 only");
    if (ini_true(get("BuildSSDIndex", "EnableDataCompression", "false")))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "EnableDataCompression (zstd posting lists) is not supported on the device");
    if (ini_true(get("BuildSSDIndex", "EnableDeltaEncoding", "false")))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "EnableDeltaEncoding is not supported on the device");
    const std::string vt = get("Base", "ValueType", "Undefined");
    const int value_type = enum_value(kValueTypes, vt);
    if (value_type < 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "unsupported ValueType %s", vt.c_str());

    sptag_b200_handle head = nullptr;
    const std::string head_dir = dir + "/" + get("Base", "HeadIndexFolder", "HeadIndex");
    if (int rc = sptag_b200_load(head_dir.c_str(), device, 0, &head)) return rc;
    auto* s = new sptag_b200_spann();
    s->head = head;
    s->quantized = quantized;
    if (quantized) {
        // A quantized index's head is a BKT index over UInt8 code rows (SPANNIndex.cpp:850-855).  The reference loads the
        // quantizer the folder's [Quantizer] section names and installs it on the head (VectorIndex.cpp:675-677,
        // SPANNIndex.cpp:39-56); its ValueType is UInt8 (SPANNIndex.cpp:1013, the type of the code rows it was built on)
        // or the quantizer's reconstruct type.  [BuildSSDIndex] EnableADC switches the one quantizer (SPANNIndex.cpp:73-76).
        if (head->q_type == 0 || head->value_type != SPTAG_B200_VT_UINT8 || head->algo != SPTAG_B200_ALGO_BKT) {
            sptag_b200_spann_destroy(s);
            return fail(SPTAG_B200_LACK_OF_INPUTS, "QuantizerFilePath is set but the head index is not a quantized BKT index");
        }
        std::string qname = get("Base", "QuantizerFilePath", "");
        qname = get("Quantizer", "QuantizerFilePath", qname.substr(qname.find_last_of("/\\") + 1).c_str());
        std::vector<char> qb;
        if (!read_file(dir + "/" + qname, qb)) {
            sptag_b200_spann_destroy(s);
            return fail(SPTAG_B200_FAILED_OPEN_FILE, "cannot read quantizer file %s", qname.c_str());
        }
        int rc = sptag_b200_set_quantizer(head, qb.data(), (int64_t)qb.size());
        if (!rc && value_type != SPTAG_B200_VT_UINT8 && value_type != head->q_rtype)
            rc = fail(SPTAG_B200_LACK_OF_INPUTS, "ValueType %s is neither UInt8 nor the quantizer's reconstruct type", vt.c_str());
        if (!rc && ini_true(get("BuildSSDIndex", "EnableADC", "false"))) rc = sptag_b200_set_param(head, "EnableADC", "1");
        if (rc) {
            sptag_b200_spann_destroy(s);
            return rc;
        }
    } else if (head->value_type != value_type || head->q_type != 0) {
        sptag_b200_spann_destroy(s);
        return fail(SPTAG_B200_LACK_OF_INPUTS, "head index value type %d does not match ValueType %s", head->value_type, vt.c_str());
    }
    if (int rc = spann_fill(s, dir, ini, placement, shared, shared_bytes)) {
        sptag_b200_spann_destroy(s);
        return rc;
    }
    *out = s;
    return SPTAG_B200_SUCCESS;
}

// cache_warm's ranking (sptag_b200_spann_cache_warm): for each sample query the head search and posting choice of a
// search with K <= SearchInternalResultNum, on staging set 0 of s, the lists counted on the device; order receives the
// lists some query chose, by count, descending, then list id.  Caller holds both of s's staging sets and checked that
// SearchInternalResultNum <= 2048.
int spann_warm_order(sptag_b200_spann* s, const SpannSnapshot& sp, const void* queries, int32_t num_queries,
                     std::vector<int>& order) {
    sptag_b200_handle h = s->head;
    const size_t nl = (size_t)s->num_lists, nq = (size_t)num_queries;
    // a search's head search and posting choice at K <= SearchInternalResultNum, on staging set 0's buffers
    const int w = std::max(sp.internal, 1);
    std::vector<int> counts(nl, 0);
    DeviceGuard guard(h->device);
    auto& st = s->staging.sets[0];
    cudaStream_t stream = st.stream;
    if (nq > 0) {
        DeviceBuffer d_counts;
        if (int rc = st.d_q.ensure(nq * query_bytes(h))) return rc;
        if (int rc = st.d_hids.ensure(nq * w * 4)) return rc;
        if (int rc = st.d_hdists.ensure(nq * w * 4)) return rc;
        if (int rc = st.d_chosen.ensure(nq * w * 4)) return rc;
        if (int rc = st.d_nchosen.ensure(nq * 4)) return rc;
        if (int rc = d_counts.ensure(nl * 4)) return rc;
        CUDA_OK(cudaMemcpyAsync(st.d_q.ptr, queries, nq * query_bytes(h), cudaMemcpyHostToDevice, stream));
        {
            std::lock_guard<std::mutex> lock(h->mu);
            if (int rc = search_device_impl(h, st.d_q.ptr, num_queries, w, (int*)st.d_hids.ptr, (float*)st.d_hdists.ptr,
                                            nullptr, stream)) {
                cudaStreamSynchronize(stream);
                return rc;
            }
        }
        SpannScanParams p;
        memset(&p, 0, sizeof(p));
        p.head_ids = (const int*)st.d_hids.ptr;
        p.head_dists = (const float*)st.d_hdists.ptr;
        p.nq = num_queries;
        p.w = w;
        p.k = w;
        p.translate = (const int*)s->d_translate.ptr;
        p.lists = posting_lists(s, sp.page_limit);
        p.internal = sp.internal;
        p.max_dist_ratio = sp.max_dist_ratio;
        CUDA_OK(cudaMemsetAsync(d_counts.ptr, 0, nl * 4, stream));
        CUDA_OK(launch_spann_choose(p, (int*)st.d_chosen.ptr, (int*)st.d_nchosen.ptr, w, stream));
        CUDA_OK(launch_spann_count((const int*)st.d_chosen.ptr, (const int*)st.d_nchosen.ptr, w, num_queries,
                                   (int*)d_counts.ptr, stream));
        g_launches += 2;
        CUDA_OK(cudaMemcpyAsync(counts.data(), d_counts.ptr, nl * 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
    }
    order.clear();
    for (size_t l = 0; l < nl; ++l)
        if (counts[l] > 0) order.push_back((int)l);
    std::sort(order.begin(), order.end(), [&](int a, int b) { return counts[a] != counts[b] ? counts[a] > counts[b] : a < b; });
    return 0;
}

// cache_warm's budget: budget_bytes, or for -1 cudaMemGetInfo's free bytes on s's device less kPostingReserve
int spann_warm_budget(const sptag_b200_spann* s, long long budget_bytes, long long& budget) {
    budget = budget_bytes;
    if (budget != -1) return 0;
    DeviceGuard guard(s->head->device);
    size_t free_bytes = 0, total_bytes = 0;
    CUDA_OK(cudaMemGetInfo(&free_bytes, &total_bytes));
    budget = std::max(0ll, (long long)free_bytes - kPostingReserve);
    return 0;
}

// Installs lists[i] on member i of g (spann_cache_install, each with its own stage parameters), then rebuilds every
// peer table.  Returns the first failure; the members installed before it keep their caches.  Caller holds GroupSets.
int spann_group_install(sptag_b200_spann_group* g, const std::vector<std::vector<int>>& lists) {
    int rc = 0;
    for (size_t i = 0; i < g->members.size(); ++i) {
        sptag_b200_spann* m = g->members[i];
        SpannSnapshot sp;
        spann_snapshot(m, sp);  // fills sp whether or not the page limit would refuse a search
        const int r = spann_cache_install(m, lists[i], stage_elems(m, sp));
        if (r && !rc) rc = r;
    }
    const int r = spann_group_peer_tables(g);
    return rc ? rc : r;
}

}  // namespace

extern "C" {

void sptag_b200_spann_destroy(sptag_b200_spann_handle s) {
    if (!s || s->group) return;  // a group member: the group owns it
    {
        DeviceGuard guard(s->head ? s->head->device : 0);
        cudaDeviceSynchronize();
        sptag_b200_handle head = s->head;
        if (s->h_postings) cudaFreeHost(s->h_postings);
        delete s;  // frees the device buffers, with the index's device current
        sptag_b200_destroy(head);
    }
}

int sptag_b200_spann_load(const char* folder, int32_t device, sptag_b200_spann_handle* out) {
    sptag_b200_spann_load_options o;
    o.struct_size = (int32_t)sizeof(o);
    o.posting_placement = SPTAG_B200_POSTINGS_DEVICE;
    return sptag_b200_spann_load_ex(folder, device, &o, out);
}

int sptag_b200_spann_load_ex(const char* folder, int32_t device, const sptag_b200_spann_load_options* options,
                             sptag_b200_spann_handle* out) {
    if (!folder || !out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    int placement = SPTAG_B200_POSTINGS_AUTO;
    if (options) {
        if (options->struct_size != (int32_t)sizeof(sptag_b200_spann_load_options))
            return fail(SPTAG_B200_FAIL, "options size mismatch: %d vs %zu", options->struct_size,
                        sizeof(sptag_b200_spann_load_options));
        placement = options->posting_placement;
        if (placement != SPTAG_B200_POSTINGS_AUTO && placement != SPTAG_B200_POSTINGS_DEVICE &&
            placement != SPTAG_B200_POSTINGS_HOST && placement != SPTAG_B200_POSTINGS_FILE)
            return fail(SPTAG_B200_LACK_OF_INPUTS, "unknown posting placement %d", placement);
    }
    return spann_open(folder, device, placement, nullptr, 0, out);
}

int sptag_b200_spann_build(const char* folder, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                           int32_t device, int64_t* out_stats) {
    SpannBuildState st;
    SpannBuildConfig c;
    if (int rc = spann_build_prepare(folder, vectors, num, dim, normalized, device, st, c)) return rc;
    const size_t edges = (size_t)num * c.replicas;
    if (edges > (size_t)INT_MAX) return fail(SPTAG_B200_MEMORY_OVERFLOW, "%zu edges: more than 2^31 - 1", edges);
    int64_t stats[8];
    if (int rc = spann_build_resident(c, st, vectors, stats)) return rc;
    if (out_stats) memcpy(out_stats, stats, sizeof(stats));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_build_ex(const char* folder, const void* vectors, int32_t num, int32_t dim, int32_t normalized,
                              int32_t device, const sptag_b200_spann_build_options* options, int64_t* out_stats) {
    long long budget = -1;
    if (options) {
        if (options->struct_size != (int32_t)sizeof(sptag_b200_spann_build_options))
            return fail(SPTAG_B200_FAIL, "options size mismatch: %d vs %zu", options->struct_size,
                        sizeof(sptag_b200_spann_build_options));
        budget = options->device_budget_bytes;
        if (budget < -1) return fail(SPTAG_B200_LACK_OF_INPUTS, "device_budget_bytes %lld is below -1", budget);
    }
    SpannBuildState st;
    SpannBuildConfig c;
    if (int rc = spann_build_prepare(folder, vectors, num, dim, normalized, device, st, c)) return rc;
    DeviceGuard guard(st.head->device);
    if (budget == -1) {  // AUTO's reserve (sptag_b200_spann_load_ex)
        size_t free_b = 0, total_b = 0;
        CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
        budget = std::max<long long>(0, (long long)free_b - (1ll << 30));
    }
    const long long edges = (long long)num * c.replicas;
    int64_t stats[12] = {0};
    if (edges <= INT_MAX && spann_resident_bytes(c, nullptr) <= budget) {
        if (int rc = spann_build_resident(c, st, vectors, stats)) return rc;
        stats[8] = 0;
        stats[9] = (num + (1 << 16) - 1) >> 16;
        stats[10] = 1;
        stats[11] = (long long)num * (long long)c.row_bytes;
    } else if (int rc = spann_build_streamed(c, st, vectors, budget, stats)) {
        return rc;
    }
    if (out_stats) memcpy(out_stats, stats, sizeof(stats));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_search(sptag_b200_spann_handle s, const void* queries, int32_t num_queries, int32_t k, int32_t* out_ids,
                            float* out_dists, int32_t* out_stats) {
    if (!s) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && (!queries || !out_ids || !out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (k < 1 || k > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside the supported range [1, 2048]", k);
    if (num_queries == 0) return SPTAG_B200_SUCCESS;
    sptag_b200_handle h = s->head;
    SpannSnapshot sp;
    if (int rc = spann_snapshot(s, sp)) return rc;
    SpannScanParams p;
    memset(&p, 0, sizeof(p));
    p.internal = sp.internal;
    p.max_dist_ratio = sp.max_dist_ratio;
    // SPANNIndex.cpp:197-201: the head search runs at K when K >= SearchInternalResultNum, else at SearchInternalResultNum
    const int w = k >= p.internal ? k : p.internal;
    if (w > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "SearchInternalResultNum %d exceeds 2048", p.internal);
    // the dedup table holds every element a query may read at half load
    const long long reads = (long long)std::min(std::max(p.internal, 0), w) * sp.longest;
    long long entries = 64;
    while (entries < 2 * reads) entries <<= 1;
    if (entries > (1ll << 30)) return fail(SPTAG_B200_MEMORY_OVERFLOW, "dedup table of %lld entries", entries);
    std::unique_lock<std::mutex> slock;
    decltype(s->staging.acquire(slock)) st = nullptr;
    if (!s->host_postings)
        st = s->staging.acquire(slock);
    else if (int rc = spann_acquire_fitted(s, sp, slock, st))
        return rc;
    DeviceGuard guard(h->device);
    cudaStream_t stream = st->stream;
    const size_t nq = (size_t)num_queries;
    const size_t qrow = query_bytes(h);  // quantized: raw vectors of the quantizer's reconstruct type
    const MetricElem me = metric_elem(h);
    int per_sm = s->quantized ? spann_pq_scan_blocks_per_sm(w, h->q_m) : spann_scan_blocks_per_sm(me.cosine, me.elem, w);
    if (per_sm < 1) return fail(SPTAG_B200_MEMORY_OVERFLOW, "the posting scan kernel does not fit on an SM at W = %d", w);
    // resident blocks, but no more dedup-table bytes than kTableBytes unless one block per SM needs more
    const long long kTableBytes = 256ll << 20;
    const long long blocks = std::max<long long>(h->num_sms, kTableBytes / (entries * 4));
    const int grid = (int)std::min<long long>(std::min<long long>((long long)num_queries, (long long)h->num_sms * per_sm), blocks);
    if (int rc = st->d_q.ensure(nq * qrow)) return rc;
    if (int rc = st->d_qpad.ensure(nq * h->row_stride)) return rc;
    if (int rc = st->d_hids.ensure(nq * w * 4)) return rc;
    if (int rc = st->d_hdists.ensure(nq * w * 4)) return rc;
    if (int rc = st->d_ids.ensure(nq * k * 4)) return rc;
    if (int rc = st->d_dists.ensure(nq * k * 4)) return rc;
    if (out_stats)
        if (int rc = st->d_stats.ensure(nq * 3 * 4)) return rc;
    if (int rc = st->d_tables.ensure((size_t)grid * entries * 4)) return rc;
    CUDA_OK(cudaMemcpyAsync(st->d_q.ptr, queries, nq * qrow, cudaMemcpyHostToDevice, stream));  // as the head search reads them
    if (!s->quantized)
        if (int rc = upload_query_rows(h, st->d_qpad.ptr, st->d_q.ptr, nq, stream)) return rc;
    SpannPqScanParams pq;
    memset(&pq, 0, sizeof(pq));
    {
        std::lock_guard<std::mutex> lock(h->mu);
        if (int rc = search_device_impl(h, st->d_q.ptr, num_queries, w, (int*)st->d_hids.ptr, (float*)st->d_hdists.ptr,
                                        nullptr, stream)) {
            cudaStreamSynchronize(stream);
            return rc;
        }
        if (s->quantized) {
            // QueryResultSet::GetQuantizedTarget, as the head search quantized it (SDC: M codes; ADC: the rotated vector
            // the scan builds the query's table from), under the same lock, so that both see one EnableADC
            pq.m = h->q_m;
            pq.ks = h->q_ks;
            pq.dsub = h->q_dsub;
            pq.adc = h->q_adc ? 1 : 0;
            int rc = 0;
            if (pq.adc) {
                const size_t dimq = (size_t)h->q_m * h->q_dsub;
                if (!(rc = st->d_codes.ensure(nq * dimq * 4)) && !(rc = st->d_adc.ensure((size_t)grid * h->q_m * h->q_ks * 4)))
                    rc = quantize_device(h, st->d_q.ptr, num_queries, nullptr, stream, (float*)st->d_codes.ptr);
                pq.qrot = (const float*)st->d_codes.ptr;
                pq.codebooks = (const float*)h->d_codebooks.ptr;
                pq.adc_tables = (float*)st->d_adc.ptr;
            } else {
                if (!(rc = st->d_codes.ensure(nq * h->q_m)))
                    rc = quantize_device(h, st->d_q.ptr, num_queries, (unsigned char*)st->d_codes.ptr, stream);
                pq.qcodes = (const unsigned char*)st->d_codes.ptr;
                pq.sdc = (const float*)h->d_sdc.ptr;
            }
            if (rc) {
                cudaStreamSynchronize(stream);
                return rc;
            }
        }
    }
    p.head_ids = (const int*)st->d_hids.ptr;
    p.head_dists = (const float*)st->d_hdists.ptr;
    p.nq = num_queries;
    p.w = w;
    p.k = k;
    p.queries = (const unsigned char*)st->d_qpad.ptr;
    p.dim = h->dim;
    p.simd_width = h->simd_width;
    p.translate = (const int*)s->d_translate.ptr;
    p.lists = posting_lists(s, sp.page_limit);
    p.tables = (int*)st->d_tables.ptr;
    p.table_entries = (int)entries;
    p.out_ids = (int*)st->d_ids.ptr;
    p.out_dists = (float*)st->d_dists.ptr;
    p.out_stats = out_stats ? (int*)st->d_stats.ptr : nullptr;
    pq.s = p;
    const void* kern = nullptr;
    if (s->host_postings) {
        // the queries' chosen lists, once; then the rounds, each a scan over its queries on the staged lists
        const int stride = std::max(p.internal, 1);
        long bytes = 0, rounds = 0, peer_bytes = 0, read_bytes = 0;
        int rc = 0;
        if (!(rc = st->d_chosen.ensure(nq * stride * 4)) && !(rc = st->d_nchosen.ensure(nq * 4))) {
            const cudaError_t e = launch_spann_choose(p, (int*)st->d_chosen.ptr, (int*)st->d_nchosen.ptr, stride, stream);
            g_launches++;
            if (e != cudaSuccess) rc = fail(SPTAG_B200_FAIL, "posting choice launch failed: %s", cudaGetErrorString(e));
        }
        auto choose = [&](int b, int, const int*& chosen, const int*& nchosen) {
            chosen = (const int*)st->d_chosen.ptr + (size_t)b * stride;
            nchosen = (const int*)st->d_nchosen.ptr + b;
            return 0;
        };
        auto run = [&](int b, int e, const PostingLists& view) {
            SpannPqScanParams r = pq;
            r.s.head_ids += (size_t)b * w;
            r.s.head_dists += (size_t)b * w;
            r.s.nq = e - b;
            r.s.queries += (size_t)b * h->row_stride;
            r.s.lists = view;
            r.s.out_ids += (size_t)b * k;
            r.s.out_dists += (size_t)b * k;
            if (r.s.out_stats) r.s.out_stats += (size_t)b * 3;
            if (r.qcodes) r.qcodes += (size_t)b * r.m;
            if (r.qrot) r.qrot += (size_t)b * r.m * r.dsub;
            const int g = std::min(grid, e - b);
            const cudaError_t err = s->quantized ? launch_spann_pq_scan(r, g, stream, &kern)
                                                 : launch_spann_scan(r.s, me.cosine, me.elem, g, stream, &kern);
            g_launches++;
            if (err != cudaSuccess) return fail(SPTAG_B200_FAIL, "posting scan launch failed: %s", cudaGetErrorString(err));
            return 0;
        };
        if (!rc)
            rc = gather_rounds(s, *st, sp, num_queries, stride, stream, choose, run, bytes, rounds, peer_bytes, read_bytes);
        if (rc) {
            cudaStreamSynchronize(stream);
            return rc;
        }
        std::lock_guard<std::mutex> lock(s->mu);
        s->last_gather_bytes = bytes;
        s->last_gather_rounds = rounds;
        s->last_peer_gather_bytes = peer_bytes;
        s->last_read_bytes = read_bytes;
    } else {
        cudaError_t e = s->quantized ? launch_spann_pq_scan(pq, grid, stream, &kern)
                                     : launch_spann_scan(p, me.cosine, me.elem, grid, stream, &kern);
        g_launches++;
        if (e != cudaSuccess) {
            cudaStreamSynchronize(stream);
            return fail(SPTAG_B200_FAIL, "posting scan launch failed: %s", cudaGetErrorString(e));
        }
    }
    if (kern) {
        std::lock_guard<std::mutex> lock(s->mu);
        s->last_posting_kernel = kern;
    }
    CUDA_OK(cudaMemcpyAsync(out_ids, st->d_ids.ptr, nq * k * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_dists, st->d_dists.ptr, nq * k * 4, cudaMemcpyDeviceToHost, stream));
    if (out_stats) CUDA_OK(cudaMemcpyAsync(out_stats, st->d_stats.ptr, nq * 3 * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_set_param(sptag_b200_spann_handle s, const char* name, const char* value) {
    if (!s || !name || !value) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    const Param<Spann>* p = find_param(kSpannParams, name);
    if (p && (p->flags & kHead)) return sptag_b200_set_param(s->head, name, value);
    std::lock_guard<std::mutex> lock(s->mu);
    return set_param(s, p, name, value);
}

int sptag_b200_spann_get_param(sptag_b200_spann_handle s, const char* name, char* value_out, int32_t capacity) {
    if (!s || !name || !value_out || capacity <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    const Param<Spann>* p = find_param(kSpannParams, name);
    if (p && (p->flags & kHead)) return sptag_b200_get_param(s->head, name, value_out, capacity);
    std::lock_guard<std::mutex> lock(s->mu);
    return get_param(s, p, name, value_out, (size_t)capacity);
}

int sptag_b200_spann_cache_warm(sptag_b200_spann_handle s, const void* queries, int32_t num_queries, int64_t budget_bytes,
                                int32_t* out_lists, int32_t capacity, int32_t* out_num_lists) {
    if (!s) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!s->host_postings) return fail(SPTAG_B200_LACK_OF_INPUTS, "the HBM cache of posting lists needs the host placement");
    if (s->group)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "a group member's cache is set by sptag_b200_spann_group_cache_warm / "
                                               "_cache_lists: its peers read its pool");
    if (num_queries < 0 || (num_queries > 0 && !queries) || !out_num_lists || capacity < 0 || (capacity > 0 && !out_lists))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (budget_bytes < -1) return fail(SPTAG_B200_LACK_OF_INPUTS, "budget %lld below -1", (long long)budget_bytes);
    *out_num_lists = 0;
    SpannSnapshot sp;
    if (int rc = spann_snapshot(s, sp)) return rc;
    if (sp.internal > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "SearchInternalResultNum %d exceeds 2048", sp.internal);
    BothSets both(s);
    DeviceGuard guard(s->head->device);
    std::vector<int> order;
    if (int rc = spann_warm_order(s, sp, queries, num_queries, order)) return rc;
    spann_cache_release(s);
    long long budget = 0;
    if (int rc = spann_warm_budget(s, budget_bytes, budget)) return rc;
    // in rank order, each list that fits what is left of the budget, whole
    const long long elem_bytes = (long long)s->head->row_stride + 4;
    std::vector<int> taken;
    for (int l : order) {
        const long long bytes = (long long)s->cnt[l] * elem_bytes;
        if (bytes > budget) continue;
        taken.push_back(l);
        budget -= bytes;
    }
    if (int rc = spann_cache_install(s, taken, stage_elems(s, sp))) return rc;
    *out_num_lists = (int32_t)taken.size();
    std::copy_n(taken.begin(), std::min<size_t>(taken.size(), (size_t)capacity), out_lists);
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_cache_lists(sptag_b200_spann_handle s, const int32_t* lists, int32_t num_lists) {
    if (!s) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!s->host_postings) return fail(SPTAG_B200_LACK_OF_INPUTS, "the HBM cache of posting lists needs the host placement");
    if (s->group)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "a group member's cache is set by sptag_b200_spann_group_cache_lists: its "
                                               "peers read its pool");
    if (num_lists < 0 || (num_lists > 0 && !lists)) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    std::vector<char> seen((size_t)s->num_lists, 0);
    for (int32_t i = 0; i < num_lists; ++i) {
        const int l = lists[i];
        if (l < 0 || l >= s->num_lists) return fail(SPTAG_B200_LACK_OF_INPUTS, "list %d outside [0, %d)", l, s->num_lists);
        if (seen[l]) return fail(SPTAG_B200_LACK_OF_INPUTS, "list %d given twice", l);
        seen[l] = 1;
    }
    SpannSnapshot sp;
    spann_snapshot(s, sp);  // fills sp whether or not the page limit would refuse a search
    BothSets both(s);
    return spann_cache_install(s, std::vector<int>(lists, lists + num_lists), stage_elems(s, sp));
}

void sptag_b200_spann_group_destroy(sptag_b200_spann_group_handle g) {
    if (!g) return;
    for (sptag_b200_spann* m : g->members) {
        m->group = nullptr;
        sptag_b200_spann_destroy(m);
    }
    if (g->h_postings) cudaFreeHost(g->h_postings);
    delete g;
}

int sptag_b200_spann_group_load(const char* folder, const int32_t* devices, int32_t num_members,
                                sptag_b200_spann_group_handle* out) {
    if (!folder || !out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    *out = nullptr;
    if (num_members < 1 || num_members > kMaxSpannPeers)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "%d members outside [1, %d]", num_members, kMaxSpannPeers);
    if (!devices) return fail(SPTAG_B200_LACK_OF_INPUTS, "null device list");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) {
        cudaGetLastError();
        count = 0;
    }
    for (int i = 0; i < num_members; ++i)
        if (devices[i] < 0 || devices[i] >= count)
            return fail(SPTAG_B200_FAIL, "member %d: device %d, %d devices visible", i, devices[i], count);
    auto* g = new sptag_b200_spann_group();
    for (int i = 0; i < num_members; ++i) {
        // the first member reads the lists into a portable pinned allocation, which the group takes; the others map it
        sptag_b200_spann_handle m = nullptr;
        const size_t bytes = i ? g->members[0]->h_posting_bytes : 0;
        if (int rc = spann_open(folder, devices[i], kPostingsPortable, g->h_postings, bytes, &m)) {
            sptag_b200_spann_group_destroy(g);
            return rc;
        }
        if (i == 0) g->h_postings = std::exchange(m->h_postings, nullptr);
        m->group = g;
        g->members.push_back(m);
    }
    // peer access both ways between the members' devices where the hardware allows it, as sptag_b200_group_create
    // enables it; a member reads the pools of the members it reaches
    const size_t n = g->members.size();
    g->reach.assign(n, std::vector<char>(n, 0));
    for (size_t i = 0; i < n; ++i) {
        for (size_t o = 0; o < n; ++o) {
            const int a = devices[i], b = devices[o];
            int can = a == b;
            if (!can && cudaDeviceCanAccessPeer(&can, a, b) == cudaSuccess && can) {
                DeviceGuard guard(a);
                const cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
                can = e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled;
            }
            cudaGetLastError();
            g->reach[i][o] = (char)(can ? 1 : 0);
        }
    }
    *out = g;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_group_member(sptag_b200_spann_group_handle g, int32_t i, sptag_b200_spann_handle* out) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!out) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    if (i < 0 || i >= (int32_t)g->members.size())
        return fail(SPTAG_B200_LACK_OF_INPUTS, "member %d outside [0, %zu)", i, g->members.size());
    *out = g->members[(size_t)i];
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_group_set_param(sptag_b200_spann_group_handle g, const char* name, const char* value) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!name || !value) return fail(SPTAG_B200_LACK_OF_INPUTS, "null argument");
    std::lock_guard<std::mutex> lock(g->params);
    for (sptag_b200_spann* m : g->members)
        if (int rc = sptag_b200_spann_set_param(m, name, value)) return rc;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_group_search(sptag_b200_spann_group_handle g, const void* queries, int32_t num_queries, int32_t k,
                                  int32_t* out_ids, float* out_dists, int64_t* out_stats) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && (!queries || !out_ids || !out_dists)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (k < 1 || k > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside the supported range [1, 2048]", k);
    // the members search with the same parameters, so that a query's result does not depend on which one runs it
    for (const char* name : {"SearchInternalResultNum", "MaxDistRatio", "SearchPostingPageLimit", "MaxCheck"}) {
        char first[64], other[64];
        if (int rc = sptag_b200_spann_get_param(g->members[0], name, first, sizeof(first))) return rc;
        for (size_t i = 1; i < g->members.size(); ++i) {
            if (int rc = sptag_b200_spann_get_param(g->members[i], name, other, sizeof(other))) return rc;
            if (strcmp(first, other) != 0)
                return fail(SPTAG_B200_LACK_OF_INPUTS, "members 0 and %zu differ in %s: %s, %s", i, name, first, other);
        }
    }
    if (num_queries == 0) return SPTAG_B200_SUCCESS;
    // member i: queries [i * per, (i + 1) * per), on a thread of its own (a search blocks once per gather round)
    const size_t n = g->members.size(), nq = (size_t)num_queries, per = (nq + n - 1) / n;
    const size_t qrow = query_bytes(g->members[0]->head);
    std::vector<int> rcs(n, 0);
    std::vector<std::string> errors(n);
    std::vector<std::thread> threads;
    for (size_t i = 0; i < n && i * per < nq; ++i) {
        threads.emplace_back([&, i] {
            const size_t b = i * per, e = std::min(nq, b + per);
            std::vector<int32_t> stats(out_stats ? (e - b) * 3 : 0);
            rcs[i] = sptag_b200_spann_search(g->members[i], (const unsigned char*)queries + b * qrow, (int32_t)(e - b), k,
                                             out_ids + b * k, out_dists + b * k, out_stats ? stats.data() : nullptr);
            if (rcs[i]) {
                errors[i] = g_last_error;
                return;
            }
            for (size_t j = 0; j < stats.size(); ++j) out_stats[b * 3 + j] = stats[j];
        });
    }
    for (std::thread& t : threads) t.join();
    for (size_t i = 0; i < n; ++i)
        if (rcs[i]) return fail(rcs[i], "member %zu: %s", i, errors[i].c_str());
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_group_cache_warm(sptag_b200_spann_group_handle g, const void* queries, int32_t num_queries,
                                      int64_t budget_bytes_per_member, int32_t* out_lists, int32_t* out_owners,
                                      int32_t capacity, int32_t* out_n) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (num_queries < 0 || (num_queries > 0 && !queries) || !out_n || capacity < 0 ||
        (capacity > 0 && (!out_lists || !out_owners)))
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (budget_bytes_per_member < -1)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "budget %lld below -1", (long long)budget_bytes_per_member);
    *out_n = 0;
    sptag_b200_spann* m0 = g->members[0];
    SpannSnapshot sp;
    if (int rc = spann_snapshot(m0, sp)) return rc;
    if (sp.internal > 2048) return fail(SPTAG_B200_LACK_OF_INPUTS, "SearchInternalResultNum %d exceeds 2048", sp.internal);
    GroupSets all(g);
    std::vector<int> order;
    if (int rc = spann_warm_order(m0, sp, queries, num_queries, order)) return rc;
    const size_t n = g->members.size();
    std::vector<long long> left(n, 0);
    for (size_t i = 0; i < n; ++i) {
        {
            DeviceGuard guard(g->members[i]->head->device);
            spann_cache_release(g->members[i]);
        }
        if (int rc = spann_warm_budget(g->members[i], budget_bytes_per_member, left[i])) {
            spann_group_peer_tables(g);
            return rc;
        }
    }
    // in rank order, each list to the member with the most budget left (the lower index of equals), if it fits there
    const long long elem_bytes = (long long)m0->head->row_stride + 4;
    std::vector<std::vector<int>> mine(n);
    std::vector<int> lists, owners;
    for (int l : order) {
        size_t o = 0;
        for (size_t i = 1; i < n; ++i)
            if (left[i] > left[o]) o = i;
        const long long bytes = (long long)m0->cnt[l] * elem_bytes;
        if (bytes > left[o]) continue;
        left[o] -= bytes;
        mine[o].push_back(l);
        lists.push_back(l);
        owners.push_back((int)o);
    }
    if (int rc = spann_group_install(g, mine)) return rc;
    *out_n = (int32_t)lists.size();
    const size_t c = std::min<size_t>(lists.size(), (size_t)capacity);
    std::copy_n(lists.begin(), c, out_lists);
    std::copy_n(owners.begin(), c, out_owners);
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_group_cache_lists(sptag_b200_spann_group_handle g, const int32_t* lists, const int32_t* owners,
                                       int32_t n) {
    if (!g) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (n < 0 || (n > 0 && (!lists || !owners))) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    const int nl = g->members[0]->num_lists, members = (int)g->members.size();
    std::vector<char> seen((size_t)nl, 0);
    std::vector<std::vector<int>> mine((size_t)members);
    for (int32_t i = 0; i < n; ++i) {
        const int l = lists[i], o = owners[i];
        if (l < 0 || l >= nl) return fail(SPTAG_B200_LACK_OF_INPUTS, "list %d outside [0, %d)", l, nl);
        if (o < 0 || o >= members) return fail(SPTAG_B200_LACK_OF_INPUTS, "owner %d outside [0, %d)", o, members);
        if (seen[l]) return fail(SPTAG_B200_LACK_OF_INPUTS, "list %d given twice", l);
        seen[l] = 1;
        mine[(size_t)o].push_back(l);
    }
    GroupSets all(g);
    return spann_group_install(g, mine);
}

}  // extern "C"

// SPANN::Index<T>::GetIterator (SPANNIndex.cpp:299-314) for every query of a batch: the SPANNResultIterator's head
// ResultIterator (an iterator on the head handle), its ExtraWorkSpace (SpannIterState, the chosen lists and the deduper)
// and its QueryResult, kept in HBM between launches.
struct sptag_b200_spann_iterator {
    sptag_b200_spann* s = nullptr;
    sptag_b200_iterator* head = nullptr;
    int nq = 0, hb = 0;  // hb: IterativeSearchHeadBatch, sampled at open
    int cap = 0;         // the QueryResult's size: the first Next's batch
    DeviceBuffer d_queries, d_state, d_posts, d_heap_d, d_heap_v, d_refill[2], d_susp[2], d_ids, d_dists, d_counts,
        d_relaxed;
    // The dedup sets (OptHashPosVector, WorkSpace.h:43-165): exact sets that double when they fill; d_dedup holds their
    // IterStates
    QueryTables dedup;
    DeviceBuffer d_dedup;
};

namespace {

void spann_iterator_free(sptag_b200_spann_iterator* it) {
    sptag_b200_iterator_close(it->head);
    DeviceGuard guard(it->s->head->device);
    delete it;  // frees the device buffers, with the index's device current
}

}  // namespace

extern "C" {

int sptag_b200_spann_iterator_open(sptag_b200_spann_handle s, const void* queries, int32_t num_queries,
                                   sptag_b200_spann_iter* out) {
    if (!s) return fail(SPTAG_B200_EMPTY_INDEX, "null handle");
    if (!out || !queries || num_queries <= 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    *out = nullptr;
    // the head iterators are not built for quantized indexes (sptag_b200_iterator_open)
    if (s->quantized) return fail(SPTAG_B200_LACK_OF_INPUTS, "SPANN iterators on quantized indexes are not supported");
    int hb = 0, entries = 0, longest = 0;
    {
        std::lock_guard<std::mutex> lock(s->mu);
        hb = s->head_batch;
        entries = s->dedup_entries;
        longest = s->longest;
    }
    if (hb < 1 || hb > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "IterativeSearchHeadBatch %d outside [1, 1024]", hb);
    if (entries == 0) {  // the lists of one head batch at half load, at most 2^14 entries to start with
        entries = 64;
        while (entries < (1 << 14) && entries < 2ll * hb * longest) entries <<= 1;
    }
    int bits = 6;
    while ((1 << bits) < entries) ++bits;
    sptag_b200_index* h = s->head;
    sptag_b200_iter head = nullptr;
    // the head ResultIterator searches with p_searchDeleted = false (SPANNResultIterator.h:25)
    if (int rc = sptag_b200_iterator_open_ex(h, queries, num_queries, 0, &head)) return rc;
    auto* it = new sptag_b200_spann_iterator();
    it->s = s;
    it->head = head;
    it->nq = num_queries;
    it->hb = hb;
    DeviceGuard guard(h->device);
    const size_t nq = (size_t)num_queries;
    int rc = 0;
    if ((rc = it->d_queries.ensure(nq * h->row_stride)) || (rc = it->d_state.ensure(nq * sizeof(SpannIterState))) ||
        (rc = it->d_posts.ensure(nq * hb * 4)) || (rc = it->d_refill[0].ensure((kIterListHeader + nq) * 4)) ||
        (rc = it->d_refill[1].ensure((kIterListHeader + nq) * 4)) || (rc = it->d_susp[0].ensure((kIterListHeader + nq) * 4)) ||
        (rc = it->d_susp[1].ensure((kIterListHeader + nq) * 4)) || (rc = it->d_counts.ensure(nq * 4)) ||
        (rc = it->d_relaxed.ensure(nq)) || (rc = it->d_dedup.ensure(nq * sizeof(IterState))) ||
        (rc = upload_query_rows(h, it->d_queries.ptr, queries, nq, nullptr)) ||
        (rc = it->dedup.open(nq, bits, QueryTables::kNoBitmap, (IterState*)it->d_dedup.ptr))) {
        spann_iterator_free(it);
        return rc;
    }
    // GetIterator: relaxedMono = false, loadedPostingNum = 0, an empty deduper and posting list; the first head batch
    // is loaded by the first Next
    SpannIterState st0 = {};
    st0.load = 1;
    st0.slots = -1;
    const std::vector<SpannIterState> st(nq, st0);
    const cudaError_t e = cudaMemcpy(it->d_state.ptr, st.data(), nq * sizeof(SpannIterState), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        spann_iterator_free(it);
        return fail(SPTAG_B200_FAIL, "SPANN iterator set-up failed: %s", cudaGetErrorString(e));
    }
    *out = it;
    return SPTAG_B200_SUCCESS;
}

int sptag_b200_spann_iterator_next(sptag_b200_spann_iter it, int32_t batch, int32_t* out_ids, float* out_dists,
                                   int32_t* out_counts, uint8_t* out_relaxed_mono) {
    if (!it || !it->s) return fail(SPTAG_B200_EMPTY_INDEX, "null iterator");
    if (!out_ids || !out_dists || !out_counts || !out_relaxed_mono) return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (batch < 1 || batch > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "batch = %d outside [1, 1024]", batch);
    sptag_b200_spann* s = it->s;
    sptag_b200_index* h = s->head;
    SpannSnapshot sp;
    if (int rc = spann_snapshot(s, sp)) return rc;
    SpannIterParams p;
    memset(&p, 0, sizeof(p));
    p.internal = sp.internal;
    // The reference has SearchInternalResultNum page buffers and indexes them by m_pi (IExtraSearcher.h:114-122,
    // ExtraFullGraphSearcher.h:405, :500): a load of more lists is undefined there
    if (it->hb > p.internal)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "IterativeSearchHeadBatch %d exceeds SearchInternalResultNum %d", it->hb,
                    p.internal);
    DeviceGuard guard(h->device);
    cudaStream_t stream = nullptr;  // the stream of the head iterator's steps
    const size_t nq = (size_t)it->nq;
    if (it->cap == 0) {  // the first Next creates the QueryResult: its size bounds every later batch
        if (int rc = it->d_heap_d.ensure(nq * batch * 4)) return rc;
        if (int rc = it->d_heap_v.ensure(nq * batch * 4)) return rc;
        it->cap = batch;
    }
    if (int rc = it->d_ids.ensure(nq * batch * 4)) return rc;
    if (int rc = it->d_dists.ensure(nq * batch * 4)) return rc;
    const MetricElem me = metric_elem(h);
    const int per_sm = spann_iter_step_blocks_per_sm(me.cosine, me.elem, it->cap);
    if (per_sm < 1) return fail(SPTAG_B200_MEMORY_OVERFLOW, "the posting step kernel does not fit on an SM");
    const long long max_grid = (long long)h->num_sms * per_sm;
    // SearchIndexIterative's first call: the head's FromNeareast(first = true) at the head batch (SPANNIndex.cpp:271-275)
    if (!it->head->stepped)
        if (int rc = nearest_step(it->head, it->hb, nullptr, nullptr, nullptr)) return rc;
    p.head_ids = (const int*)it->head->d_ids.ptr;
    p.nq = it->nq;
    p.hb = it->hb;
    p.batch = batch;
    p.fresh = 1;
    p.queries = (const unsigned char*)it->d_queries.ptr;
    p.dim = h->dim;
    p.simd_width = h->simd_width;
    p.lists = posting_lists(s, sp.page_limit);
    p.st = (SpannIterState*)it->d_state.ptr;
    p.posts = (int*)it->d_posts.ptr;
    p.heap_d = (float*)it->d_heap_d.ptr;
    p.heap_v = (int*)it->d_heap_v.ptr;
    p.cap = it->cap;
    p.tables = (unsigned int* const*)it->dedup.d_tables.ptr;
    p.dedup = it->dedup.state;
    p.out_ids = (int*)it->d_ids.ptr;
    p.out_dists = (float*)it->d_dists.ptr;
    p.out_counts = (int*)it->d_counts.ptr;
    p.out_relaxed = (unsigned char*)it->d_relaxed.ptr;
    auto lists = [&](int refill, int susp, bool clear_refill) -> int {
        p.refill = (unsigned int*)it->d_refill[refill].ptr;
        p.susp = (unsigned int*)it->d_susp[susp].ptr;
        if (clear_refill) CUDA_OK(cudaMemsetAsync(p.refill, 0, kIterListHeader * 4, stream));
        CUDA_OK(cudaMemsetAsync(p.susp, 0, kIterListHeader * 4, stream));
        return 0;
    };
    const void* kern = nullptr;
    auto step = [&](const SpannIterParams& sp_, long long n) -> int {
        const cudaError_t e = launch_spann_iter_step(sp_, me.cosine, me.elem, (int)std::min(n, max_grid), stream, &kern);
        g_launches++;
        if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "posting step launch failed: %s", cudaGetErrorString(e));
        return 0;
    };
    // Host placement: a staging set for the call, whose stage each launch's rounds fill (gather_rounds over the launch's
    // queries, each round a launch over its sub-list)
    std::unique_lock<std::mutex> slock;
    decltype(s->staging.acquire(slock)) gs = nullptr;
    if (s->host_postings)
        if (int rc = spann_acquire_fitted(s, sp, slock, gs)) return rc;
    long gather_bytes = 0, gather_rounds_n = 0, gather_peer_bytes = 0, read_bytes = 0;
    if (gs) {
        if (int rc = gs->d_chosen.ensure(nq * it->hb * 4)) return rc;
        if (int rc = gs->d_nchosen.ensure(nq * 4)) return rc;
        if (int rc = gs->d_sub.ensure((kIterListHeader + nq) * 4)) return rc;
    }
    auto launch = [&](long long n) -> int {
        if (!gs) return step(p, n);
        unsigned int* sub = (unsigned int*)gs->d_sub.ptr;
        auto choose = [&](int b, int e, const int*& chosen, const int*& nchosen) {
            chosen = (const int*)gs->d_chosen.ptr;
            nchosen = (const int*)gs->d_nchosen.ptr;
            const cudaError_t err = launch_spann_iter_chosen(p, b, e, (int*)gs->d_chosen.ptr, (int*)gs->d_nchosen.ptr, sub, stream);
            g_launches++;
            if (err != cudaSuccess) return fail(SPTAG_B200_FAIL, "posting choice launch failed: %s", cudaGetErrorString(err));
            return 0;
        };
        auto run = [&](int b, int e, const PostingLists& view) {
            SpannIterParams r = p;
            r.list = sub;
            r.lists = view;
            return step(r, e - b);
        };
        return gather_rounds(s, *gs, sp, (int)n, it->hb, stream, choose, run, gather_bytes, gather_rounds_n,
                             gather_peer_bytes, read_bytes);
    };
    // Rounds: the posting step over the queries of the round; queries whose tables must grow run again (same round);
    // then the head's FromNeareast(false) for the queries whose postings ran out, and the posting step over those.
    int cur = 0, scur = 0;
    if (int rc = lists(cur, scur, true)) return rc;
    if (int rc = launch(it->nq)) return rc;
    p.fresh = 0;
    long rounds = 0;
    for (;;) {
        unsigned hdr[2][kIterListHeader];  // the refill and suspension lists' headers, read with one synchronisation
        CUDA_OK(cudaMemcpyAsync(hdr[0], p.refill, sizeof(hdr[0]), cudaMemcpyDeviceToHost, stream));
        if (int rc = it->dedup.double_listed(p.susp, hdr[1], true, stream)) return rc;
        if (hdr[1][0] > 0) {  // the listed tables doubled: run those queries on (they append to the same refill list)
            p.list = p.susp;
            scur ^= 1;
            if (int rc = lists(cur, scur, false)) return rc;
            if (int rc = launch(hdr[1][0])) return rc;
            continue;
        }
        if (hdr[0][0] == 0) break;
        // SearchIndexIterativeFromNeareast(head, false) for the queries on the refill list (SPANNIndex.cpp:281-285)
        if (int rc = nearest_step(it->head, it->hb, nullptr, nullptr, p.refill)) return rc;
        ++rounds;
        p.list = p.refill;
        cur ^= 1;
        if (int rc = lists(cur, scur, true)) return rc;
        if (int rc = launch(hdr[0][0])) return rc;
    }
    CUDA_OK(cudaMemcpyAsync(out_ids, it->d_ids.ptr, nq * batch * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_dists, it->d_dists.ptr, nq * batch * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_counts, it->d_counts.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_relaxed_mono, it->d_relaxed.ptr, nq, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    std::lock_guard<std::mutex> lock(s->mu);
    s->last_iter_rounds = rounds;
    s->last_iter_dedup_bytes = (long)it->dedup.bytes();
    if (kern) s->last_posting_kernel = kern;
    if (gs) {
        s->last_gather_bytes = gather_bytes;
        s->last_gather_rounds = gather_rounds_n;
        s->last_peer_gather_bytes = gather_peer_bytes;
        s->last_read_bytes = read_bytes;
    }
    return SPTAG_B200_SUCCESS;
}

void sptag_b200_spann_iterator_close(sptag_b200_spann_iter it) {
    if (it) spann_iterator_free(it);
}

}  // extern "C"

// ---- Multi-index scan ----

namespace {

// The per-index iterators of one multi-index scan, closed when the call returns however it returns
struct ScanIterators {
    std::vector<sptag_b200_iter> its;
    ~ScanIterators() {
        for (sptag_b200_iter it : its) sptag_b200_iterator_close(it);
    }
};

}  // namespace

extern "C" {

int sptag_b200_multi_scan(const sptag_b200_handle* indexes, int32_t num_indexes, const void* const* queries,
                          const float* weights, int32_t num_queries, int32_t k, int32_t term_cond, int32_t search_limit,
                          int32_t* out_ids, float* out_scores, int32_t* out_counts, int32_t* out_stats) {
    if (!indexes || !queries || !out_ids || !out_scores || !out_counts || num_queries <= 0)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "null buffer");
    if (num_indexes < 1 || num_indexes > kMultiScanMaxIndexes)
        return fail(SPTAG_B200_LACK_OF_INPUTS, "num_indexes = %d outside [1, %d]", num_indexes, kMultiScanMaxIndexes);
    if (k < 1 || k > 1024) return fail(SPTAG_B200_LACK_OF_INPUTS, "k = %d outside [1, 1024]", k);
    const int n = num_indexes;
    for (int i = 0; i < n; ++i)
        if (!indexes[i] || !queries[i]) return fail(SPTAG_B200_LACK_OF_INPUTS, "null handle or query buffer of index %d", i);
    sptag_b200_index* h0 = indexes[0];
    for (int i = 0; i < n; ++i) {
        sptag_b200_index* h = indexes[i];
        if (h->algo != SPTAG_B200_ALGO_BKT) return fail(SPTAG_B200_FAIL, "ITERATIVE NOT SUPPORT FOR KDT");
        if (h->q_type != 0) return fail(SPTAG_B200_LACK_OF_INPUTS, "iterators on quantized indexes are not built");
        std::lock_guard<std::mutex> lock(h->mu);
        // GetDistance(target_j, vid) reads row vid of every index: they must hold the same ids
        if (h->device != h0->device || h->n != h0->n || h->id_offset != h0->id_offset)
            return fail(SPTAG_B200_LACK_OF_INPUTS, "index %d differs from index 0 in device, vector count or id offset", i);
    }
    // Init: GetIterator(target_i, true) on every index
    ScanIterators iters;
    for (int i = 0; i < n; ++i) {
        sptag_b200_iter it = nullptr;
        if (int rc = sptag_b200_iterator_open_ex(indexes[i], queries[i], num_queries, 1, &it)) return rc;
        iters.its.push_back(it);
    }
    DeviceGuard guard(h0->device);
    cudaStream_t stream = nullptr;  // the stream of the iterator steps
    const size_t nq = (size_t)num_queries;
    std::vector<DeviceBuffer> d_q(n);
    DeviceBuffer d_cross, d_state, d_heap_s, d_heap_v, d_list[2], d_ids, d_scores, d_counts, d_stats, d_seen;
    QueryTables seen;  // seenSet, one table per query; d_seen holds their IterStates
    int bits = 7;
    int rc = 0;
    for (int i = 0; i < n && !rc; ++i) rc = d_q[i].ensure(nq * indexes[i]->row_stride);
    if (rc || (rc = d_cross.ensure(nq * n * n * 4)) || (rc = d_state.ensure(nq * sizeof(MultiScanState))) ||
        (rc = d_heap_s.ensure(nq * k * 4)) || (rc = d_heap_v.ensure(nq * k * 4)) ||
        (rc = d_list[0].ensure((kIterListHeader + nq) * 4)) || (rc = d_list[1].ensure((kIterListHeader + nq) * 4)) ||
        (rc = d_ids.ensure(nq * k * 4)) || (rc = d_scores.ensure(nq * k * 4)) || (rc = d_counts.ensure(nq * 4)) ||
        (rc = d_stats.ensure(nq * 16)) || (rc = d_seen.ensure(nq * sizeof(IterState))))
        return rc;
    const std::vector<MultiScanState> st(nq, MultiScanState{0, 0, -1, 0});
    std::vector<unsigned> list0(kIterListHeader + nq, 0);
    list0[0] = (unsigned)nq;
    for (size_t q = 0; q < nq; ++q) list0[kIterListHeader + q] = (unsigned)q;
    for (int i = 0; i < n; ++i)
        if (int rc2 = upload_query_rows(indexes[i], d_q[i].ptr, queries[i], nq, stream)) return rc2;
    if (int rc2 = seen.open(nq, bits, QueryTables::kNoBitmap, (IterState*)d_seen.ptr)) return rc2;
    CUDA_OK(cudaMemcpy(d_state.ptr, st.data(), nq * sizeof(MultiScanState), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_list[0].ptr, list0.data(), list0.size() * 4, cudaMemcpyHostToDevice));

    MultiScanRound c;
    memset(&c, 0, sizeof(c));
    MultiScanMergeParams mp;
    memset(&mp, 0, sizeof(mp));
    mp.n = n;
    mp.k = k;
    mp.id_offset = h0->id_offset;
    mp.term_cond = (unsigned int)term_cond;
    mp.search_limit = (unsigned long long)(long long)search_limit;
    for (int i = 0; i < n; ++i) mp.weight[i] = weights ? weights[i] : 1.0f;  // rankFunc's sum equals unit weights
    mp.cross = (const float*)d_cross.ptr;
    mp.st = (MultiScanState*)d_state.ptr;
    mp.heap_s = (float*)d_heap_s.ptr;
    mp.heap_v = (int*)d_heap_v.ptr;
    mp.tables = (unsigned int* const*)seen.d_tables.ptr;
    mp.seen = seen.state;
    const int max_grid = std::max(1, h0->num_sms) * 32;
    long long rounds = 0;
    unsigned active = (unsigned)nq;
    for (int cur = 0; active > 0; cur ^= 1, ++rounds) {
        // every running query has run `rounds` rounds and this one inserts at most n ids, and no table holds more than the
        // index's ids: keep every table below half load
        const long long fill_bound = std::min<long long>((long long)n * (rounds + 1), (long long)h0->n);
        if (fill_bound > (1ll << (bits - 1))) {
            std::vector<unsigned> qs(active);
            CUDA_OK(cudaMemcpy(qs.data(), (unsigned*)d_list[cur].ptr + kIterListHeader, active * 4, cudaMemcpyDeviceToHost));
            while (fill_bound > (1ll << (bits - 1))) ++bits;
            if (bits > 30) return fail(SPTAG_B200_MEMORY_OVERFLOW, "seen-set table of 2^%d entries", bits);
            const std::vector<int> nb(active, bits);
            if (int rc2 = seen.grow(qs, nb, true, stream)) return rc2;
        }
        const unsigned* list = (const unsigned*)d_list[cur].ptr;
        for (int i = 0; i < n; ++i)  // Next(1) on every index
            if (int rc2 = next_step(iters.its[i], 1, nullptr, nullptr, nullptr, nullptr, list)) return rc2;
        const int grid = (int)std::min<long long>(active, max_grid);
        for (int i = 0; i < n; ++i) {  // the step's results: [nq x 1], allocated by the first step
            c.ids[i] = (const int*)iters.its[i]->d_ids.ptr;
            c.dists[i] = (const float*)iters.its[i]->d_dists.ptr;
            c.counts[i] = (const int*)iters.its[i]->d_counts.ptr;
        }
        for (int j = 0; j < n && n > 1; ++j) {  // GetDistance(target_j, vid) for the other indexes' candidates
            const sptag_b200_index* h = indexes[j];
            MultiScanDistParams dp;
            dp.list = list;
            dp.n = n;
            dp.target = j;
            dp.id_offset = h0->id_offset;
            dp.c = c;
            dp.queries = (const unsigned char*)d_q[j].ptr;
            dp.rows = (const unsigned char*)h->d_vectors.ptr;
            dp.row_stride = h->row_stride;
            dp.dim = h->dim;
            dp.simd_width = h->simd_width;
            dp.cross = (float*)d_cross.ptr;
            const MetricElem me = metric_elem(h);
            const cudaError_t e = launch_multi_scan_distance(dp, me.cosine, me.elem, grid, stream);
            g_launches++;
            if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "multi-scan distance launch failed: %s", cudaGetErrorString(e));
        }
        mp.c = c;
        mp.list = list;
        mp.next = (unsigned*)d_list[cur ^ 1].ptr;
        CUDA_OK(cudaMemsetAsync(mp.next, 0, kIterListHeader * 4, stream));
        const cudaError_t e = launch_multi_scan_merge(mp, grid, stream);
        g_launches++;
        if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "multi-scan merge launch failed: %s", cudaGetErrorString(e));
        CUDA_OK(cudaMemcpyAsync(&active, mp.next, 4, cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
    }
    MultiScanDrainParams dr;
    dr.nq = num_queries;
    dr.k = k;
    dr.id_offset = h0->id_offset;
    dr.st = (MultiScanState*)d_state.ptr;
    dr.seen = seen.state;
    dr.heap_s = (float*)d_heap_s.ptr;
    dr.heap_v = (int*)d_heap_v.ptr;
    dr.out_ids = (int*)d_ids.ptr;
    dr.out_scores = (float*)d_scores.ptr;
    dr.out_counts = (int*)d_counts.ptr;
    dr.out_stats = (int*)d_stats.ptr;
    const cudaError_t e = launch_multi_scan_drain(dr, (int)std::min<long long>((long long)nq, max_grid), stream);
    g_launches++;
    if (e != cudaSuccess) return fail(SPTAG_B200_FAIL, "multi-scan drain launch failed: %s", cudaGetErrorString(e));
    CUDA_OK(cudaMemcpyAsync(out_ids, d_ids.ptr, nq * k * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_scores, d_scores.ptr, nq * k * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpyAsync(out_counts, d_counts.ptr, nq * 4, cudaMemcpyDeviceToHost, stream));
    if (out_stats) CUDA_OK(cudaMemcpyAsync(out_stats, d_stats.ptr, nq * 16, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    return SPTAG_B200_SUCCESS;
}

}  // extern "C"
