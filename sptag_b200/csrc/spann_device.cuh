// spann_device.cuh -- pieces shared by the posting-side kernels: the SPANN posting scans (kern_spann.cu on raw rows,
// kern_spann_pq.cu on PQ code rows), the posting step of SPANN iterators (kern_spann_iter.cu) and the multi-index scan's
// cross distances (kern_multi_scan.cu).  QueryResultSet's comparator, Heapify, AddPoint of a chunk and SortResult, the
// distance and the row distance of a chunk, LoadingHeadInfo's truncation, the posting scan's body, and the launchers'
// dispatch, occupancy query and launch.
#pragma once
#include "search_kernels.cuh"
#include "spann_scan.h"

#include <climits>
#include <type_traits>

namespace sptag_b200 {
namespace {

// Calls f(cos, el) with the runtime metric flag and element code (0 float, 1 int8, 2 uint8, 3 int16) as compile-time
// constants (std::bool_constant, std::integral_constant<int, ELEM>), so that f can name its kernel's <COSINE, ELEM>
// instantiation
template <typename F>
auto with_cosine_elem(bool cosine, int elem, F&& f) {
    using T = std::true_type;
    using N = std::false_type;
    switch (elem) {
    case 1: return cosine ? f(T(), std::integral_constant<int, 1>()) : f(N(), std::integral_constant<int, 1>());
    case 2: return cosine ? f(T(), std::integral_constant<int, 2>()) : f(N(), std::integral_constant<int, 2>());
    case 3: return cosine ? f(T(), std::integral_constant<int, 3>()) : f(N(), std::integral_constant<int, 3>());
    default: return cosine ? f(T(), std::integral_constant<int, 0>()) : f(N(), std::integral_constant<int, 0>());
    }
}

// Blocks of one warp of kernel k with smem bytes of dynamic shared memory that fit on one SM (0: none, or the query
// failed)
inline int warp_blocks_per_sm(const void* k, size_t smem) {
    int fit = 0;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fit, k, 32, smem) != cudaSuccess) return 0;
    return fit;
}

// Launches kernel k on `grid` blocks of one warp with smem bytes of dynamic shared memory; returns the launch error
template <typename P>
cudaError_t launch_warp_blocks(void (*k)(P), const P& p, int grid, size_t smem, cudaStream_t stream) {
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    k<<<grid, 32, smem, stream>>>(p);
    return cudaGetLastError();
}

// BasicResult operator< (QueryResultSet.h:17-20)
__device__ __forceinline__ bool res_less(float da, int va, float db, int vb) {
    return da < db || (da == db && va < vb);
}

// QueryResultSet::Heapify(count) on (dist, vid) arrays, exactly as written (QueryResultSet.h:99-112)
__device__ void heapify(float* d, int* v, int count) {
    int parent = 0, next = 1;
    const int maxidx = count - 1;
    while (next < maxidx) {
        if (res_less(d[next], v[next], d[next + 1], v[next + 1])) next++;
        if (res_less(d[parent], v[parent], d[next], v[next])) {
            const float td = d[next];
            const int tv = v[next];
            d[next] = d[parent];
            v[next] = v[parent];
            d[parent] = td;
            v[parent] = tv;
            parent = next;
            next = (parent << 1) + 1;
        } else {
            break;
        }
    }
    if (next == maxidx && res_less(d[parent], v[parent], d[next], v[next])) {
        const float td = d[next];
        const int tv = v[next];
        d[next] = d[parent];
        v[next] = v[parent];
        d[parent] = td;
        v[parent] = tv;
    }
}

// QueryResultSet::AddPoint (QueryResultSet.h:77-87) of a chunk's cnt (<= 32) candidates (cd, cv), in element order, into
// the size-entry heap (rd, rv).  AddPoint's Heapify stops at `next < maxidx`, so which entries survive depends on the
// insertion order: the heap is replayed in element order by one lane.  The lanes only skip work: a candidate that does
// not beat the current root cannot beat any later root (a replacement never raises the root), so the chunk's candidates
// are tested against the root, the first that beats it is applied, and the rest are re-tested against the new root.  The
// warp calls it together after a __syncwarp.
__device__ __forceinline__ void add_points(float* rd, int* rv, int size, const float* cd, const int* cv, int cnt) {
    const int lane = threadIdx.x;
    int from = 0;
    for (;;) {
        const float root_d = rd[0];
        const int root_v = rv[0];
        const bool beats = lane >= from && lane < cnt && res_less(cd[lane], cv[lane], root_d, root_v);
        const unsigned bm = __ballot_sync(kFull, beats);
        if (bm == 0) break;
        const int first = __ffs(bm) - 1;
        if (lane == 0) {
            rd[0] = cd[first];
            rv[0] = cv[first];
            heapify(rd, rv, size);
        }
        __syncwarp();
        from = first + 1;
    }
    __syncwarp();
}

// QueryResultSet::SortResult (QueryResultSet.h:89-96) of the size-entry heap (rd, rv), by lane 0; the warp calls it
// together
__device__ __forceinline__ void sort_result(float* rd, int* rv, int size) {
    if (threadIdx.x == 0) {
        for (int i = size - 1; i >= 0; --i) {
            const float td = rd[0];
            const int tv = rv[0];
            rd[0] = rd[i];
            rv[0] = rv[i];
            rd[i] = td;
            rv[i] = tv;
            heapify(rd, rv, i);
        }
    }
    __syncwarp();
}

// ComputeDistance(query, row) by one half-warp with the trees of the search kernels (both are symmetric bit for bit)
template <bool COSINE, int ELEM>
__device__ __forceinline__ float spann_distance(const unsigned char* row, const unsigned char* q, int dim, int j,
                                                int simd_width) {
    if (ELEM == 0) {
        QueryRegs<0> qr;
        if (simd_width != 16)
            return half_warp_distance_w<COSINE>(reinterpret_cast<const float*>(row), reinterpret_cast<const float*>(q), dim, j,
                                                simd_width);
        return half_warp_distance<0, COSINE>(reinterpret_cast<const float*>(row), qr, reinterpret_cast<const float*>(q), dim, j);
    }
    return half_warp_distance_elem_w<COSINE, ELEM>(row, q, dim, j, simd_width);
}

// Elements of list l that a search reads (posting_searched)
__device__ __forceinline__ int searched_count(const PostingLists pl, int l) {
    return posting_searched(pl.cnt[l], pl.pages[l], pl.page_limit, pl.vector_info_size);
}

// The postings a search reads (SPANNIndex.cpp:213-234), by one lane: limitDist = result[0].Dist * MaxDistRatio (float),
// then per head result until VID -1: translate it in place in (rd, rv) (INT_MAX: no vector, (MaxDist, -1)), and choose
// its list while fewer than SearchInternalResultNum are chosen, its distance is within limitDist and the list holds
// elements at the page limit (CheckValidPosting, :931-934).  Appends the chosen lists to posts in result order, counting
// them in np and their elements in total (both start at 0).  The posting scan reads exactly these lists.  (p by
// reference and np / total as the caller's variables: so the scan's instructions stay those of the rule written out.)
__device__ __forceinline__ void choose_postings(const SpannScanParams& p, float* rd, int* rv, int* posts, int& np,
                                                long long& total) {
    const float limit = __fmul_rn(rd[0], p.max_dist_ratio);
    for (int i = 0; i < p.w; ++i) {
        const int pid = rv[i];
        if (pid == -1) break;
        const int t = p.translate[pid];
        if (t == INT_MAX) {
            rv[i] = -1;
            rd[i] = SPTAG_B200_MAXDIST;
        } else {
            rv[i] = t;
        }
        if (np >= p.internal || ((double)limit > 0.1 && rd[i] > limit)) continue;
        const int tc = searched_count(p.lists, pid);
        if (tc == 0) continue;
        posts[np++] = pid;
        total += tc;
    }
}

// SearchDiskIndexIterative's load of the head iterator's latest batch for query q (SPANNIndex.cpp:420-442), by one lane:
// its lists up to the first -1 that hold elements at the page limit (CheckValidPosting), in result order, written to
// posts; returns their number
__device__ __forceinline__ int load_postings(const SpannIterParams p, int q, int* posts) {
    int m = 0;
    for (int i = 0; i < p.hb; ++i) {
        const int pid = p.head_ids[(size_t)q * p.hb + i];
        if (pid == -1) break;
        if (searched_count(p.lists, pid) > 0) posts[m++] = pid;
    }
    return m;
}

// The distances of a chunk to the query row qrow on raw rows: a half-warp per row, two rows at a time, with the head
// index's DistanceUtils tree.  chunk(pl, base, cl, cnt, cd): cd[r] = the distance to element cl[r] of the list whose first
// element is base (its off[l]), for r < cnt.
template <bool COSINE, int ELEM>
struct RowDistance {
    const unsigned char* qrow;
    int dim, simd_width;
    int j, half;  // the lane's place in its half-warp, and which half-warp

    __device__ __forceinline__ void begin_query(const SpannScanParams& p, int q) {
        qrow = p.queries + (size_t)q * p.lists.row_stride;
    }

    __device__ __forceinline__ void chunk(const PostingLists pl, long long base, const int* cl, int cnt, float* cd) {
        for (int r0 = 0; r0 < cnt; r0 += 2) {
            const int r = min(r0 + half, cnt - 1);
            const unsigned char* row = pl.rows + (size_t)(base + cl[r]) * pl.row_stride;
            const float d = spann_distance<COSINE, ELEM>(row, qrow, dim, j, simd_width);
            if (j == 0 && r0 + half < cnt) cd[r] = d;
        }
    }
};

// The SPANN posting scan (SPANN::Index<T>::SearchIndex after its head search, SPANNIndex.cpp:193-250, and
// ExtraFullGraphSearcher<T>::SearchIndex, ExtraFullGraphSearcher.h:226-375), one warp per query:
//   translate the head results and choose the postings (lane 0, in result order), Reverse(), then for every chosen list
//   and element in order: the deduper, the distance and add_points, then sort_result.
// Dist is the distance of one flavour (kern_spann.cu: RowDistance on raw rows, kern_spann_pq.cu: PQ code rows):
//   dist.begin_query(p, q)                    before the first list of query q (the warp is converged)
//   dist.chunk(p.lists, first, cl, cnt, cd)   cd[r] = distance of the query to element cl[r] of the list whose first
//                                             element is first, for r < cnt (<= 32); the warp calls it together, cd is
//                                             read after a __syncwarp
// smem holds spann_scan_smem(p.w) bytes.  p is taken by value, and so are the posting-list views of the helpers: with a
// reference the raw-row kernels' instructions differed from those of the scan written out in the kernel, with a copy only
// the registers of two parameter loads do.
template <typename Dist>
__device__ __forceinline__ void spann_scan_body(const SpannScanParams p, unsigned char* smem, Dist& dist) {
    const int lane = threadIdx.x;
    float* rd = reinterpret_cast<float*>(smem);            // m_results dists [w]
    int* rv = reinterpret_cast<int*>(rd + p.w);            // m_results vids [w]
    int* posts = rv + p.w;                                 // m_postingIDs [w]
    float* cd = reinterpret_cast<float*>(posts + p.w);     // chunk candidates [32]
    int* cv = reinterpret_cast<int*>(cd + 32);
    int* cl = cv + 32;                                     // candidate element index in its list
    int* shared_int = cl + 32;                             // [0] postings chosen, [1] table entries in use
    int* table = p.tables + (size_t)blockIdx.x * p.table_entries;
    for (int q = blockIdx.x; q < p.nq; q += gridDim.x) {
        const int* hid = p.head_ids + (size_t)q * p.w;
        const float* hd = p.head_dists + (size_t)q * p.w;
        for (int i = lane; i < p.w; i += 32) {
            rv[i] = hid[i];
            rd[i] = hd[i];
        }
        __syncwarp();
        if (lane == 0) {
            int np = 0;
            long long total = 0;
            choose_postings(p, rd, rv, posts, np, total);
            shared_int[0] = np;
            // the deduper needs room for every element this query reads; the table keeps at most half its entries used
            int entries = 64;
            while (entries < p.table_entries && (long long)entries < 2 * total) entries <<= 1;
            shared_int[1] = entries;
        }
        __syncwarp();
        const int np = shared_int[0], entries = shared_int[1];
        for (int i = lane; i < entries; i += 32) table[i] = 0;
        for (int i = lane; i < p.w / 2; i += 32) {  // Reverse()
            const int o = p.w - 1 - i;
            const float td = rd[i];
            const int tv = rv[i];
            rd[i] = rd[o];
            rv[i] = rv[o];
            rd[o] = td;
            rv[o] = tv;
        }
        __syncwarp();
        dist.begin_query(p, q);
        int elements = 0, ndist = 0;
        for (int pi = 0; pi < np; ++pi) {
            const int l = posts[pi];
            const int tc = searched_count(p.lists, l);
            const long long first = p.lists.off[l];
            elements += tc;
            for (int base = 0; base < tc; base += 32) {
                const int i = base + lane;
                const bool in = i < tc;
                const int vid = in ? p.lists.ids[first + i] : 0;
                // m_deduper.CheckAndSet(vid) in element order (WorkSpace.h:113-117): an id seen earlier is skipped.  Among
                // equal ids of this chunk only the lowest lane may insert; -1 maps to the empty key and is never "seen".
                const unsigned same = __match_any_sync(kFull, in ? vid : INT_MIN);
                bool keep = in && (vid == -1 || (__ffs(same) - 1) == lane);
                if (keep && vid != -1) {
                    const unsigned key = (unsigned)vid + 1u;
                    unsigned h = vhash_home(key, 32 - __ffs(entries) + 1) & (unsigned)(entries - 1);
                    for (;;) {
                        const int prev = atomicCAS(&table[h], 0, (int)key);
                        if (prev == 0) break;
                        if (prev == (int)key) {
                            keep = false;
                            break;
                        }
                        h = (h + 1) & (unsigned)(entries - 1);
                    }
                }
                const unsigned km = __ballot_sync(kFull, keep);
                const int cnt = __popc(km);
                if (keep) {
                    const int slot = __popc(km & ((1u << lane) - 1u));
                    cv[slot] = vid;
                    cl[slot] = i;
                }
                __syncwarp();
                dist.chunk(p.lists, first, cl, cnt, cd);
                ndist += cnt;
                __syncwarp();
                add_points(rd, rv, p.w, cd, cv, cnt);
            }
        }
        sort_result(rd, rv, p.w);
        for (int i = lane; i < p.k; i += 32) {
            p.out_ids[(size_t)q * p.k + i] = rv[i];
            p.out_dists[(size_t)q * p.k + i] = rd[i];
        }
        if (p.out_stats && lane == 0) {
            p.out_stats[(size_t)q * 3 + 0] = np;
            p.out_stats[(size_t)q * 3 + 1] = elements;
            p.out_stats[(size_t)q * 3 + 2] = ndist;
        }
        __syncwarp();
    }
}

}  // namespace
}  // namespace sptag_b200
