// The kernels of a multi-index scan (multi_scan.h): the cross distances of a round's candidates, the merge that replays
// MultiIndexScan::Next's loop body (MultiIndexScan.cpp:87-160) and the final drain, in a translation unit of their own.
#include "multi_scan.h"
#include "spann_device.cuh"

namespace sptag_b200 {
namespace {

// One warp per running query; each half-warp computes GetDistance(target_j, vid) = ComputeDistance(target_j, row_j[vid])
// (BKT/Index.h:145-147) for the candidate of one other index, with index j's summation tree.  Both halves always run the
// distance (its shuffles span the warp); a half without a candidate reads row 0 and drops the value.
template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32) multi_scan_distance_kernel(const MultiScanDistParams p) {
    const int lane = threadIdx.x, j = lane & 15, half = lane >> 4;
    const int n_list = (int)p.list[0];
    for (int li = blockIdx.x; li < n_list; li += gridDim.x) {
        const int q = (int)p.list[kIterListHeader + li];
        const unsigned char* qrow = p.queries + (size_t)q * p.row_stride;
        for (int i0 = 0; i0 < p.n; i0 += 2) {
            const int i = i0 + half;
            const bool want = i < p.n && i != p.target && p.c.counts[i][q] > 0;
            const int vid = want ? p.c.ids[i][q] - p.id_offset : 0;
            const float d = spann_distance<COSINE, ELEM>(p.rows + (size_t)vid * p.row_stride, qrow, p.dim, j, p.simd_width);
            if (want && j == 0) p.cross[((size_t)q * p.n + i) * p.n + p.target] = d;
        }
    }
}

// WeightedRankFunc (MultiIndexScan.cpp:41-49) as GCC compiles it with -O3 -march=x86-64-v3: blocks of 8, then one of 4,
// add the rounded products one after another (vmulps + vaddss); the last n % 4 terms are contracted (vfmadd231ss)
__device__ __forceinline__ float weighted_rank(const float* d, const float* w, int n) {
    float acc = 0.0f;
    int i = 0;
    for (; n - i >= 8; i += 8)
        for (int t = 0; t < 8; ++t) acc = __fadd_rn(acc, __fmul_rn(d[i + t], w[i + t]));
    if (n - i >= 4) {
        for (int t = 0; t < 4; ++t) acc = __fadd_rn(acc, __fmul_rn(d[i + t], w[i + t]));
        i += 4;
    }
    for (; i < n; ++i) acc = __fmaf_rn(d[i], w[i], acc);
    return acc;
}

// libstdc++'s heap algorithms (bits/stl_heap.h, GCC 13) on std::priority_queue<pair<float, SizeType>> with
// pq_item_compare (MultiIndexScan.h:67-74): a < b when a.first < b.first; ids never take part
__device__ __forceinline__ void heap_push_hole(float* s, int* v, int hole, int top, float vs, int vv) {
    int parent = (hole - 1) / 2;
    while (hole > top && s[parent] < vs) {
        s[hole] = s[parent];
        v[hole] = v[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    s[hole] = vs;
    v[hole] = vv;
}

// priority_queue::push: push_back + push_heap
__device__ __forceinline__ void heap_push(float* s, int* v, int& size, float vs, int vv) {
    heap_push_hole(s, v, size, 0, vs, vv);
    ++size;
}

// priority_queue::pop: pop_heap (__pop_heap + __adjust_heap) + pop_back
__device__ __forceinline__ void heap_pop(float* s, int* v, int& size) {
    const int len = size - 1;
    if (len > 0) {
        const float vs = s[len];
        const int vv = v[len];
        s[len] = s[0];
        v[len] = v[0];
        int hole = 0, child = 0;
        while (child < (len - 1) / 2) {
            child = 2 * (child + 1);
            if (s[child] < s[child - 1]) child--;
            s[hole] = s[child];
            v[hole] = v[child];
            hole = child;
        }
        if ((len & 1) == 0 && child == (len - 2) / 2) {
            child = 2 * (child + 1);
            s[hole] = s[child - 1];
            v[hole] = v[child - 1];
            hole = child - 1;
        }
        heap_push_hole(s, v, hole, 0, vs, vv);
    }
    size = len;
}

// One warp per running query, the work on lane 0: the round's candidates in index order, as the for loop of
// MultiIndexScan::Next, then its termination test with useTimer = false.  The seen set is inserted into without a
// bound check: the host grows the tables so that a round cannot pass half load.
__global__ void __launch_bounds__(32) multi_scan_merge_kernel(const MultiScanMergeParams p) {
    if (threadIdx.x != 0) return;
    const int n_list = (int)p.list[0];
    for (int li = blockIdx.x; li < n_list; li += gridDim.x) {
        const int q = (int)p.list[kIterListHeader + li];
        MultiScanState st = p.st[q];
        IterState& ss = p.seen[q];
        unsigned int* table = p.tables[q];
        const int bits = ss.vbits;
        const unsigned mask = (1u << bits) - 1u;
        int fill = ss.vfill;
        float* hs = p.heap_s + (size_t)q * p.k;
        int* hv = p.heap_v + (size_t)q * p.k;
        int end = -1;
        for (int i = 0; i < p.n; ++i) {
            if (p.c.counts[i][q] == 0) {  // "no more result": terminate, the indexes after i are not asked
                end = 2 + i;
                break;
            }
            const int vid = p.c.ids[i][q] - p.id_offset;
            const unsigned key = (unsigned)vid + 1u;
            unsigned h = vhash_home((unsigned)vid, 32 - bits), cur;
            while ((cur = table[h]) != 0u && cur != key) h = (h + 1u) & mask;
            if (cur == key) continue;  // seen: nothing changes
            table[h] = key;
            ++fill;
            float d[kMultiScanMaxIndexes];
            for (int j = 0; j < p.n; ++j) d[j] = j == i ? p.c.dists[i][q] : p.cross[((size_t)q * p.n + i) * p.n + j];
            const float score = weighted_rank(d, p.weight, p.n);
            if (st.size == p.k && hs[0] <= score) {
                ++st.drops;
            } else {
                st.drops = 0;
                if (st.size == p.k) heap_pop(hs, hv, st.size);
                heap_push(hs, hv, st.size, score, vid);
            }
        }
        ++st.rounds;
        if (end < 0) {
            if ((unsigned)st.drops >= p.term_cond)
                end = 0;
            else if ((unsigned long long)fill >= p.search_limit)
                end = 1;
        }
        st.end = end;
        p.st[q] = st;
        ss.vfill = fill;
        if (end < 0) p.next[kIterListHeader + atomicAdd(p.next, 1u)] = (unsigned)q;
    }
}

// Next until false: pq drained largest first onto outputStk, which pops smallest first (MultiIndexScan.cpp:150-170)
__global__ void __launch_bounds__(32) multi_scan_drain_kernel(const MultiScanDrainParams p) {
    for (int q = blockIdx.x; q < p.nq; q += gridDim.x) {
        const MultiScanState st = p.st[q];
        int* oi = p.out_ids + (size_t)q * p.k;
        float* os = p.out_scores + (size_t)q * p.k;
        if (threadIdx.x == 0) {
            float* hs = p.heap_s + (size_t)q * p.k;
            int* hv = p.heap_v + (size_t)q * p.k;
            int size = st.size;
            for (int t = st.size - 1; t >= 0; --t) {
                oi[t] = hv[0] + p.id_offset;
                os[t] = hs[0];
                heap_pop(hs, hv, size);
            }
            p.out_counts[q] = st.size;
            if (p.out_stats) {
                int* o = p.out_stats + (size_t)q * 4;
                o[0] = st.rounds;
                o[1] = p.seen[q].vfill;
                o[2] = st.drops;
                o[3] = st.end;
            }
        }
        for (int t = st.size + (int)threadIdx.x; t < p.k; t += 32) {
            oi[t] = -1;
            os[t] = SPTAG_B200_MAXDIST;
        }
    }
}

}  // namespace

cudaError_t launch_multi_scan_distance(const MultiScanDistParams& p, bool cosine, int elem, int grid, cudaStream_t stream) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        multi_scan_distance_kernel<cos, el><<<grid, 32, 0, stream>>>(p);
        return cudaGetLastError();
    });
}

cudaError_t launch_multi_scan_merge(const MultiScanMergeParams& p, int grid, cudaStream_t stream) {
    multi_scan_merge_kernel<<<grid, 32, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_multi_scan_drain(const MultiScanDrainParams& p, int grid, cudaStream_t stream) {
    multi_scan_drain_kernel<<<grid, 32, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace sptag_b200
