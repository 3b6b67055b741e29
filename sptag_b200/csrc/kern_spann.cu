// SPANN posting scan (SPANN::Index<T>::SearchIndex after its head search, SPANNIndex.cpp:193-250, and
// ExtraFullGraphSearcher<T>::SearchIndex, ExtraFullGraphSearcher.h:226-375), one warp per query:
//   translate the head results and choose the postings (lane 0, in result order), Reverse(), then for every chosen list
//   and element in order: the deduper, the distance (the head index's DistanceUtils tree, a half-warp per row) and
//   QueryResultSet::AddPoint, then SortResult (QueryResultSet.h:77-112).
// AddPoint's Heapify stops at `next < maxidx`, so which entries survive depends on the insertion order: the heap is
// replayed in element order by one lane.  The lanes only skip work: a candidate that does not beat the current root
// cannot beat any later root (a replacement never raises the root), so each chunk tests its candidates against the
// root, applies the first that beats it, and re-tests the rest against the new root.
#include "spann_device.cuh"
#include "spann_scan.h"

#include <climits>

namespace sptag_b200 {
namespace {

template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32) spann_scan_kernel(const SpannScanParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x, j = lane & 15, half = lane >> 4;
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
            // SPANNIndex.cpp:213-234: limitDist = result[0].Dist * MaxDistRatio (float), then per result until VID -1
            const float limit = __fmul_rn(rd[0], p.max_dist_ratio);
            int np = 0;
            long long total = 0;
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
                const int tc = searched_count(p, pid);
                if (tc == 0) continue;  // CheckValidPosting (:931-934)
                posts[np++] = pid;
                total += tc;
            }
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
        const unsigned char* qrow = p.queries + (size_t)q * p.row_stride;
        int elements = 0, ndist = 0;
        for (int pi = 0; pi < np; ++pi) {
            const int l = posts[pi];
            const int tc = searched_count(p, l);
            elements += tc;
            for (int base = 0; base < tc; base += 32) {
                const int i = base + lane;
                const bool in = i < tc;
                const int vid = in ? p.ids[p.off[l] + i] : 0;
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
                for (int r0 = 0; r0 < cnt; r0 += 2) {
                    const int r = min(r0 + half, cnt - 1);
                    const unsigned char* row = p.rows + (size_t)(p.off[l] + cl[r]) * p.row_stride;
                    const float d = spann_distance<COSINE, ELEM>(row, qrow, p.dim, j, p.simd_width);
                    if (j == 0 && r0 + half < cnt) cd[r] = d;
                }
                ndist += cnt;
                __syncwarp();
                // AddPoint in element order (QueryResultSet.h:77-87)
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
                        heapify(rd, rv, p.w);
                    }
                    __syncwarp();
                    from = first + 1;
                }
                __syncwarp();
            }
        }
        if (lane == 0) {  // SortResult (QueryResultSet.h:89-96)
            for (int i = p.w - 1; i >= 0; --i) {
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

size_t spann_scan_smem(int w) { return (size_t)w * 12 + 3 * 32 * 4 + 16; }

int spann_scan_blocks_per_sm(bool cosine, int elem, int w) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        return warp_blocks_per_sm((const void*)spann_scan_kernel<cos, el>, spann_scan_smem(w));
    });
}

cudaError_t launch_spann_scan(const SpannScanParams& p, bool cosine, int elem, int grid, cudaStream_t stream) {
    const size_t smem = spann_scan_smem(p.w);
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        void (*k)(const SpannScanParams) = spann_scan_kernel<cos, el>;
        if (smem > 48 * 1024) {
            cudaError_t e = cudaFuncSetAttribute((const void*)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        k<<<grid, 32, smem, stream>>>(p);
        return cudaGetLastError();
    });
}


}  // namespace sptag_b200
