// The posting step of SPANN iterators (SpannIterParams, spann_scan.h), in a translation unit of its own so that the
// posting scan kernel's code does not change with it.  Its row distance and result set are the posting scan's
// (spann_device.cuh).
#include "spann_device.cuh"
#include "spann_scan.h"

#include <climits>

namespace sptag_b200 {
namespace {

// The posting step of SPANN iterators (SpannIterParams), one warp per query.  The reference finds one new element per
// SearchNextInPosting call: offset++, skip the element if m_deduper.CheckAndSet reports it seen, else ComputeDistance +
// AddPoint and stop; at the end of a list pi++, offset = 0; the call returns !(pi == postingIDs.size())
// (ExtraFullGraphSearcher.h:131-147, :492-510), and SearchIndexIterative counts a result when it returns true.  Here a
// chunk of up to 32 elements at (pi, offset) is looked up in the deduper without inserting; an element is new if it is not
// in the set and is the first of its id in the chunk (-1 is always new: its key is the empty key).  The chunk is cut after
// the (batch - count)-th new element, so that only the elements the reference's calls consume are inserted and offset
// ends where the reference's does; the kept elements get their distances and add_points in element order.  A new element
// that is the last one of the last list is AddPoint'ed and inserted, but its call returns false: it is not counted and the
// head is asked for its next batch.
template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(32) spann_iter_step_kernel(const SpannIterParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x;
    float* rd = reinterpret_cast<float*>(smem);         // the call's QueryResult [batch]
    int* rv = reinterpret_cast<int*>(rd + p.cap);
    float* cd = reinterpret_cast<float*>(rv + p.cap);   // chunk candidates [32]
    int* cv = reinterpret_cast<int*>(cd + 32);
    int* cl = cv + 32;                                  // candidate element index in its list
    int* shared_int = cl + 32;                          // [0] postings chosen
    const int n = p.list ? (int)p.list[0] : p.nq;
    for (int li = blockIdx.x; li < n; li += gridDim.x) {
        const int q = p.list ? (int)p.list[kIterListHeader + li] : li;
        SpannIterState& st = p.st[q];
        IterState& ds = p.dedup[q];
        int* posts = p.posts + (size_t)q * p.hb;
        float* hd = p.heap_d + (size_t)q * p.cap;
        int* hv = p.heap_v + (size_t)q * p.cap;
        int np = st.np, pi = st.pi, offset = st.offset, loaded = st.loaded, relaxed = st.relaxed, load = st.load;
        int count = st.count, batch = st.batch;
        const int slots = st.slots;
        bool stop = false;
        if (p.fresh) {
            // Next(batch): the first call sizes the QueryResult, a later one is capped by its result count; then Reset()
            // (SPANNResultIterator.h:39-49)
            batch = slots < 0 ? p.batch : min(p.batch, slots);
            count = 0;
            for (int i = lane; i < batch; i += 32) {
                rd[i] = SPTAG_B200_MAXDIST;
                rv[i] = -1;
            }
        } else {
            for (int i = lane; i < batch; i += 32) {
                rd[i] = hd[i];
                rv[i] = hv[i];
            }
            // continueSearch = SearchIndexIterativeFromNeareast(head, false): false when its first result is no vector
            // (SPANNIndex.cpp:283-285, BKTIndex.cpp:580-583)
            if (st.await_head) stop = p.head_ids[(size_t)q * p.hb] < 0;
        }
        unsigned int* table = p.tables[q];
        const int bits = ds.vbits;
        const unsigned mask = (1u << bits) - 1u;
        int fill = ds.vfill;
        RowDistance<COSINE, ELEM> dist{p.queries + (size_t)q * p.lists.row_stride, p.dim, p.simd_width, lane & 15, lane >> 4};
        int outcome = 0;  // 0: the call ends here, 1: the postings ran out (refill), 2: the table must grow (suspend)
        __syncwarp();
        while (!stop && count < batch) {
            if (load) {  // SearchDiskIndexIterative with m_loadPosting (SPANNIndex.cpp:420-442)
                if (lane == 0) shared_int[0] = load_postings(p, q, posts);
                __syncwarp();
                np = shared_int[0];
                if (loaded >= p.internal) relaxed = 1;
                loaded += np;
                pi = offset = 0;
                load = 0;
                __syncwarp();
            }
            if (pi == np) {
                outcome = 1;
                break;
            }
            if (fill + 32 > (1 << (bits - 1))) {
                outcome = 2;
                break;
            }
            const int l = posts[pi];
            const int tc = searched_count(p.lists, l);
            if (offset >= tc) {  // the page limit was lowered since this list was started
                ++pi;
                offset = 0;
                continue;
            }
            const long long base = p.lists.off[l];
            const int i = offset + lane;
            const bool in = i < tc;
            const int vid = in ? p.lists.ids[base + i] : 0;
            bool seen = false;
            if (in && vid != -1) {  // the deduper's lookup, without the insert (L2: the inserts are atomics)
                const unsigned key = (unsigned)vid + 1u;
                for (unsigned h = vhash_home((unsigned)vid, 32 - bits), cur; (cur = __ldcg(&table[h])) != 0u; h = (h + 1u) & mask)
                    if (cur == key) {
                        seen = true;
                        break;
                    }
            }
            const unsigned same = __match_any_sync(kFull, in ? vid : INT_MIN);
            const bool is_new = in && (vid == -1 || (!seen && (__ffs(same) - 1) == lane));
            const unsigned nm = __ballot_sync(kFull, is_new);
            const int need = batch - count;
            int end = min(32, tc - offset);  // elements the reference's calls consume from this chunk
            if (__popc(nm) > need) {
                unsigned m = nm;
                for (int k = 1; k < need; ++k) m &= m - 1u;
                end = __ffs(m);
            }
            const unsigned km = end == 32 ? nm : nm & ((1u << end) - 1u);
            const bool keep = (km >> lane) & 1u;
            if (keep && vid != -1) {  // the kept ids are distinct and not in the table
                unsigned h = vhash_home((unsigned)vid, 32 - bits);
                while (atomicCAS(&table[h], 0u, (unsigned)vid + 1u) != 0u) h = (h + 1u) & mask;
            }
            fill += __popc(__ballot_sync(kFull, keep && vid != -1));
            const int cnt = __popc(km);
            if (keep) {
                const int slot = __popc(km & ((1u << lane) - 1u));
                cv[slot] = vid;
                cl[slot] = i;
            }
            __syncwarp();
            dist.chunk(p.lists, base, cl, cnt, cd);
            __syncwarp();
            add_points(rd, rv, batch, cd, cv, cnt);
            offset += end;
            const bool last_of_last = pi == np - 1 && offset == tc && ((km >> (end - 1)) & 1u);
            if (offset == tc) {
                ++pi;
                offset = 0;
            }
            count += cnt - (last_of_last ? 1 : 0);
        }
        if (outcome == 0) {
            sort_result(rd, rv, batch);
            for (int i = lane; i < p.batch; i += 32) {  // SetResultNum(resultCount)
                p.out_ids[(size_t)q * p.batch + i] = i < count ? rv[i] : -1;
                p.out_dists[(size_t)q * p.batch + i] = i < count ? rd[i] : SPTAG_B200_MAXDIST;
            }
        } else {
            for (int i = lane; i < batch; i += 32) {
                hd[i] = rd[i];
                hv[i] = rv[i];
            }
            if (lane == 0) {
                unsigned int* to = outcome == 1 ? p.refill : p.susp;
                to[kIterListHeader + atomicAdd(to, 1u)] = (unsigned)q;
            }
        }
        if (lane == 0) {
            st.np = np;
            st.pi = pi;
            st.offset = offset;
            st.loaded = loaded;
            st.relaxed = relaxed;
            st.load = outcome == 1 ? 1 : load;  // m_loadPosting = true after the head's next batch
            st.count = count;
            st.batch = batch;
            st.slots = outcome == 0 ? count : slots;
            st.await_head = outcome == 1;
            ds.vfill = fill;
            if (outcome == 0) {
                p.out_counts[q] = count;
                p.out_relaxed[q] = (unsigned char)relaxed;
            }
        }
        __syncwarp();
    }
}

size_t spann_iter_step_smem(int cap) { return (size_t)cap * 8 + 3 * 32 * 4 + 16; }

}  // namespace
int spann_iter_step_blocks_per_sm(bool cosine, int elem, int cap) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        return warp_blocks_per_sm((const void*)spann_iter_step_kernel<cos, el>, spann_iter_step_smem(cap));
    });
}

cudaError_t launch_spann_iter_step(const SpannIterParams& p, bool cosine, int elem, int grid, cudaStream_t stream,
                                   const void** kernel) {
    return with_cosine_elem(cosine, elem, [&](auto cos, auto el) {
        *kernel = (const void*)spann_iter_step_kernel<cos, el>;
        return launch_warp_blocks(spann_iter_step_kernel<cos, el>, p, grid, spann_iter_step_smem(p.cap), stream);
    });
}

}  // namespace sptag_b200
