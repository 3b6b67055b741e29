// aux_kernels.cuh -- the small device kernels around the search kernel: stand-alone distance batch, graph-refinement
// rebuild (RelativeNeighborhoodGraph::RebuildNeighbors), PQ/OPQ query-side kernels and the shard merge.  Included by
// sptag_b200.cu only (the search kernels themselves are instantiated in kern_*.cu).
#pragma once
#include "search_kernels.cuh"

namespace sptag_b200 {

// ------------------------------------------------------------------------------------------
// stand-alone batched distance kernel (inner-loop parity): one half-warp per (query, id)
// ------------------------------------------------------------------------------------------
template <bool COSINE, int ELEM>
__global__ void distance_batch_kernel(const unsigned char* vectors, unsigned long long row_stride_bytes, int n,
                                      int dim, const void* queries_v, int nq, const int* ids, int ids_per_query,
                                      float* out, int simd_width) {
    const int lane = threadIdx.x & 31;
    const int j = lane & 15;
    const long long hw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const long long total = (long long)nq * ids_per_query;
    // all 32 lanes of a warp run the same number of iterations (shuffles inside)
    const long long pair = hw >> 1;
    const long long npairs = (total + 1) >> 1;
    if (pair >= npairs) return;
    const bool valid = hw < total;
    const long long item = valid ? hw : total - 1;
    const int q = (int)(item / ids_per_query);
    const int id = ids[item];
    const bool ok = (id >= 0 && id < n);
    float d;
    if (ELEM == 0) {
        const float* row = reinterpret_cast<const float*>(vectors + (size_t)(ok ? id : 0) * row_stride_bytes);
        const float* qv = reinterpret_cast<const float*>(queries_v) + (size_t)q * dim;
        QueryRegs<0> qr;
        if (simd_width != 16)
            d = half_warp_distance_w<COSINE>(row, qv, dim, j, simd_width);
        else
            d = half_warp_distance<0, COSINE>(row, qr, qv, dim, j);
    } else {
        // the host pads the query stride to a multiple of 4 bytes (2-/4-byte loads in the lane terms)
        const unsigned char* qv = reinterpret_cast<const unsigned char*>(queries_v) +
                                  (size_t)q * (((size_t)dim * (ELEM == 3 ? 2 : 1) + 3) & ~(size_t)3);
        d = half_warp_distance_elem_w<COSINE, ELEM>(vectors + (size_t)(ok ? id : 0) * row_stride_bytes, qv, dim, j, simd_width);
    }
    if (valid && j == 0) out[item] = ok ? d : SPTAG_B200_MAXDIST;
}

// ------------------------------------------------------------------------------------------
// RelativeNeighborhoodGraph::RebuildNeighbors (RelativeNeighborhoodGraph.h:20-38), one warp per node: walk the node's
// ascending refine-search list, keep a candidate unless an already kept neighbour is closer to it than the node is
// (rng_factor * d(kept, cand) < d(node, cand)).  The reference tests the kept neighbours one by one and stops at the
// first that rejects; the verdict is an AND over all of them, so testing two per step (one per half-warp) with an
// early exit is the same function.  Distances are the index's ComputeDistance, i.e. the same summation trees.
// ------------------------------------------------------------------------------------------
template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(128) rebuild_neighbors_kernel(const unsigned char* __restrict__ vectors,
                                                                unsigned long long row_stride_bytes, int dim,
                                                                int first_node, int num_nodes,
                                                                const int* __restrict__ res_ids,
                                                                const float* __restrict__ res_dists, int num_results,
                                                                int neighborhood, float rng_factor,
                                                                int* __restrict__ out_graph, int simd_width) {
    extern __shared__ int kept_sm[];  // neighborhood ints per warp
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = lane & 15, half = lane >> 4;
    const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    if (w >= num_nodes) return;
    int* kept = kept_sm + warp * neighborhood;
    const int node = first_node + (int)w;
    const int* ids = res_ids + (size_t)w * num_results;
    const float* ds = res_dists + (size_t)w * num_results;
    int count = 0;
    for (int r = 0; r < num_results && count < neighborhood; ++r) {
        const int vid = ids[r];
        if (vid < 0) break;
        if (vid == node) continue;
        const float dist = ds[r];
        const unsigned char* cand = vectors + (size_t)vid * row_stride_bytes;
        bool good = true;
        for (int k0 = 0; k0 < count && good; k0 += 2) {
            const int k = min(k0 + half, count - 1);
            const unsigned char* row = vectors + (size_t)kept[k] * row_stride_bytes;
            float d;
            if (ELEM == 0) {
                QueryRegs<0> qr;
                if (simd_width != 16)
                    d = half_warp_distance_w<COSINE>(reinterpret_cast<const float*>(row), reinterpret_cast<const float*>(cand), dim,
                                                     j, simd_width);
                else
                    d = half_warp_distance<0, COSINE>(reinterpret_cast<const float*>(row), qr,
                                                      reinterpret_cast<const float*>(cand), dim, j);
            } else {
                d = half_warp_distance_elem_w<COSINE, ELEM>(row, cand, dim, j, simd_width);
            }
            const bool reject = (j == 0) && (__fmul_rn(rng_factor, d) < dist);
            if (__any_sync(kFull, reject)) good = false;
        }
        if (good) {
            if (lane == 0) kept[count] = vid;
            ++count;
            __syncwarp();
        }
    }
    __syncwarp();
    for (int t = lane; t < neighborhood; t += 32) out_graph[(size_t)w * neighborhood + t] = (t < count) ? kept[t] : -1;
}

// Installing a refined graph: rows whose last slot named a duplicate group keep naming it (NeighborhoodGraph.h:395-401)
// (the row width may change with the install: RefineGraph's passes run on rows NeighborhoodScale times wider)
__global__ void carry_backpointers_kernel(const int* __restrict__ old_graph, int* __restrict__ new_graph, int n, int old_degree,
                                          int new_degree) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int last = old_graph[(size_t)i * old_degree + old_degree - 1];
    if (last < -1) new_graph[(size_t)i * new_degree + new_degree - 1] = last;
}

// ------------------------------------------------------------------------------------------
// Index mutation (AddIndex / DeleteIndex, BKTIndex.cpp:876-970, KDTIndex.cpp:602-696)
// ------------------------------------------------------------------------------------------

// COMMON::Utils::Normalize (CommonUtils.h:62-76) on rows [first, first + num), one thread per row: a double accumulator in
// element order (a product of two values of T is exact in double, so contracting it into an FMA changes nothing), then
// (T)(x / len * base).  The integer casts truncate toward zero like the reference's cvttsd2si.
template <typename T>
__device__ __forceinline__ T cast_from_double(double v) {
    if (sizeof(T) == 4) return (T)__double2float_rn(v);
    return (T)__double2int_rz(v);
}
template <typename T>
__global__ void normalize_rows_kernel(unsigned char* vectors, unsigned long long row_stride_bytes, int first, int num, int dim,
                                      int base) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= num) return;
    T* a = reinterpret_cast<T*>(vectors + (size_t)(first + r) * row_stride_bytes);
    double len = 0.0;
    for (int j = 0; j < dim; ++j) {
        const double v = (double)a[j];
        len = __dadd_rn(len, __dmul_rn(v, v));
    }
    len = __dsqrt_rn(len);
    if (len < 1e-6) {
        const T val = cast_from_double<T>(__dmul_rn(__ddiv_rn(1.0, __dsqrt_rn((double)dim)), (double)base));
        for (int j = 0; j < dim; ++j) a[j] = val;
    } else {
        for (int j = 0; j < dim; ++j) a[j] = cast_from_double<T>(__dmul_rn(__ddiv_rn((double)a[j], len), (double)base));
    }
}

// DeleteIndex(id) for a batch (Labelset::Insert, Labelset.h:59-76) in call order: an id that is out of range, already
// tombstoned, or repeated earlier in the same batch gets VectorNotFound; the first occurrence of a live id tombstones it.
// Three launches: first[id] = INT_MAX, first[id] = min(batch position), then the winners flip the byte and count.
// Only a byte of 1 is a tombstone (Labelset::Contains / Insert test == 1): rows the reference added and saved carry 0xff.
__global__ void tombstone_reset_kernel(const int* __restrict__ ids, int num, int n, int* __restrict__ first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < num && ids[i] >= 0 && ids[i] < n) first[ids[i]] = 0x7fffffff;
}
__global__ void tombstone_order_kernel(const int* __restrict__ ids, int num, int n, int* __restrict__ first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < num && ids[i] >= 0 && ids[i] < n) atomicMin(&first[ids[i]], i);
}
__global__ void tombstone_apply_kernel(const int* __restrict__ ids, int num, int n, const int* __restrict__ first,
                                       signed char* __restrict__ deleted, int* __restrict__ codes, int* __restrict__ count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num) return;
    const int id = ids[i];
    int code = 0x14;  // VectorNotFound
    if (id >= 0 && id < n && first[id] == i && deleted[id] != 1) {
        deleted[id] = 1;
        atomicAdd(count, 1);
        code = 0;
    }
    codes[i] = code;
}

// DeleteIndex(vectors) step for one query (BKTIndex.cpp:882-887): every result with Dist < 1e-6 is tombstoned.  The search
// returned ids plus the shard offset.  One warp.
__global__ void tombstone_close_kernel(const int* __restrict__ ids, const float* __restrict__ dists, int k, int id_offset,
                                       signed char* __restrict__ deleted, int* __restrict__ count) {
    for (int j = threadIdx.x; j < k; j += 32) {
        const int id = ids[j] < 0 ? -1 : ids[j] - id_offset;
        if (id >= 0 && (double)dists[j] < 1e-6 && deleted[id] != 1) {
            deleted[id] = 1;
            atomicAdd(count, 1);
        }
    }
}

// ComputeDistance(a, b) by one half-warp, the summation trees of rebuild_neighbors_kernel (both distances are symmetric
// bit for bit: (a - b)^2 = (b - a)^2 and a * b = b * a exactly)
template <bool COSINE, int ELEM>
__device__ __forceinline__ float row_distance(const unsigned char* a, const unsigned char* b, int dim, int j, int simd_width) {
    if (ELEM == 0) {
        QueryRegs<0> qr;
        if (simd_width != 16)
            return half_warp_distance_w<COSINE>(reinterpret_cast<const float*>(a), reinterpret_cast<const float*>(b), dim, j,
                                                simd_width);
        return half_warp_distance<0, COSINE>(reinterpret_cast<const float*>(a), qr, reinterpret_cast<const float*>(b), dim, j);
    }
    return half_warp_distance_elem_w<COSINE, ELEM>(a, b, dim, j, simd_width);
}

// RelativeNeighborhoodGraph::InsertNeighbors (RelativeNeighborhoodGraph.h:40-82) as RefineNode(updateNeighbors = true) runs
// it (NeighborhoodGraph.h:549-559): for every item of the added node's refine-search list, in list order until the first
// VID < 0 and skipping the node itself, insert the node into the item's row.  The items' rows are distinct and no call
// reads another item's row, so one warp per item computes exactly the sequential loop.  Per row: walk the slots (the last
// one excluded when it holds a duplicate back-pointer); the first slot that is empty, or farther from the row's owner than
// the node (ties: the smaller id first), takes the node and the displaced entries shift right while each is no farther
// from the owner than from the node; a slot whose entry is closer to the node than the node is to the owner ends the walk.
// The two distances of a step are computed at once, one per half-warp.
template <bool COSINE, int ELEM>
__global__ void __launch_bounds__(128) insert_neighbors_kernel(const unsigned char* __restrict__ vectors,
                                                               unsigned long long row_stride_bytes, int dim, int node,
                                                               const int* __restrict__ res_ids,
                                                               const float* __restrict__ res_dists, int num_results,
                                                               int* __restrict__ graph, int degree, int simd_width) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = lane & 15, half = lane >> 4;
    const int w = blockIdx.x * (blockDim.x >> 5) + warp;
    if (w >= num_results) return;
    // RefineNode stops at the first VID < 0
    for (int t0 = 0; t0 <= w; t0 += 32) {
        const int t = t0 + lane;
        if (__any_sync(kFull, t <= w && res_ids[t] < 0)) return;
    }
    const int target = res_ids[w];
    if (target == node) return;
    const float insert_dist = res_dists[w];
    int* row = graph + (size_t)target * degree;
    const unsigned char* node_vec = vectors + (size_t)target * row_stride_bytes;   // the row's owner
    const unsigned char* insert_vec = vectors + (size_t)node * row_stride_bytes;   // the node being added
    const int check = (row[degree - 1] < -1) ? degree - 1 : degree;
    for (int k = 0; k < check; ++k) {
        int tmp = row[k];
        __syncwarp();
        if (tmp < 0) {
            if (lane == 0) row[k] = node;
            return;
        }
        const unsigned char* tmp_vec = vectors + (size_t)tmp * row_stride_bytes;
        // half 0: d(tmp, owner); half 1: d(tmp, inserted)
        float d = row_distance<COSINE, ELEM>(tmp_vec, half ? insert_vec : node_vec, dim, j, simd_width);
        float d_owner = __shfl_sync(kFull, d, 0), d_ins = __shfl_sync(kFull, d, 16);
        if (d_owner > insert_dist || (insert_dist == d_owner && node < tmp)) {
            if (lane == 0) row[k] = node;
            __syncwarp();
            while (++k < check && d_owner <= d_ins) {
                const int next = row[k];
                __syncwarp();
                if (lane == 0) row[k] = tmp;
                __syncwarp();
                tmp = next;
                if (tmp < 0) return;
                tmp_vec = vectors + (size_t)tmp * row_stride_bytes;
                d = row_distance<COSINE, ELEM>(tmp_vec, half ? insert_vec : node_vec, dim, j, simd_width);
                d_owner = __shfl_sync(kFull, d, 0);
                d_ins = __shfl_sync(kFull, d, 16);
            }
            return;
        } else if (d_ins < insert_dist) {
            return;
        }
    }
}

// ------------------------------------------------------------------------------------------
// NeighborhoodGraph::RebuildGraph (NeighborhoodGraph.h:404-456): EnableRebuild's in-degree repair.  Rows hold 2 x ns
// candidates; the first ns/2 stay; the other ns - ns/2 slots are refilled from entries [ns/2, 2 ns): the ones whose target's
// in-degree is below ns/2 first, then the earliest others, in index order; the in-degree array follows every change.
// The reference runs its node loop under OpenMP with an unsynchronised in-degree array, so only its one-thread order is a
// function of the input; that order is inherently sequential over the nodes (node i's choice depends on what nodes < i
// did), so ONE warp walks the nodes, lane-parallel inside a row.  Offline, default-off in the reference.
// Duplicate-group back-pointers (< -1, last slot) are not neighbours: read as -1 here, re-attached by the caller.
// ------------------------------------------------------------------------------------------
__global__ void indegree_count_kernel(const int* __restrict__ graph, long long n, int stride, int ns, int* __restrict__ indegree) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * ns) return;
    const int v = graph[(t / ns) * stride + (t % ns)];
    if (v >= 0) atomicAdd(&indegree[v], 1);
}

constexpr int kRebuildMaxChunks = 48;  // (2 ns - ns/2) / 32 chunks: ns <= 1024

__global__ void __launch_bounds__(32) rebuild_graph_kernel(const int* __restrict__ old_graph, int n, int stride, int ns,
                                                           int* indegree, int* __restrict__ new_graph) {
    __shared__ unsigned lowmask[kRebuildMaxChunks], validmask[kRebuildMaxChunks];
    const int lane = threadIdx.x;
    const unsigned lt = (1u << lane) - 1u;
    const int start = ns / 2, thr = ns / 2, need = ns - start, span = 2 * ns - start;
    const int chunks = (span + 31) / 32;
    for (int i = 0; i < n; ++i) {
        const int* row = old_graph + (size_t)i * stride;
        int* out = new_graph + (size_t)i * ns;
        for (int j = lane; j < start; j += 32) {
            const int v = row[j];
            out[j] = v < -1 ? -1 : v;
        }
        // which candidates point at a node with a low in-degree (as it is after nodes 0 .. i-1)
        int c1 = 0;
        for (int ch = 0; ch < chunks; ++ch) {
            const int c = ch * 32 + lane;
            const bool in = c < span;
            int v = in ? row[start + c] : -1;
            if (v < -1) v = -1;
            const bool low = in && v >= 0 && __ldcg(&indegree[v]) < thr;
            const unsigned lm = __ballot_sync(kFull, low), vm = __ballot_sync(kFull, in);
            if (lane == 0) {
                lowmask[ch] = lm;
                validmask[ch] = vm;
            }
            c1 += __popc(lm);
        }
        __syncwarp();
        // the reserved set in index order: the low ones (the first `need` of them), topped up with the earliest others
        const bool enough = c1 >= need;
        int remaining = enough ? need : need - c1;  // how many of the rationed class may still be taken
        int placed = 0;
        for (int ch = 0; ch < chunks; ++ch) {
            const unsigned lm = lowmask[ch], vm = validmask[ch];
            const unsigned rationed = enough ? lm : (vm & ~lm);
            const int take = min(__popc(rationed), remaining);
            const bool rat_sel = ((rationed >> lane) & 1u) && (__popc(rationed & lt) < take);
            const bool sel = enough ? rat_sel : (((lm >> lane) & 1u) || rat_sel);
            const unsigned sm = __ballot_sync(kFull, sel);
            remaining -= take;
            const int c = ch * 32 + lane;
            int v = (c < span) ? row[start + c] : -1;
            if (v < -1) v = -1;
            if (sel) {
                out[start + placed + __popc(sm & lt)] = v;
                if (v >= 0) atomicAdd(&indegree[v], 1);
            }
            placed += __popc(sm);
            // the entries this pass overwrites, [start, ns), give their in-degree back
            if (c < ns - start && v >= 0) atomicSub(&indegree[v], 1);
        }
        __threadfence();  // node i + 1 reads the in-degrees this node wrote
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------
// PQ / OPQ quantizer kernels (query side + tables; PQQuantizer.h:138-180, :333-348, OPQQuantizer.h:96-121)
// ------------------------------------------------------------------------------------------

// PQQuantizer::InitializeDistanceTables (PQQuantizer.h:333-348): sdc[i][j][k] = L2(codebook[i][j], codebook[i][k])
__global__ void sdc_table_kernel(const float* __restrict__ codebooks, int m, int ks, int dsub, float* __restrict__ sdc) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)m * ks * ks;
    if (t >= total) return;
    const int k = (int)(t % ks);
    const int j = (int)((t / ks) % ks);
    const int i = (int)(t / ((long long)ks * ks));
    const float* base = codebooks + (size_t)i * ks * dsub;
    sdc[t] = exact_dist_thread<false>(base + (size_t)j * dsub, base + (size_t)k * dsub, dsub);
}

// IQuantizer::QuantizeVector(raw, codes, ADC=false) for a batch: one CTA per raw vector.
//   OPQ: rot[i] = m_base - m_fdot(vec, OPQMatrix_T row i) with m_base = 1 and m_fdot = float cosine distance
//        (OPQQuantizer.h:96-121, :198-206); PQ: rot = vec.
//   then per sub-vector the first codeword with the strictly smallest L2 distance (PQQuantizer.h:158-179).
// raw_type: 0 int8, 1 uint8, 2 int16, 3 float (the quantizer's reconstruct type).
__global__ void pq_quantize_kernel(const unsigned char* __restrict__ raw, int raw_type, long long raw_stride_bytes,
                                   int nvec, const float* __restrict__ codebooks, const float* __restrict__ rotation_t,
                                   int m, int ks, int dsub, unsigned char* __restrict__ codes,
                                   float* __restrict__ rotated_out) {
    extern __shared__ float qsm[];  // vec[dim] | rot[dim]
    const int dim = m * dsub;
    float* vec = qsm;
    float* rot = qsm + dim;
    const int v = blockIdx.x;
    if (v >= nvec) return;
    const unsigned char* src = raw + (size_t)v * raw_stride_bytes;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float f;
        switch (raw_type) {
        case 0: f = (float)reinterpret_cast<const signed char*>(src)[i]; break;
        case 1: f = (float)src[i]; break;
        case 2: f = (float)reinterpret_cast<const short*>(src)[i]; break;
        default: f = reinterpret_cast<const float*>(src)[i]; break;
        }
        vec[i] = f;
    }
    __syncthreads();
    const float* q = vec;
    if (rotation_t != nullptr) {
        for (int i = threadIdx.x; i < dim; i += blockDim.x)
            rot[i] = __fsub_rn(1.0f, exact_dist_thread<true>(vec, rotation_t + (size_t)i * dim, dim));
        __syncthreads();
        q = rot;
    }
    if (rotated_out != nullptr) {  // ADC mode: the search kernel builds the distance table from the rotated vector
        for (int i = threadIdx.x; i < dim; i += blockDim.x) rotated_out[(size_t)v * dim + i] = q[i];
        return;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    for (int i = warp; i < m; i += nwarps) {
        float best = INFINITY;
        int bestj = 0x7fffffff;
        for (int j = lane; j < ks; j += 32) {
            const float d = exact_dist_thread<false>(q + (size_t)i * dsub, codebooks + ((size_t)i * ks + j) * dsub, dsub);
            if (d < best) {  // increasing j per lane: strict '<' keeps the first minimum
                best = d;
                bestj = j;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(kFull, best, o);
            const int oj = __shfl_xor_sync(kFull, bestj, o);
            if (ob < best || (ob == best && oj < bestj)) {
                best = ob;
                bestj = oj;
            }
        }
        if (lane == 0) codes[(size_t)v * m + i] = (unsigned char)bestj;
    }
}

// IQuantizer::ReconstructVector for a batch of code rows: one CTA per row (NeighborhoodGraph::RefineNode on a quantized
// index reconstructs the node's row and lets SetTarget quantize the reconstruction again, NeighborhoodGraph.h:538-543).
//   PQQuantizer<float> (PQQuantizer.h:196-205): the codewords, copied.
//   OPQQuantizer<T> (OPQQuantizer.h:124-131): out[i] = (T)(m_base - m_fdot(pre, row i of m_OPQMatrix)), m_base = 1,
//   m_fdot = float cosine distance (:198-206); (T) = the C cast (truncation toward zero).
// raw_type: 0 int8, 1 uint8, 2 int16, 3 float.  out rows are packed (dim elements of the reconstruct type).
__global__ void pq_reconstruct_kernel(const unsigned char* __restrict__ codes, unsigned long long code_stride_bytes, int nvec,
                                      const float* __restrict__ codebooks, const float* __restrict__ rotation, int m,
                                      int ks, int dsub, int raw_type, unsigned char* __restrict__ out) {
    extern __shared__ float qsm[];  // pre[dim]
    const int dim = m * dsub;
    const int v = blockIdx.x;
    if (v >= nvec) return;
    const unsigned char* code = codes + (size_t)v * code_stride_bytes;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        const int sv = i / dsub, e = i - sv * dsub;
        qsm[i] = codebooks[((size_t)sv * ks + code[sv]) * dsub + e];
    }
    __syncthreads();
    const size_t esize = (raw_type == 3) ? 4 : (raw_type == 2 ? 2 : 1);
    unsigned char* dst = out + (size_t)v * dim * esize;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float f = qsm[i];
        if (rotation != nullptr) f = __fsub_rn(1.0f, exact_dist_thread<true>(qsm, rotation + (size_t)i * dim, dim));
        switch (raw_type) {
        case 0: reinterpret_cast<signed char*>(dst)[i] = (signed char)(__float2int_rz(f) & 0xff); break;
        case 1: dst[i] = (unsigned char)(__float2int_rz(f) & 0xff); break;
        case 2: reinterpret_cast<short*>(dst)[i] = (short)(__float2int_rz(f) & 0xffff); break;
        default: reinterpret_cast<float*>(dst)[i] = f; break;
        }
    }
}

// RebuildNeighbors on a quantized index: ComputeDistance(kept row, candidate row) is the quantizer's L2Distance on two
// code rows -- the SDC table sum in sub-vector order with one float accumulator (PQQuantizer.h:120-127).  One warp per
// node; lane k tests the candidate against kept neighbour k (32 kept rows per pass), any rejection drops it -- the
// reference's loop with its early exit is the same predicate.
__global__ void __launch_bounds__(128) rebuild_neighbors_pq_kernel(const unsigned char* __restrict__ codes,
                                                                   unsigned long long row_stride_bytes, int m, int ks,
                                                                   const float* __restrict__ sdc, int first_node,
                                                                   int num_nodes, const int* __restrict__ res_ids,
                                                                   const float* __restrict__ res_dists, int num_results,
                                                                   int neighborhood, float rng_factor,
                                                                   int* __restrict__ out_graph) {
    extern __shared__ int kept_sm[];  // neighborhood ints per warp
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    if (w >= num_nodes) return;
    int* kept = kept_sm + warp * neighborhood;
    const int node = first_node + (int)w;
    const int* ids = res_ids + (size_t)w * num_results;
    const float* ds = res_dists + (size_t)w * num_results;
    int count = 0;
    for (int r = 0; r < num_results && count < neighborhood; ++r) {
        const int vid = ids[r];
        if (vid < 0) break;
        if (vid == node) continue;
        const float dist = ds[r];
        const unsigned char* cand = codes + (size_t)vid * row_stride_bytes;
        bool good = true;
        for (int k0 = 0; k0 < count && good; k0 += 32) {
            bool reject = false;
            if (k0 + lane < count) {
                const unsigned char* row = codes + (size_t)kept[k0 + lane] * row_stride_bytes;
                float acc = 0.0f;
                for (int i = 0; i < m; ++i)
                    acc = __fadd_rn(acc, __ldg(sdc + ((size_t)i * ks + row[i]) * ks + cand[i]));
                reject = __fmul_rn(rng_factor, acc) < dist;
            }
            if (__any_sync(kFull, reject)) good = false;
        }
        if (good) {
            if (lane == 0) kept[count] = vid;
            ++count;
            __syncwarp();
        }
    }
    __syncwarp();
    for (int t = lane; t < neighborhood; t += 32) out_graph[(size_t)w * neighborhood + t] = (t < count) ? kept[t] : -1;
}

// ------------------------------------------------------------------------------------------
// k-way merge of per-shard top-k lists (QueryResultSet.h:17-26 comparator): one thread per query
// ------------------------------------------------------------------------------------------
__global__ void merge_topk_kernel(const int* __restrict__ ids, const float* __restrict__ dists, int num_lists,
                                  int nq, int k, int* __restrict__ out_ids, float* __restrict__ out_dists) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    // every list is ascending; keep one cursor per list (num_lists <= 16)
    int cur[16];
    for (int l = 0; l < num_lists; ++l) cur[l] = 0;
    for (int o = 0; o < k; ++o) {
        int bl = -1, bid = -1;
        float bd = 0.0f;
        for (int l = 0; l < num_lists; ++l) {
            if (cur[l] >= k) continue;
            const size_t at = ((size_t)l * nq + q) * k + cur[l];
            const int id = ids[at];
            const float d = dists[at];
            if (id < 0) {  // unfilled tail of this list
                cur[l] = k;
                continue;
            }
            if (bl < 0 || d < bd || (d == bd && id < bid)) {
                bl = l;
                bd = d;
                bid = id;
            }
        }
        if (bl < 0) {
            out_ids[(size_t)q * k + o] = -1;
            out_dists[(size_t)q * k + o] = SPTAG_B200_MAXDIST;
        } else {
            out_ids[(size_t)q * k + o] = bid;
            out_dists[(size_t)q * k + o] = bd;
            cur[bl]++;
        }
    }
}

// Same merge reading every shard's list where the shard's search kernel left it: `lists.ids[l]` / `lists.dists[l]` are
// [nq x k] arrays that may live in ANOTHER GPU's HBM (peer access over NVLink): the gather and the merge are one kernel,
// there is no staging copy and no collective call (sptag_b200_group_search).
struct ShardLists {
    const int* ids[16];
    const float* dists[16];
};
__global__ void merge_topk_peer_kernel(const ShardLists lists, int num_lists, int nq, int k, int* __restrict__ out_ids,
                                       float* __restrict__ out_dists) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    int cur[16];
    for (int l = 0; l < num_lists; ++l) cur[l] = 0;
    for (int o = 0; o < k; ++o) {
        int bl = -1, bid = -1;
        float bd = 0.0f;
        for (int l = 0; l < num_lists; ++l) {
            if (cur[l] >= k) continue;
            const size_t at = (size_t)q * k + cur[l];
            const int id = lists.ids[l][at];
            const float d = lists.dists[l][at];
            if (id < 0) {  // unfilled tail of this list
                cur[l] = k;
                continue;
            }
            if (bl < 0 || d < bd || (d == bd && id < bid)) {
                bl = l;
                bd = d;
                bid = id;
            }
        }
        if (bl < 0) {
            out_ids[(size_t)q * k + o] = -1;
            out_dists[(size_t)q * k + o] = SPTAG_B200_MAXDIST;
        } else {
            out_ids[(size_t)q * k + o] = bid;
            out_dists[(size_t)q * k + o] = bd;
            cur[bl]++;
        }
    }
}

}  // namespace sptag_b200
