// The gather path of posting lists in pinned host memory (PostingGather, spann_scan.h): which lists a round's queries
// read, their union and stage offsets, and the copy of their searched prefixes from mapped host memory into the HBM
// stage that the unchanged scan and posting-step kernels then read; with an HBM cache of lists, the union of the uncached
// ones only and the view's offsets into the cache and the stage, and the counts that rank lists for the cache.
#include "spann_device.cuh"
#include "spann_scan.h"

#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>

namespace sptag_b200 {
namespace {

// choose_postings for every query of p, one warp per query: its head results copied to shared memory as the scan
// copies them (the rule translates them in place), lane 0 chooses
__global__ void __launch_bounds__(32) spann_choose_kernel(const SpannScanParams p, int* chosen, int* nchosen, int stride) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* rd = reinterpret_cast<float*>(smem);
    int* rv = reinterpret_cast<int*>(rd + p.w);
    for (int q = blockIdx.x; q < p.nq; q += gridDim.x) {
        for (int i = threadIdx.x; i < p.w; i += 32) {
            rv[i] = p.head_ids[(size_t)q * p.w + i];
            rd[i] = p.head_dists[(size_t)q * p.w + i];
        }
        __syncwarp();
        if (threadIdx.x == 0) {
            int np = 0;
            long long total = 0;
            choose_postings(p, rd, rv, chosen + (size_t)q * stride, np, total);
            nchosen[q] = np;
        }
        __syncwarp();
    }
}

// What the posting step reads for the queries li in [b, e) of its launch: load_postings when the query loads the head's
// latest batch (it then reads nothing else), else the rest of its lists
__global__ void spann_iter_chosen_kernel(const SpannIterParams p, int b, int e, int* chosen, int* nchosen,
                                         unsigned int* sub) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) sub[0] = (unsigned)(e - b);
    const int li = b + i;
    if (li >= e) return;
    const int q = p.list ? (int)p.list[kIterListHeader + li] : li;
    sub[kIterListHeader + i] = (unsigned)q;
    int* out = chosen + (size_t)i * p.hb;
    const SpannIterState st = p.st[q];
    if (st.load) {
        nchosen[i] = load_postings(p, q, out);
        return;
    }
    const int* posts = p.posts + (size_t)q * p.hb;
    for (int j = st.pi; j < st.np; ++j) out[j - st.pi] = posts[j];
    nchosen[i] = max(st.np - st.pi, 0);
}

// With a cache (CACHED), only the lists it does not hold join the union
template <bool CACHED>
__global__ void spann_mark_kernel(const int* chosen, const int* nchosen, int stride, int n, const long long* resident,
                                  unsigned char* flags) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < (long long)n * stride;
         t += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(t / stride), j = (int)(t % stride);
        if (j < nchosen[q] && (!CACHED || resident[chosen[t]] < 0)) flags[chosen[t]] = 1;
    }
}

// counts[l] += the items that chose list l
__global__ void spann_count_kernel(const int* chosen, const int* nchosen, int stride, int n, int* counts) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < (long long)n * stride;
         t += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(t / stride), j = (int)(t % stride);
        if (j < nchosen[q]) atomicAdd(&counts[chosen[t]], 1);
    }
}

// The view's offsets with a cache: a cached list's first element in the pool, a union list's in this set's stage
__global__ void spann_view_off_kernel(const PostingGather g) {
    for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < g.num_lists; l += gridDim.x * blockDim.x) {
        const long long r = g.resident[l];
        g.view_off[l] = r >= 0 ? r : g.stage_base + g.stage_off[l];
    }
}

__global__ void spann_union_len_kernel(const PostingGather g) {
    for (int l = blockIdx.x * blockDim.x + threadIdx.x; l <= g.num_lists; l += gridDim.x * blockDim.x)
        g.len[l] = l < g.num_lists && g.flags[l] ? searched_count(g.host, l) : 0;
}

// One CTA per union list at a time: its rows as 16-byte words (row_stride is a multiple of 16), kUnroll loads in flight
// per thread before their stores, then its ids.  PEERS: a list g.peers.first places in a peer's pool is read from
// there (HBM of the same device, or over NVLink), the others from mapped host memory.
constexpr int kGatherThreads = 256;
constexpr int kUnroll = 8;
template <bool PEERS>
__global__ void __launch_bounds__(kGatherThreads) spann_gather_kernel(const PostingGather g) {
    const int n = *g.nlists;
    const long long words_per_row = (long long)(g.host.row_stride / 16);
    for (int u = blockIdx.x; u < n; u += gridDim.x) {
        const int l = g.lists[u];
        long long from = g.host.off[l];
        const long long to = g.stage_off[l], c = g.len[l];
        const unsigned char* rows = g.host.rows;
        const int* ids = g.host.ids;
        if (PEERS) {
            const long long first = g.peers.first[l];
            if (first >= 0) {
                const int o = g.peers.owner[l];
                from = first;
                rows = g.peers.rows[o];
                ids = g.peers.ids[o];
                if (threadIdx.x == 0) atomicAdd(g.peers.elems, (unsigned long long)c);
            }
        }
        const uint4* src = reinterpret_cast<const uint4*>(rows) + from * words_per_row;
        uint4* dst = reinterpret_cast<uint4*>(g.stage_rows) + to * words_per_row;
        const long long words = c * words_per_row;
        for (long long w0 = threadIdx.x; w0 < words; w0 += (long long)kUnroll * kGatherThreads) {
            uint4 v[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const long long w = w0 + (long long)j * kGatherThreads;
                if (w < words) v[j] = src[w];
            }
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const long long w = w0 + (long long)j * kGatherThreads;
                if (w < words) dst[w] = v[j];
            }
        }
        for (long long i = threadIdx.x; i < c; i += kGatherThreads) g.stage_ids[to + i] = ids[from + i];
    }
}

// The file placement's unpack: one CTA per list of a piece.  The list's raw bytes (16-byte aligned in the window) come
// into shared memory as aligned 16-byte words, a chunk of whole records at a time; each record is then cut out at its
// byte offset, which need not be a multiple of 4 (vis 21, 37, ...).
constexpr int kUnpackThreads = 256;
constexpr int kUnpackChunk = 32 << 10;  // shared bytes of one chunk, unless one record needs more
constexpr int kUnpackSlack = 32;        // readable bytes past a chunk: unpack_word reads up to 20 bytes past its offset

// Loads bytes [a, b) of the list at src into sm as the aligned 16-byte words that cover them; returns where byte a is
__device__ __forceinline__ int unpack_load(const uint4* src, long long a, long long b, uint4* sm) {
    const long long w0 = a >> 4;
    const int words = (int)(((b + 15) >> 4) - w0);  // at most a chunk's
    src += w0;
    for (int i = threadIdx.x; i < words; i += kUnpackThreads) sm[i] = src[i];
    return (int)(a & 15);
}

__device__ __forceinline__ unsigned unpack_u32(const unsigned char* sm, int o) {
    const unsigned* w = reinterpret_cast<const unsigned*>(sm + (o & ~3));
    return __funnelshift_r(w[0], w[1], (o & 3) * 8);
}

// The 16 bytes at offset o of sm, the bytes from `valid` on zeroed (a row's padding)
__device__ __forceinline__ uint4 unpack_word(const unsigned char* sm, int o, int valid) {
    const unsigned* w = reinterpret_cast<const unsigned*>(sm + (o & ~3));
    const int sh = (o & 3) * 8;
    unsigned v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned x = __funnelshift_r(w[k], w[k + 1], sh);
        const int keep = valid - 4 * k;
        v[k] = keep >= 4 ? x : keep <= 0 ? 0u : x & ((1u << (8 * keep)) - 1u);
    }
    return make_uint4(v[0], v[1], v[2], v[3]);
}

// n rows of row_bytes, row i at offset base + i * step of sm, to dst at wpr 16-byte words per row
__device__ __forceinline__ void unpack_rows(const unsigned char* sm, int base, int step, int n, int row_bytes, int wpr,
                                            uint4* dst) {
    for (int t = threadIdx.x; t < n * wpr; t += kUnpackThreads) {
        const int i = t / wpr, j = t - i * wpr, valid = row_bytes - 16 * j;
        dst[(long long)i * wpr + j] = valid > 0 ? unpack_word(sm, base + i * step + 16 * j, valid) : make_uint4(0, 0, 0, 0);
    }
}

template <bool REARRANGED>
__global__ void __launch_bounds__(kUnpackThreads) spann_file_unpack_kernel(const PostingGather g,
                                                                          const FilePieceList* table,
                                                                          const unsigned char* window, int chunk) {
    extern __shared__ __align__(16) unsigned char smem[];
    uint4* sm = reinterpret_cast<uint4*>(smem);
    const FilePieceList pl = table[blockIdx.x];
    const int l = pl.list;
    const long long len = g.len[l], to = g.stage_off[l];
    const int vis = g.host.vector_info_size, rb = vis - 4, wpr = (int)(g.host.row_stride / 16);
    const uint4* src = reinterpret_cast<const uint4*>(window + pl.window_off);
    uint4* rows = reinterpret_cast<uint4*>(g.stage_rows) + to * wpr;
    int* ids = g.stage_ids + to;
    if (!REARRANGED) {  // element i: [id | row] at i * vis
        const int per = (chunk - 16) / vis;
        for (long long e0 = 0; e0 < len; e0 += per) {
            const int n = (int)min((long long)per, len - e0);
            __syncthreads();  // the last chunk is consumed
            const int base = unpack_load(src, e0 * vis, (e0 + n) * vis, sm);
            __syncthreads();
            unpack_rows(smem, base + 4, vis, n, rb, wpr, rows + e0 * wpr);
            for (int i = threadIdx.x; i < n; i += kUnpackThreads) ids[e0 + i] = (int)unpack_u32(smem, base + i * vis);
        }
    } else {  // every row (rb bytes each), then every id, of the whole list (ExtraFullGraphSearcher.h:1186-1195)
        const long long cnt = g.host.cnt[l], per = (chunk - 16) / rb, per_id = (chunk - 16) / 4;
        for (long long e0 = 0; e0 < len; e0 += per) {
            const int n = (int)min(per, len - e0);
            __syncthreads();
            const int base = unpack_load(src, e0 * rb, (e0 + n) * rb, sm);
            __syncthreads();
            unpack_rows(smem, base, rb, n, rb, wpr, rows + e0 * wpr);
        }
        for (long long e0 = 0; e0 < len; e0 += per_id) {
            const int n = (int)min(per_id, len - e0);
            __syncthreads();
            const int base = unpack_load(src, rb * cnt + 4 * e0, rb * cnt + 4 * (e0 + n), sm);
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += kUnpackThreads) ids[e0 + i] = (int)unpack_u32(smem, base + 4 * i);
        }
    }
}

// The stage offsets (exclusive sum of g.len) and the compacted union (the flagged list numbers); with temp null, the
// scratch bytes the two need
cudaError_t union_cub(const PostingGather& g, void* temp, size_t& bytes, cudaStream_t stream) {
    const thrust::counting_iterator<int> list_numbers(0);
    if (!temp) {
        size_t scan = 0, select = 0;
        cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, scan, g.len, g.stage_off, g.num_lists + 1, stream);
        if (e == cudaSuccess)
            e = cub::DeviceSelect::Flagged(nullptr, select, list_numbers, g.flags, g.lists, g.nlists, g.num_lists, stream);
        bytes = std::max(scan, select);
        return e;
    }
    cudaError_t e = cub::DeviceScan::ExclusiveSum(temp, bytes, g.len, g.stage_off, g.num_lists + 1, stream);
    if (e == cudaSuccess)
        e = cub::DeviceSelect::Flagged(temp, bytes, list_numbers, g.flags, g.lists, g.nlists, g.num_lists, stream);
    return e;
}

}  // namespace

size_t spann_union_temp_bytes(int num_lists) {
    PostingGather g = {};
    g.num_lists = num_lists;
    size_t bytes = 0;
    return union_cub(g, nullptr, bytes, nullptr) == cudaSuccess ? bytes : 0;
}

cudaError_t launch_spann_choose(const SpannScanParams& p, int* chosen, int* nchosen, int stride, cudaStream_t stream) {
    // W <= 2048: at most 16 KB of head results
    spann_choose_kernel<<<std::min(p.nq, 65535), 32, (size_t)p.w * 8, stream>>>(p, chosen, nchosen, stride);
    return cudaGetLastError();
}

cudaError_t launch_spann_iter_chosen(const SpannIterParams& p, int b, int e, int* chosen, int* nchosen, unsigned int* sub,
                                     cudaStream_t stream) {
    const int n = std::max(e - b, 1);
    spann_iter_chosen_kernel<<<(n + 127) / 128, 128, 0, stream>>>(p, b, e, chosen, nchosen, sub);
    return cudaGetLastError();
}

cudaError_t launch_spann_union(const PostingGather& g, const int* chosen, const int* nchosen, int stride, int n,
                               cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(g.flags, 0, (size_t)g.num_lists, stream);
    if (e != cudaSuccess) return e;
    const long long marks = (long long)n * stride;
    if (marks > 0) {
        const int grid = (int)std::min<long long>((marks + 255) / 256, 4096);
        if (g.resident)
            spann_mark_kernel<true><<<grid, 256, 0, stream>>>(chosen, nchosen, stride, n, g.resident, g.flags);
        else
            spann_mark_kernel<false><<<grid, 256, 0, stream>>>(chosen, nchosen, stride, n, nullptr, g.flags);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    spann_union_len_kernel<<<std::min((g.num_lists + 256) / 256, 4096), 256, 0, stream>>>(g);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    size_t bytes = g.temp_bytes;
    if ((e = union_cub(g, g.temp, bytes, stream)) != cudaSuccess || !g.resident) return e;
    spann_view_off_kernel<<<std::min((g.num_lists + 255) / 256, 4096), 256, 0, stream>>>(g);
    return cudaGetLastError();
}

cudaError_t launch_spann_count(const int* chosen, const int* nchosen, int stride, int n, int* counts, cudaStream_t stream) {
    const long long marks = (long long)n * stride;
    if (marks > 0)
        spann_count_kernel<<<(int)std::min<long long>((marks + 255) / 256, 4096), 256, 0, stream>>>(chosen, nchosen, stride,
                                                                                                   n, counts);
    return cudaGetLastError();
}

cudaError_t launch_spann_gather(const PostingGather& g, int grid, cudaStream_t stream) {
    if (g.peers.first)
        spann_gather_kernel<true><<<grid, kGatherThreads, 0, stream>>>(g);
    else
        spann_gather_kernel<false><<<grid, kGatherThreads, 0, stream>>>(g);
    return cudaGetLastError();
}

cudaError_t launch_spann_file_unpack(const PostingGather& g, const FilePieceList* table, int n, const unsigned char* window,
                                     bool rearranged, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int record = rearranged ? g.host.vector_info_size - 4 : g.host.vector_info_size;
    const int chunk = std::max(kUnpackChunk, (record + 15) / 16 * 16 + 16);  // at least one record per chunk
    const size_t smem = (size_t)chunk + kUnpackSlack;
    auto kernel = rearranged ? spann_file_unpack_kernel<true> : spann_file_unpack_kernel<false>;
    if (smem > (48u << 10)) {  // records over 32 KB: the opt-in maximum, one value for every caller
        int dev = 0, optin = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e == cudaSuccess && smem > (size_t)optin) e = cudaErrorInvalidValue;
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
        if (e != cudaSuccess) return e;
    }
    kernel<<<n, kUnpackThreads, smem, stream>>>(g, table, window, chunk);
    return cudaGetLastError();
}

}  // namespace sptag_b200
