// SPANN posting scan on PQ/OPQ code rows (ExtraFullGraphSearcher<std::uint8_t>, SPANNIndex.cpp:93-99, :122-128): the
// body of spann_scan_body (spann_device.cuh) with the quantizer's distance, ComputeDistance(GetQuantizedTarget(), row)
// (ExtraFullGraphSearcher.h:120-130) = PQQuantizer::L2Distance (PQQuantizer.h:110-128):
//   SDC  sum_i sdc[(i*Ks + q_i)*Ks + y_i], q = the query's M codes
//   ADC  sum_i table[i*Ks + y_i], table = the query's M x Ks distances to the codewords (PQQuantizer.h:141-157)
// in sub-vector order with one fp32 accumulator, the sum compute_dists_pq does in the head search.  Lane r computes
// candidate r of the chunk.
#include "spann_device.cuh"
#include "spann_scan.h"

namespace sptag_b200 {
namespace {

struct PqDistance {
    const SpannPqScanParams& pp;
    unsigned* qoff;  // [m] the offsets of the query's table rows (shared memory)
    const float* tb;
    int lane;

    __device__ __forceinline__ void begin_query(const SpannScanParams&, int q) {
        if (pp.adc) {
            // the table the head search built for this query (search_kernel_defs.cuh), into this block's arena
            float* table = pp.adc_tables + (size_t)blockIdx.x * pp.m * pp.ks;
            const float* qrot = pp.qrot + (size_t)q * pp.m * pp.dsub;
            const int total = pp.m * pp.ks;
            for (int t = lane; t < total; t += 32) {
                const int i = t / pp.ks;
                table[t] = exact_dist_thread<false>(qrot + (size_t)i * pp.dsub, pp.codebooks + (size_t)t * pp.dsub, pp.dsub);
            }
            for (int i = lane; i < pp.m; i += 32) qoff[i] = (unsigned)(i * pp.ks);
            tb = table;
        } else {
            const unsigned char* qc = pp.qcodes + (size_t)q * pp.m;
            for (int i = lane; i < pp.m; i += 32) qoff[i] = (unsigned)((i * pp.ks + (int)qc[i]) * pp.ks);
            tb = pp.sdc;
        }
        __syncwarp();
    }

    __device__ __forceinline__ void chunk(const PostingLists pl, long long base, const int* cl, int cnt, float* cd) {
        if (lane >= cnt) return;
        const unsigned char* row = pl.rows + (size_t)(base + cl[lane]) * pl.row_stride;  // 16-byte aligned
        float acc = 0.0f;
        const int m4 = pp.m & ~3;
        int i = 0;
        for (; i < m4; i += 4) {
            const unsigned w = *reinterpret_cast<const unsigned*>(row + i);
            const float t0 = tb[qoff[i] + __byte_perm(w, 0u, 0x4440u)];
            const float t1 = tb[qoff[i + 1] + __byte_perm(w, 0u, 0x4441u)];
            const float t2 = tb[qoff[i + 2] + __byte_perm(w, 0u, 0x4442u)];
            const float t3 = tb[qoff[i + 3] + __byte_perm(w, 0u, 0x4443u)];
            acc = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(acc, t0), t1), t2), t3);
        }
        for (; i < pp.m; ++i) acc = __fadd_rn(acc, tb[qoff[i] + (unsigned)row[i]]);
        cd[lane] = acc;
    }
};

__global__ void __launch_bounds__(32) spann_pq_scan_kernel(const SpannPqScanParams pp) {
    extern __shared__ __align__(16) unsigned char smem[];
    PqDistance dist{pp, reinterpret_cast<unsigned*>(smem + spann_scan_smem(pp.s.w)), nullptr, (int)threadIdx.x};
    spann_scan_body(pp.s, smem, dist);
}

}  // namespace

size_t spann_pq_scan_smem(int w, int m) { return spann_scan_smem(w) + (size_t)m * 4; }

int spann_pq_scan_blocks_per_sm(int w, int m) {
    return warp_blocks_per_sm((const void*)spann_pq_scan_kernel, spann_pq_scan_smem(w, m));
}

cudaError_t launch_spann_pq_scan(const SpannPqScanParams& p, int grid, cudaStream_t stream, const void** kernel) {
    *kernel = (const void*)spann_pq_scan_kernel;
    return launch_warp_blocks(spann_pq_scan_kernel, p, grid, spann_pq_scan_smem(p.s.w, p.m), stream);
}

}  // namespace sptag_b200
