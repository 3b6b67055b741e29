// TEST INFRASTRUCTURE.  Builds and searches PQ/OPQ-quantized SPANN indexes with the unmodified reference, so that
// tests/golden/make_golden_spann_pq.py can record what SPANN::Index<std::uint8_t>::SearchIndex returns on them.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage:
//   spann_pq_ref build <folder> <quantizer file> <rearrange 0/1> <n> <M> <codes file> <SSDIndexFileNum> [<threads>]
//       IndexBuilder's route for a quantized index (IndexBuilder/main.cpp:51-57, :107): a SPANN index over UInt8 code
//       rows, LoadQuantizer(file) (the quantizer goes to the head as well, SPANNIndex.cpp:39-56), then BuildIndex on the
//       n x M codes (VectorIndex.cpp:437-439) with the recipe of tests/cpp/spann_ref.cpp (L2, Ratio 0.1, ReplicaCount 4,
//       ExcludeHead, EnablePostingListRearrange as given), then SaveIndex(folder).  [Base] QuantizerFilePath names the
//       head's copy of the quantizer (SPANNIndex.cpp:874): quantizer.bin.  One thread by default.
//   spann_pq_ref search <folder> <queries file> <nq> <K> <adc 0/1> <out prefix> [<threads>]
//       VectorIndex::LoadIndex(folder), SetQuantizerADC(adc) on it (one quantizer for the head and the postings,
//       VectorIndex.h:136-138), then per RAW query (ReconstructDim values of the quantizer's reconstruct type)
//         <out>.head_ids / .head_dists  [nq x W] the head index's SearchIndex at W = max(K, SearchInternalResultNum),
//                                       as SPANN::Index::SearchIndex runs it (SPANNIndex.cpp:197-203), head-local ids
//         <out>.ids / .dists            [nq x K] SPANN::Index::SearchIndex(QueryResult&) (SPANNIndex.cpp:193-250)
//       threads > 1 searches the queries in parallel (tools/spann_pq_bench.py); <out>.ms gets the wall time of that loop.
// Files are raw row-major arrays (ids: int32).  Exit code 0 = every call succeeded.
#include <omp.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/Common/IQuantizer.h"
#include "inc/Core/Common/QueryResultSet.h"
#include "inc/Core/SPANN/Index.h"
#include "inc/Core/VectorIndex.h"
#include "inc/Helper/Logging.h"

using namespace SPTAG;

class QuietLogger : public Helper::Logger {
public:
    void Logging(const char*, Helper::LogLevel level, const char*, int, const char*, const char* format, ...) override {
        if (level < Helper::LogLevel::LL_Error) return;
        va_list args;
        va_start(args, format);
        std::vfprintf(stderr, format, args);
        va_end(args);
    }
};

static bool read_all(const std::string& path, std::vector<char>& out, size_t bytes) {
    out.resize(bytes);
    FILE* f = std::fopen(path.c_str(), "rb");
    if (!f) return false;
    const bool ok = std::fread(out.data(), 1, bytes, f) == bytes;
    std::fclose(f);
    return ok;
}

static bool write_all(const std::string& path, const void* p, size_t bytes) {
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = std::fwrite(p, 1, bytes, f) == bytes;
    std::fclose(f);
    return ok;
}

static int build(int argc, char** argv) {
    if (argc < 9) return 100;
    const std::string folder = argv[2], qfile = argv[3], rearrange = argv[4];
    const SizeType n = std::atoi(argv[5]);
    const DimensionType m = std::atoi(argv[6]);
    const std::string file_num = argv[8], threads = argc > 9 ? argv[9] : "1";
    const size_t bytes = (size_t)n * m;
    std::vector<char> data;
    if (!read_all(argv[7], data, bytes)) return 101;
    std::shared_ptr<VectorIndex> idx = VectorIndex::CreateInstance(IndexAlgoType::SPANN, VectorValueType::UInt8);
    if (!idx) return 102;
    if (idx->LoadQuantizer(qfile) != ErrorCode::Success || !idx->m_pQuantizer) return 105;
    if ((DimensionType)idx->m_pQuantizer->GetNumSubvectors() != m) return 106;
    idx->SetParameter("IndexAlgoType", "BKT", "Base");
    idx->SetParameter("IndexDirectory", folder.c_str(), "Base");  // the build writes its intermediate files there
    idx->SetParameter("DistCalcMethod", "L2", "Base");
    idx->SetParameter("QuantizerFilePath", "quantizer.bin", "Base");
    idx->SetParameter("isExecute", "true", "SelectHead");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "SelectHead");
    idx->SetParameter("Ratio", "0.1", "SelectHead");
    idx->SetParameter("isExecute", "true", "BuildHead");
    idx->SetParameter("RefineIterations", "3", "BuildHead");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "BuildHead");
    idx->SetParameter("isExecute", "true", "BuildSSDIndex");
    idx->SetParameter("BuildSsdIndex", "true", "BuildSSDIndex");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "BuildSSDIndex");
    idx->SetParameter("ReplicaCount", "4", "BuildSSDIndex");
    idx->SetParameter("SSDIndexFileNum", file_num.c_str(), "Base");
    idx->SetParameter("ExcludeHead", "true", "BuildSSDIndex");
    idx->SetParameter("PostingPageLimit", "12", "BuildSSDIndex");
    idx->SetParameter("SearchPostingPageLimit", "12", "BuildSSDIndex");
    idx->SetParameter("InternalResultNum", "64", "BuildSSDIndex");
    idx->SetParameter("SearchInternalResultNum", "64", "BuildSSDIndex");
    idx->SetParameter("EnablePostingListRearrange", rearrange == "1" ? "true" : "false", "BuildSSDIndex");
    ByteArray arr = ByteArray::Alloc(bytes);
    std::memcpy(arr.Data(), data.data(), bytes);
    std::shared_ptr<VectorSet> vec(new BasicVectorSet(arr, VectorValueType::UInt8, m, n));
    std::shared_ptr<MetadataSet> meta;
    if (idx->BuildIndex(vec, meta) != ErrorCode::Success) return 103;
    return idx->SaveIndex(folder) == ErrorCode::Success ? 0 : 104;
}

static int search(int argc, char** argv) {
    if (argc < 8) return 100;
    std::shared_ptr<VectorIndex> index;
    if (VectorIndex::LoadIndex(argv[2], index) != ErrorCode::Success || !index) return 110;
    auto* spann = dynamic_cast<SPANN::Index<std::uint8_t>*>(index.get());
    if (!spann || !index->m_pQuantizer) return 111;
    const int nq = std::atoi(argv[4]), k = std::atoi(argv[5]), adc = std::atoi(argv[6]);
    const std::string out = argv[7];
    const int threads = argc > 8 ? std::atoi(argv[8]) : 1;
    index->SetQuantizerADC(adc != 0);
    const size_t qbytes = index->m_pQuantizer->ReconstructSize();
    std::vector<char> qbuf;
    if (!read_all(argv[3], qbuf, (size_t)nq * qbytes)) return 101;
    const int internal = spann->GetOptions()->m_searchInternalResultNum;
    const int w = k >= internal ? k : internal;
    std::shared_ptr<VectorIndex> head = spann->GetMemoryIndex();
    std::vector<int> ids((size_t)nq * k), hids((size_t)nq * w);
    std::vector<float> dists((size_t)nq * k), hdists((size_t)nq * w);
    int bad = 0;
    if (threads <= 1) {
        for (int i = 0; i < nq; ++i) {
            COMMON::QueryResultSet<std::uint8_t> hr((const std::uint8_t*)(qbuf.data() + i * qbytes), w);
            head->SearchIndex(hr);
            for (int j = 0; j < w; ++j) {
                hids[(size_t)i * w + j] = hr.GetResult(j)->VID;
                hdists[(size_t)i * w + j] = hr.GetResult(j)->Dist;
            }
        }
    }
    omp_set_num_threads(threads > 1 ? threads : 1);
    const auto t0 = std::chrono::steady_clock::now();
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : bad)
    for (int i = 0; i < nq; ++i) {
        QueryResult r(qbuf.data() + i * qbytes, k, false);
        if (index->SearchIndex(r) != ErrorCode::Success) ++bad;
        for (int j = 0; j < k; ++j) {
            ids[(size_t)i * k + j] = r.GetResult(j)->VID;
            dists[(size_t)i * k + j] = r.GetResult(j)->Dist;
        }
    }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (bad) return 112;
    bool ok = write_all(out + ".ids", ids.data(), ids.size() * 4) && write_all(out + ".dists", dists.data(), dists.size() * 4);
    if (threads <= 1)
        ok = ok && write_all(out + ".head_ids", hids.data(), hids.size() * 4) &&
             write_all(out + ".head_dists", hdists.data(), hdists.size() * 4);
    ok = ok && write_all(out + ".ms", &ms, sizeof(ms));
    return ok ? 0 : 113;
}

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
    if (argc < 2) return 100;
    const std::string op = argv[1];
    if (op == "build") return build(argc, argv);
    if (op == "search") return search(argc, argv);
    return 100;
}
