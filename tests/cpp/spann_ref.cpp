// TEST INFRASTRUCTURE.  Builds and searches SPANN indexes with the unmodified reference, so that
// tests/golden/make_golden_spann.py can record what SPANN::Index<T>::SearchIndex returns.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage:
//   spann_ref build <folder> <Float|Int8> <L2|Cosine> <rearrange 0/1> <n> <dim> <data file> <SSDIndexFileNum>
//                   <ExcludeHead 0/1> [<threads>]
//       the build recipe of tests/cpp/spann_head_dropin.cpp (Test/src/AlgoTest.cpp:23-42: SelectHead -> BuildHead ->
//       BuildSSDIndex) with Ratio 0.1 (lists long enough to truncate), ReplicaCount 4, EnablePostingListRearrange as given, then SaveIndex(folder).  One thread by
//       default, so that a rebuild writes the same files.
//   spann_ref search <folder> <queries file> <nq> <K> <out prefix> [<threads>]
//       VectorIndex::LoadIndex(folder) (every search parameter comes from the folder's indexloader.ini), then per query
//         <out>.head_ids / .head_dists  [nq x W] the head index's SearchIndex at W = max(K, SearchInternalResultNum),
//                                       as SPANN::Index::SearchIndex runs it (SPANNIndex.cpp:197-203), head-local ids
//         <out>.ids / .dists            [nq x K] SPANN::Index::SearchIndex(QueryResult&) (SPANNIndex.cpp:193-250)
//       threads > 1 searches the queries in parallel (tools/spann_bench.py); <out>.ms gets the wall time of that loop.
// Files are raw row-major arrays of the index's value type (ids: int32).  Exit code 0 = every call succeeded.
#include <omp.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

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
    if (argc < 11) return 100;
    const std::string folder = argv[2], vt = argv[3], metric = argv[4], rearrange = argv[5];
    const SizeType n = std::atoi(argv[6]);
    const DimensionType dim = std::atoi(argv[7]);
    const std::string file_num = argv[9], exclude_head = argv[10], threads = argc > 11 ? argv[11] : "1";
    const VectorValueType type = vt == "Int8" ? VectorValueType::Int8 : VectorValueType::Float;
    const size_t bytes = (size_t)n * dim * (type == VectorValueType::Int8 ? 1 : 4);
    std::vector<char> data;
    if (!read_all(argv[8], data, bytes)) return 101;
    std::shared_ptr<VectorIndex> idx = VectorIndex::CreateInstance(IndexAlgoType::SPANN, type);
    if (!idx) return 102;
    idx->SetParameter("IndexAlgoType", "BKT", "Base");
    idx->SetParameter("IndexDirectory", folder.c_str(), "Base");  // the build writes its intermediate files there
    idx->SetParameter("DistCalcMethod", metric.c_str(), "Base");
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
    // ExcludeHead false puts the head vectors into posting lists too (and writes MaxSize into the translate map,
    // SPANNIndex.cpp:914-924)
    idx->SetParameter("ExcludeHead", exclude_head == "1" ? "true" : "false", "BuildSSDIndex");
    idx->SetParameter("PostingPageLimit", "12", "BuildSSDIndex");
    idx->SetParameter("SearchPostingPageLimit", "12", "BuildSSDIndex");
    idx->SetParameter("InternalResultNum", "64", "BuildSSDIndex");
    idx->SetParameter("SearchInternalResultNum", "64", "BuildSSDIndex");
    idx->SetParameter("EnablePostingListRearrange", rearrange == "1" ? "true" : "false", "BuildSSDIndex");
    ByteArray arr = ByteArray::Alloc(bytes);
    std::memcpy(arr.Data(), data.data(), bytes);
    std::shared_ptr<VectorSet> vec(new BasicVectorSet(arr, type, dim, n));
    std::shared_ptr<MetadataSet> meta;
    if (idx->BuildIndex(vec, meta) != ErrorCode::Success) return 103;
    return idx->SaveIndex(folder) == ErrorCode::Success ? 0 : 104;
}

template <typename T>
static int search_t(VectorIndex* index, const std::vector<char>& qbuf, int nq, int k, const std::string& out, int threads) {
    auto* spann = dynamic_cast<SPANN::Index<T>*>(index);
    if (!spann) return 111;
    const DimensionType dim = index->GetFeatureDim();
    const int internal = spann->GetOptions()->m_searchInternalResultNum;
    const int w = k >= internal ? k : internal;
    std::shared_ptr<VectorIndex> head = spann->GetMemoryIndex();
    const T* q = reinterpret_cast<const T*>(qbuf.data());
    std::vector<int> ids((size_t)nq * k), hids((size_t)nq * w);
    std::vector<float> dists((size_t)nq * k), hdists((size_t)nq * w);
    int bad = 0;
    if (threads <= 1) {
        for (int i = 0; i < nq; ++i) {
            COMMON::QueryResultSet<T> hr(q + (size_t)i * dim, w);
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
        QueryResult r(q + (size_t)i * dim, k, false);
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

static int search(int argc, char** argv) {
    if (argc < 7) return 100;
    std::shared_ptr<VectorIndex> index;
    if (VectorIndex::LoadIndex(argv[2], index) != ErrorCode::Success || !index) return 110;
    const int nq = std::atoi(argv[4]), k = std::atoi(argv[5]);
    const int threads = argc > 7 ? std::atoi(argv[7]) : 1;
    const bool i8 = index->GetVectorValueType() == VectorValueType::Int8;
    std::vector<char> qbuf;
    if (!read_all(argv[3], qbuf, (size_t)nq * index->GetFeatureDim() * (i8 ? 1 : 4))) return 101;
    return i8 ? search_t<std::int8_t>(index.get(), qbuf, nq, k, argv[6], threads)
              : search_t<float>(index.get(), qbuf, nq, k, argv[6], threads);
}

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
    if (argc < 2) return 100;
    const std::string op = argv[1];
    if (op == "build") return build(argc, argv);
    if (op == "search") return search(argc, argv);
    return 100;
}
