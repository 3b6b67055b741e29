// TEST INFRASTRUCTURE.  Builds, searches and iterates SPANN indexes of every element type (Float, Int8, UInt8, Int16) with
// the unmodified reference, so that tests/golden/make_golden_spann_elem.py can record what SPANN::Index<T> returns.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// The recipes and file formats are those of tests/cpp/spann_ref.cpp (build, search) and tests/cpp/spann_iter_ref.cpp
// (iterate), on one thread, with every buffer sized by the index's element size.
// usage:
//   spann_elem_ref build <folder> <Float|Int8|UInt8|Int16> <L2|Cosine> <rearrange 0/1> <n> <dim> <data file>
//                        <SSDIndexFileNum> <ExcludeHead 0/1>
//       SelectHead -> BuildHead -> BuildSSDIndex (Ratio 0.1, ReplicaCount 4, EnablePostingListRearrange as given), then
//       SaveIndex(folder)
//   spann_elem_ref search <folder> <queries file> <nq> <K> <out prefix>
//       <out>.head_ids / .head_dists [nq x W] the head index's SearchIndex at W = max(K, SearchInternalResultNum),
//       head-local ids; <out>.ids / .dists [nq x K] SPANN::Index::SearchIndex(QueryResult&)
//   spann_elem_ref <folder> <queries file> <nq> <out prefix> <b0,b1,...>
//       GetIterator and Next(b) for each b of the schedule: <out>.counts [calls x nq] int32, <out>.relaxed [calls x nq]
//       uint8, <out>.ids / .dists per call one [nq x b_c] block, the first resultNum results then (-1, MaxDist)
// Files are raw row-major arrays of the index's value type (ids: int32).  Exit code 0 = every call succeeded.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/Common/QueryResultSet.h"
#include "inc/Core/ResultIterator.h"
#include "inc/Core/SPANN/Index.h"
#include "inc/Core/SearchQuery.h"
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

static VectorValueType value_type(const std::string& vt) {
    if (vt == "Float") return VectorValueType::Float;
    if (vt == "Int8") return VectorValueType::Int8;
    if (vt == "UInt8") return VectorValueType::UInt8;
    if (vt == "Int16") return VectorValueType::Int16;
    return VectorValueType::Undefined;
}

static int build(int argc, char** argv) {
    if (argc < 11) return 100;
    const std::string folder = argv[2], metric = argv[4], rearrange = argv[5];
    const VectorValueType type = value_type(argv[3]);
    if (type == VectorValueType::Undefined) return 100;
    const SizeType n = std::atoi(argv[6]);
    const DimensionType dim = std::atoi(argv[7]);
    const std::string file_num = argv[9], exclude_head = argv[10];
    const size_t bytes = (size_t)n * dim * GetValueTypeSize(type);
    std::vector<char> data;
    if (!read_all(argv[8], data, bytes)) return 101;
    std::shared_ptr<VectorIndex> idx = VectorIndex::CreateInstance(IndexAlgoType::SPANN, type);
    if (!idx) return 102;
    idx->SetParameter("IndexAlgoType", "BKT", "Base");
    idx->SetParameter("IndexDirectory", folder.c_str(), "Base");  // the build writes its intermediate files there
    idx->SetParameter("DistCalcMethod", metric.c_str(), "Base");
    idx->SetParameter("isExecute", "true", "SelectHead");
    idx->SetParameter("NumberOfThreads", "1", "SelectHead");
    idx->SetParameter("Ratio", "0.1", "SelectHead");
    idx->SetParameter("isExecute", "true", "BuildHead");
    idx->SetParameter("RefineIterations", "3", "BuildHead");
    idx->SetParameter("NumberOfThreads", "1", "BuildHead");
    idx->SetParameter("isExecute", "true", "BuildSSDIndex");
    idx->SetParameter("BuildSsdIndex", "true", "BuildSSDIndex");
    idx->SetParameter("NumberOfThreads", "1", "BuildSSDIndex");
    idx->SetParameter("ReplicaCount", "4", "BuildSSDIndex");
    idx->SetParameter("SSDIndexFileNum", file_num.c_str(), "Base");
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
static int search_t(VectorIndex* index, const std::vector<char>& qbuf, int nq, int k, const std::string& out) {
    auto* spann = dynamic_cast<SPANN::Index<T>*>(index);
    if (!spann) return 111;
    const DimensionType dim = index->GetFeatureDim();
    const int internal = spann->GetOptions()->m_searchInternalResultNum;
    const int w = k >= internal ? k : internal;
    std::shared_ptr<VectorIndex> head = spann->GetMemoryIndex();
    const T* q = reinterpret_cast<const T*>(qbuf.data());
    std::vector<int> ids((size_t)nq * k), hids((size_t)nq * w);
    std::vector<float> dists((size_t)nq * k), hdists((size_t)nq * w);
    for (int i = 0; i < nq; ++i) {
        COMMON::QueryResultSet<T> hr(q + (size_t)i * dim, w);
        head->SearchIndex(hr);
        for (int j = 0; j < w; ++j) {
            hids[(size_t)i * w + j] = hr.GetResult(j)->VID;
            hdists[(size_t)i * w + j] = hr.GetResult(j)->Dist;
        }
    }
    for (int i = 0; i < nq; ++i) {
        QueryResult r(q + (size_t)i * dim, k, false);
        if (index->SearchIndex(r) != ErrorCode::Success) return 112;
        for (int j = 0; j < k; ++j) {
            ids[(size_t)i * k + j] = r.GetResult(j)->VID;
            dists[(size_t)i * k + j] = r.GetResult(j)->Dist;
        }
    }
    const bool ok = write_all(out + ".ids", ids.data(), ids.size() * 4) &&
                    write_all(out + ".dists", dists.data(), dists.size() * 4) &&
                    write_all(out + ".head_ids", hids.data(), hids.size() * 4) &&
                    write_all(out + ".head_dists", hdists.data(), hdists.size() * 4);
    return ok ? 0 : 113;
}

static int search(int argc, char** argv) {
    if (argc < 7) return 100;
    std::shared_ptr<VectorIndex> index;
    if (VectorIndex::LoadIndex(argv[2], index) != ErrorCode::Success || !index) return 110;
    const int nq = std::atoi(argv[4]), k = std::atoi(argv[5]);
    const VectorValueType type = index->GetVectorValueType();
    std::vector<char> qbuf;
    if (!read_all(argv[3], qbuf, (size_t)nq * index->GetFeatureDim() * GetValueTypeSize(type))) return 101;
    switch (type) {
        case VectorValueType::Float: return search_t<float>(index.get(), qbuf, nq, k, argv[6]);
        case VectorValueType::Int8: return search_t<std::int8_t>(index.get(), qbuf, nq, k, argv[6]);
        case VectorValueType::UInt8: return search_t<std::uint8_t>(index.get(), qbuf, nq, k, argv[6]);
        case VectorValueType::Int16: return search_t<std::int16_t>(index.get(), qbuf, nq, k, argv[6]);
        default: return 111;
    }
}

static int iterate(int argc, char** argv) {
    if (argc < 6) return 100;
    std::shared_ptr<VectorIndex> index;
    if (VectorIndex::LoadIndex(argv[1], index) != ErrorCode::Success || !index) return 110;
    const int nq = std::atoi(argv[3]);
    const std::string out = argv[4];
    std::vector<int> schedule;
    for (const char* c = argv[5]; *c;) {
        schedule.push_back(std::atoi(c));
        while (*c && *c != ',') ++c;
        if (*c == ',') ++c;
    }
    const size_t row = (size_t)index->GetFeatureDim() * GetValueTypeSize(index->GetVectorValueType());
    std::vector<char> qbuf;
    if (!read_all(argv[2], qbuf, (size_t)nq * row)) return 101;
    std::vector<size_t> at(schedule.size() + 1, 0);  // where call c's [nq x b_c] block starts
    for (size_t c = 0; c < schedule.size(); ++c) at[c + 1] = at[c] + (size_t)nq * schedule[c];
    std::vector<int> ids(at.back()), counts(schedule.size() * nq);
    std::vector<float> dists(at.back());
    std::vector<unsigned char> relaxed(schedule.size() * nq);
    for (int i = 0; i < nq; ++i) {
        std::shared_ptr<ResultIterator> it = index->GetIterator(qbuf.data() + (size_t)i * row);
        if (!it) return 112;
        for (size_t c = 0; c < schedule.size(); ++c) {
            const int b = schedule[c];
            std::shared_ptr<QueryResult> r = it->Next(b);
            const int num = r->GetResultNum();
            counts[c * nq + i] = num;
            relaxed[c * nq + i] = it->GetRelaxedMono() ? 1 : 0;
            for (int j = 0; j < b; ++j) {
                ids[at[c] + (size_t)i * b + j] = j < num ? r->GetResult(j)->VID : -1;
                dists[at[c] + (size_t)i * b + j] = j < num ? r->GetResult(j)->Dist : MaxDist;
            }
        }
        it->Close();
    }
    const bool ok = write_all(out + ".ids", ids.data(), ids.size() * 4) && write_all(out + ".dists", dists.data(), dists.size() * 4) &&
                    write_all(out + ".counts", counts.data(), counts.size() * 4) &&
                    write_all(out + ".relaxed", relaxed.data(), relaxed.size());
    return ok ? 0 : 113;
}

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
    if (argc < 2) return 100;
    const std::string op = argv[1];
    if (op == "build") return build(argc, argv);
    if (op == "search") return search(argc, argv);
    return iterate(argc, argv);
}
