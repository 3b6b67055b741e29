// vector_index_adapter.hpp -- C++ host-side mirror of the reference's search interface on top of the
// C ABI (include/sptag_b200.h).  Header-only; links only against libsptag_b200.so.
//
// It mirrors, for the search path only, the reference types a caller touches:
//   SPTAG::BasicResult    AnnService/inc/Core/SearchResult.h:65-78   (VID, Dist; Meta stays on the host side)
//   SPTAG::QueryResult    AnnService/inc/Core/SearchQuery.h:15-254   (target pointer, K results)
//   SPTAG::VectorIndex    AnnService/inc/Core/VectorIndex.h:41,103   (the two SearchIndex overloads,
//                         LoadIndex, SetParameter/GetParameter, GetNumSamples/GetFeatureDim)
//   SPTAG::ErrorCode      AnnService/inc/Core/DefinitionList.h:54-68 (same numeric values)
// with the same names, argument meaning and error behaviour, so existing call sites
// (Wrappers/src/CoreInterface.cpp:206-238, IndexSearcher/main.cpp:194-217) compile against it by
// switching the namespace -- for hosts that do NOT link the reference at all.  Hosts that do use the real subclass,
// sptag_vector_index.hpp (`class SPTAG::B200::Index : public SPTAG::VectorIndex`, compiled against the reference's
// headers), which is the drop-in proper.
#pragma once

#include <cfloat>
#include <limits>
#include <cstdint>
#include <cstring>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sptag_b200.h"

namespace SPTAG_B200 {

typedef std::int32_t SizeType;
typedef std::int32_t DimensionType;
const float MaxDist = (std::numeric_limits<float>::max)() / 10;  // Common.h:122

enum class ErrorCode : std::uint16_t {
    Success = 0x0000,
    Fail = 0x0001,
    FailedOpenFile = 0x0002,
    ParamNotFound = 0x0010,
    FailedParseValue = 0x0011,
    MemoryOverFlow = 0x0012,
    LackOfInputs = 0x0013,
    VectorNotFound = 0x0014,
    EmptyIndex = 0x0015,
    EmptyData = 0x0016,
    DimensionSizeMismatch = 0x0017,
};

// SearchResult.h:65-78 without the metadata blob (metadata never crosses the device boundary;
// a wrapping VectorIndex fills it from its own MetadataSet exactly as BKTIndex.cpp:611-618 does)
struct BasicResult {
    SizeType VID;
    float Dist;
    bool RelaxedMono;  // SearchResult.h: set by ResultIterator::Next (ResultIterator.cpp:47-50)
    BasicResult() : VID(-1), Dist(MaxDist), RelaxedMono(false) {}
    BasicResult(SizeType p_vid, float p_dist) : VID(p_vid), Dist(p_dist), RelaxedMono(false) {}
};

// SearchQuery.h:15-254: a target plus K result slots (owning or viewing a caller buffer)
class QueryResult {
public:
    QueryResult(const void* p_target, int p_resultNum, bool /*p_withMeta*/ = false)
        : m_target(p_target), m_resultNum(p_resultNum), m_own(p_resultNum), m_results(m_own.data()) {}
    QueryResult(const void* p_target, int p_resultNum, bool /*p_withMeta*/, BasicResult* p_results)
        : m_target(p_target), m_resultNum(p_resultNum), m_results(p_results) {}
    const void* GetTarget() const { return m_target; }
    void SetTarget(const void* p_target) { m_target = p_target; }
    int GetResultNum() const { return m_resultNum; }
    void SetResultNum(int p_resultNum) { m_resultNum = p_resultNum; }  // SearchQuery.h:114-117
    BasicResult* GetResult(int i) const { return i < m_resultNum ? m_results + i : nullptr; }
    BasicResult* GetResults() const { return m_results; }
    void Reset() {
        for (int i = 0; i < m_resultNum; ++i) m_results[i] = BasicResult();
    }

private:
    const void* m_target;
    int m_resultNum;
    std::vector<BasicResult> m_own;
    BasicResult* m_results;
};

// ResultIterator.h / ResultIterator.cpp: a resumable search for one target, over sptag_b200_iterator_*.
class ResultIterator {
public:
    ResultIterator(sptag_b200_handle p_index, const void* p_target, bool p_searchDeleted = false) : m_target(p_target) {
        if (sptag_b200_iterator_open_ex(p_index, p_target, 1, p_searchDeleted ? 1 : 0, &m_it) != 0) m_it = nullptr;
    }
    ~ResultIterator() { Close(); }
    ResultIterator(const ResultIterator&) = delete;
    ResultIterator& operator=(const ResultIterator&) = delete;
    bool IsOpen() const { return m_it != nullptr; }

    // ResultIterator::Next (ResultIterator.cpp:31-55): the first call sizes the QueryResult; later batches are capped
    // by the previous result count
    std::shared_ptr<QueryResult> Next(int batch) {
        if (m_queryResult == nullptr)
            m_queryResult = std::make_shared<QueryResult>(m_target, batch, true);
        else if (batch <= m_queryResult->GetResultNum())
            m_queryResult->SetResultNum(batch);
        else
            batch = m_queryResult->GetResultNum();
        m_queryResult->Reset();
        if (m_it == nullptr || batch < 1) {
            m_queryResult->SetResultNum(0);
            return m_queryResult;
        }
        std::vector<std::int32_t> ids((size_t)batch);
        std::vector<float> dists((size_t)batch);
        std::int32_t count = 0;
        std::uint8_t relaxed = 0;
        if (sptag_b200_iterator_next(m_it, batch, ids.data(), dists.data(), &count, &relaxed) != 0) count = 0;
        m_relaxedMono = relaxed != 0;
        for (int i = 0; i < count; ++i) {
            BasicResult* r = m_queryResult->GetResult(i);
            r->VID = ids[(size_t)i];
            r->Dist = dists[(size_t)i];
            r->RelaxedMono = m_relaxedMono;
        }
        m_queryResult->SetResultNum(count);
        return m_queryResult;
    }
    bool GetRelaxedMono() const { return m_relaxedMono; }
    void Close() {
        if (m_it != nullptr) sptag_b200_iterator_close(m_it);
        m_it = nullptr;
    }
    const void* GetTarget() const { return m_target; }

private:
    sptag_b200_iter m_it = nullptr;
    const void* m_target;
    std::shared_ptr<QueryResult> m_queryResult;
    bool m_relaxedMono = false;
};

class VectorIndex {
public:
    ~VectorIndex() { sptag_b200_destroy(m_handle); }
    VectorIndex(const VectorIndex&) = delete;
    VectorIndex& operator=(const VectorIndex&) = delete;

    // VectorIndex::LoadIndex(folder, index) (VectorIndex.cpp:617-681)
    static ErrorCode LoadIndex(const std::string& p_loaderFilePath, std::shared_ptr<VectorIndex>& p_vectorIndex,
                               int device = -1, SizeType idOffset = 0) {
        sptag_b200_handle h = nullptr;
        int rc = sptag_b200_load(p_loaderFilePath.c_str(), device, idOffset, &h);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        p_vectorIndex.reset(new VectorIndex(h));
        return ErrorCode::Success;
    }

    // From arrays already in host memory (what BKT::Index<T> holds after BuildIndex/LoadIndexData)
    static ErrorCode Create(const sptag_b200_index_desc& desc, std::shared_ptr<VectorIndex>& p_vectorIndex) {
        sptag_b200_handle h = nullptr;
        int rc = sptag_b200_create(&desc, &h);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        p_vectorIndex.reset(new VectorIndex(h));
        return ErrorCode::Success;
    }

    // VectorIndex::SearchIndex(QueryResult&, bool) (VectorIndex.h:41; BKTIndex.cpp:595-620).
    // One query is one tiny batch on the device; prefer the batched overload.
    ErrorCode SearchIndex(QueryResult& p_query, bool p_searchDeleted = false) const {
        return SearchWith(p_query.GetTarget(), 1, p_query.GetResultNum(), p_searchDeleted, 0, nullptr, p_query.GetResults());
    }

    // VectorIndex::SearchIndex(const void*, int, int, bool, BasicResult*) (VectorIndex.h:103,
    // VectorIndex.cpp:454-463).  p_results is caller-owned [p_vectorCount x p_neighborCount].
    // (metadata: this mirror has no MetadataSet; the real subclass, sptag_vector_index.hpp, fills Meta)
    ErrorCode SearchIndex(const void* p_vector, int p_vectorCount, int p_neighborCount, bool /*p_withMeta*/,
                          BasicResult* p_results) const {
        return SearchWith(p_vector, p_vectorCount, p_neighborCount, false, 0, nullptr, p_results);
    }

    // VectorIndex::SearchIndexWithFilter (VectorIndex.h:57, BKTIndex.cpp:622-647).  The reference's callback sees the
    // vector's metadata; here the predicate receives the vector id (the caller owns the id -> metadata mapping) and is
    // evaluated once per vector on the host before the batch runs on the device.
    template <typename Pred>
    ErrorCode SearchIndexWithFilter(QueryResult& p_query, Pred p_allowed, int maxCheck = 0, bool p_searchDeleted = false) const {
        if (!m_handle) return ErrorCode::EmptyIndex;
        const SizeType n = GetNumSamples();
        std::vector<std::uint8_t> allowed((size_t)n);
        for (SizeType i = 0; i < n; ++i) allowed[(size_t)i] = p_allowed(i) ? 1 : 0;
        return SearchWith(p_query.GetTarget(), 1, p_query.GetResultNum(), p_searchDeleted, maxCheck, allowed.data(),
                          p_query.GetResults());
    }

    // VectorIndex::RefineSearchIndex (VectorIndex.h:53, BKTIndex.cpp:698-711) for a base vector of the index: the
    // refine-flavoured search (MaxCheckForRefineGraph, searchDuplicated = false) with sample `p_node` as the query.
    // The result buffer of p_query receives the K = GetResultNum() nearest, like the reference's call in
    // NeighborhoodGraph::RefineNode (NeighborhoodGraph.h:534-545).
    ErrorCode RefineSearchIndex(SizeType p_node, QueryResult& p_query) const {
        if (!m_handle) return ErrorCode::EmptyIndex;
        const int k = p_query.GetResultNum();
        if (k < 2) return ErrorCode::LackOfInputs;
        std::vector<std::int32_t> ids((size_t)k);
        std::vector<float> dists((size_t)k);
        int rc = sptag_b200_refine_graph(m_handle, p_node, 1, k - 1, sptag_b200_graph_degree(m_handle), 1.0f, nullptr,
                                         ids.data(), dists.data(), 0);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        for (int i = 0; i < k; ++i) {
            p_query.GetResult(i)->VID = ids[(size_t)i];
            p_query.GetResult(i)->Dist = dists[(size_t)i];
        }
        return ErrorCode::Success;
    }

    // One NeighborhoodGraph::RefineGraph pass (NeighborhoodGraph.h:459-488: RefineNode for every node) on the device;
    // p_newGraph (nullable) receives GetNumSamples() x neighbourhood-size rows; p_install replaces the index's graph.
    ErrorCode RefineGraphPass(int p_cef, float p_rngFactor = 1.0f, std::int32_t* p_newGraph = nullptr, bool p_install = true) {
        if (!m_handle) return ErrorCode::EmptyIndex;
        return static_cast<ErrorCode>(sptag_b200_refine_graph(m_handle, 0, sptag_b200_num_vectors(m_handle), p_cef,
                                                              sptag_b200_graph_degree(m_handle), p_rngFactor, p_newGraph,
                                                              nullptr, nullptr, p_install ? 1 : 0));
    }

    // NeighborhoodGraph::SaveGraph (NeighborhoodGraph.h:606-615) for the index's current -- e.g. device-refined -- graph:
    // a graph.bin the reference's LoadIndex reads
    ErrorCode SaveGraph(const std::string& p_graphFile) const {
        if (!m_handle) return ErrorCode::EmptyIndex;
        const std::int32_t rows = sptag_b200_num_vectors(m_handle), cols = sptag_b200_graph_degree(m_handle);
        std::vector<std::int32_t> g((size_t)rows * cols);
        int rc = sptag_b200_get_graph(m_handle, g.data());
        if (rc != 0) return static_cast<ErrorCode>(rc);
        FILE* f = std::fopen(p_graphFile.c_str(), "wb");
        if (!f) return ErrorCode::FailedOpenFile;
        bool ok = std::fwrite(&rows, 4, 1, f) == 1 && std::fwrite(&cols, 4, 1, f) == 1 &&
                  std::fwrite(g.data(), 4, g.size(), f) == g.size();
        ok = (std::fclose(f) == 0) && ok;
        return ok ? ErrorCode::Success : ErrorCode::Fail;
    }

    // VectorIndex::AddIndex (VectorIndex.h:37, BKTIndex.cpp:902-970) without metadata: sptag_b200_add
    ErrorCode AddIndex(const void* p_data, SizeType p_vectorNum, DimensionType p_dimension, bool p_normalized = false) {
        if (!m_handle) return ErrorCode::EmptyIndex;
        return static_cast<ErrorCode>(sptag_b200_add(m_handle, p_data, p_vectorNum, p_dimension, p_normalized ? 1 : 0, nullptr));
    }

    // VectorIndex::DeleteIndex(const SizeType&) (VectorIndex.h:181, BKTIndex.cpp:893-899): Success or VectorNotFound
    ErrorCode DeleteIndex(const SizeType& p_id) {
        if (!m_handle) return ErrorCode::EmptyIndex;
        std::int32_t code = 0;
        const int rc = sptag_b200_delete(m_handle, &p_id, 1, &code);
        return static_cast<ErrorCode>(rc != 0 ? rc : code);
    }

    // VectorIndex::DeleteIndex(const void*, SizeType) (VectorIndex.h:39, BKTIndex.cpp:876-890), single-thread order
    ErrorCode DeleteIndex(const void* p_vectors, SizeType p_vectorNum) {
        if (!m_handle) return ErrorCode::EmptyIndex;
        return static_cast<ErrorCode>(sptag_b200_delete_vectors(m_handle, p_vectors, p_vectorNum));
    }

    // VectorIndex::SaveIndex(folder) (VectorIndex.h:87): a folder the reference's LoadIndex and this LoadIndex read
    ErrorCode SaveIndex(const std::string& p_folderPath) const {
        if (!m_handle) return ErrorCode::EmptyIndex;
        return static_cast<ErrorCode>(sptag_b200_save(m_handle, p_folderPath.c_str()));
    }

    // VectorIndex::GetIterator (VectorIndex.h:43, BKTIndex.cpp:650-657); nullptr where the reference returns nullptr
    // (index not ready, KDT)
    std::shared_ptr<ResultIterator> GetIterator(const void* p_target, bool p_searchDeleted = false) const {
        if (!m_handle) return nullptr;
        auto it = std::make_shared<ResultIterator>(m_handle, p_target, p_searchDeleted);
        if (!it->IsOpen()) return nullptr;
        return it;
    }

    // VectorIndex::SetParameter / GetParameter (BKTIndex.cpp:980-1025)
    ErrorCode SetParameter(const char* p_param, const char* p_value, const char* /*p_section*/ = nullptr) {
        return static_cast<ErrorCode>(sptag_b200_set_param(m_handle, p_param, p_value));
    }
    std::string GetParameter(const char* p_param, const char* /*p_section*/ = nullptr) const {
        char buf[64] = {0};
        if (sptag_b200_get_param(m_handle, p_param, buf, sizeof(buf)) != 0) return std::string();
        return std::string(buf);
    }
    SizeType GetNumSamples() const { return sptag_b200_num_vectors(m_handle); }
    DimensionType GetFeatureDim() const { return sptag_b200_dim(m_handle); }
    bool IsReady() const { return m_handle != nullptr; }
    sptag_b200_handle Handle() const { return m_handle; }

private:
    // p_searchDeleted, maxCheck and the filter map are per-call arguments of the C ABI (sptag_b200_search_options):
    // nothing is written into the handle, so threads mixing different values do not interact
    ErrorCode SearchWith(const void* p_vector, int p_vectorCount, int p_neighborCount, bool p_searchDeleted, int p_maxCheck,
                         const std::uint8_t* p_allowed, BasicResult* p_results) const {
        if (!m_handle) return ErrorCode::EmptyIndex;
        const size_t n = static_cast<size_t>(p_vectorCount) * p_neighborCount;
        std::vector<std::int32_t> ids(n);
        std::vector<float> dists(n);
        sptag_b200_search_options o;
        std::memset(&o, 0, sizeof(o));
        o.struct_size = (std::int32_t)sizeof(o);
        o.search_deleted = p_searchDeleted ? 1 : 0;
        o.max_check = p_maxCheck;
        o.allowed = p_allowed;
        int rc = sptag_b200_search_ex(m_handle, p_vector, p_vectorCount, p_neighborCount, &o, ids.data(), dists.data(), nullptr);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        for (size_t i = 0; i < n; ++i) {  // scatter the POD SoA into the caller's AoS
            p_results[i].VID = ids[i];
            p_results[i].Dist = dists[i];
        }
        return ErrorCode::Success;
    }
    explicit VectorIndex(sptag_b200_handle h) : m_handle(h) {}
    sptag_b200_handle m_handle;
};

}  // namespace SPTAG_B200
