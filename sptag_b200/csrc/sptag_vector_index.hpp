// sptag_vector_index.hpp -- the drop-in: a real `SPTAG::VectorIndex` subclass whose search path runs on the B200.
//
// Compiles against the reference's own headers (AnnService/inc) and links libsptag_b200.so through the C ABI
// (include/sptag_b200.h).  `SPTAG::B200::Index` wraps an ordinary CPU index (BKT::Index<T> / KDT::Index<T>, e.g. what
// VectorIndex::LoadIndex returned) and
//   * serves the search entry points from the device:
//       SearchIndex(QueryResult&, bool)                         VectorIndex.h:41   (BKTIndex.cpp:595-620)
//       SearchIndex(const void*, int, int, bool, BasicResult*)  VectorIndex.h:103  (VectorIndex.cpp:454-463)
//       SearchIndexWithFilter                                   VectorIndex.h:57   (BKTIndex.cpp:622-647)
//       RefineSearchIndex                                       VectorIndex.h:53   (BKTIndex.cpp:698-711)
//       GetIterator / RentWorkSpace / SearchIndexIterativeNext / SearchIndexIterativeEnd /
//       SearchIndexIterativeFromNeareast                        VectorIndex.h:43-51 (BKTIndex.cpp:354-427, :543-595,
//                                                               :650-696) -- so the reference's own ResultIterator
//                                                               (ResultIterator.cpp) and SPANN's head-index calls
//                                                               (SPANNIndex.cpp:203, :259-285) run on top of it unchanged
//   * fills `Meta` from the wrapped index's MetadataSet exactly like BKTIndex.cpp:611-618 (metadata never crosses
//     the device boundary),
//   * forwards every other virtual (build, add, delete, save, parameters, samples, quantizer ...) to the wrapped index;
//     after a mutating call the device copy is re-synchronised lazily before the next search.
//
// The device copy is made from the wrapped index's own serialisation (VectorIndex::SaveIndexData into memory
// blobs: vectors / tree / graph / deletes, BKT/Index.h:151-159, BKTIndex.cpp:129-141), so it needs no folder and
// is bit-identical to what SaveIndex would write.
//
// Existing callers (Wrappers/src/CoreInterface.cpp:206-238 AnnIndex::Search / BatchSearch, IndexSearcher/main.cpp,
// Server/SearchExecutor.cpp:83, SPANNIndex.cpp:203) hold a std::shared_ptr<VectorIndex>; they switch with
//     std::shared_ptr<SPTAG::VectorIndex> idx;  SPTAG::VectorIndex::LoadIndex(folder, idx);
//     idx = SPTAG::B200::Index::Attach(idx, /*device*/ 0);          // <- the one added line
#pragma once

#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "inc/Core/VectorIndex.h"
#include "inc/Core/ResultIterator.h"
#include "inc/Core/Common/QueryResultSet.h"
#include "inc/Helper/DiskIO.h"

#include "../../include/sptag_b200.h"

namespace SPTAG {
namespace B200 {

class Index : public VectorIndex {
public:
    // Wraps `p_cpu` and uploads it to `p_device`; nullptr if the index type is not searchable on the device (the
    // caller keeps using p_cpu then).  p_idOffset: added to returned ids (vector-partition shards).
    static std::shared_ptr<VectorIndex> Attach(std::shared_ptr<VectorIndex> p_cpu, int p_device = -1, SizeType p_idOffset = 0) {
        if (!p_cpu) return nullptr;
        std::shared_ptr<Index> idx(new Index(std::move(p_cpu), p_device, p_idOffset));
        if (idx->Sync() != ErrorCode::Success) return nullptr;
        return idx;
    }

    ~Index() override {
        CloseAllIterators();
        if (m_handle) sptag_b200_destroy(m_handle);
    }

    sptag_b200_handle Handle() const { return m_handle; }
    const std::shared_ptr<VectorIndex>& Wrapped() const { return m_cpu; }

    // Re-uploads the wrapped index (after AddIndex / DeleteIndex / RefineIndex / MergeIndex on it)
    ErrorCode Sync() const {
        std::lock_guard<std::mutex> lock(m_syncLock);
        return SyncLocked();
    }

    // ------------------------------------------------------------------------------------------------
    // the search path, served by the device
    // ------------------------------------------------------------------------------------------------
    ErrorCode SearchIndex(QueryResult& p_query, bool p_searchDeleted = false) const override {
        if (!m_cpu->IsReady()) return ErrorCode::EmptyIndex;
        ErrorCode ec = SearchBatch(p_query.GetTarget(), 1, p_query.GetResultNum(), p_searchDeleted, 0, nullptr,
                                   p_query.GetResults());
        if (ec != ErrorCode::Success) return ec;
        FillMeta(p_query, p_query.GetResultNum());
        return ErrorCode::Success;
    }

    // VectorIndex.cpp:454-463: the reference strides the queries by value size x GetFeatureDim() and runs
    // SearchIndex(QueryResult&) per query; here the whole batch is one kernel launch
    ErrorCode SearchIndex(const void* p_vector, int p_vectorCount, int p_neighborCount, bool p_withMeta,
                          BasicResult* p_results) const override {
        if (!m_cpu->IsReady()) return ErrorCode::EmptyIndex;
        ErrorCode ec = SearchBatch(p_vector, p_vectorCount, p_neighborCount, false, 0, nullptr, p_results);
        if (ec != ErrorCode::Success) return ec;
        MetadataSet* meta = p_withMeta ? m_cpu->GetMetadata() : nullptr;
        if (meta != nullptr) {
            const size_t n = (size_t)p_vectorCount * p_neighborCount;
            for (size_t i = 0; i < n; ++i)
                p_results[i].Meta = (p_results[i].VID < 0) ? ByteArray::c_empty : meta->GetMetadataCopy(Local(p_results[i].VID));
        }
        return ErrorCode::Success;
    }

    // BKTIndex.cpp:622-647.  The device cannot call back into host code, so filterFunc is evaluated once per vector
    // into a byte map (the reference evaluates it lazily on the vectors it is about to add -- same verdicts).
    ErrorCode SearchIndexWithFilter(QueryResult& p_query, std::function<bool(const ByteArray&)> filterFunc, int maxCheck = 0,
                                    bool p_searchDeleted = false) const override {
        if (!m_cpu->IsReady()) return ErrorCode::EmptyIndex;
        if (GetIndexAlgoType() != IndexAlgoType::BKT) return m_cpu->SearchIndexWithFilter(p_query, filterFunc, maxCheck, p_searchDeleted);
        MetadataSet* meta = m_cpu->GetMetadata();
        const SizeType n = m_cpu->GetNumSamples();
        std::vector<std::uint8_t> allowed((size_t)n, 1);
        if (filterFunc && meta != nullptr)
            for (SizeType i = 0; i < n; ++i) allowed[(size_t)i] = filterFunc(meta->GetMetadata(i)) ? 1 : 0;
        ErrorCode ec = SearchBatch(p_query.GetTarget(), 1, p_query.GetResultNum(), p_searchDeleted, maxCheck,
                                   allowed.data(), p_query.GetResults());
        if (ec != ErrorCode::Success) return ec;
        FillMeta(p_query, p_query.GetResultNum());
        return ErrorCode::Success;
    }

    // BKTIndex.cpp:698-711: MaxCheckForRefineGraph, searchDuplicated = false, no metadata
    ErrorCode RefineSearchIndex(QueryResult& p_query, bool p_searchDeleted = false) const override {
        const ErrorCode ready = Ready();
        if (ready != ErrorCode::Success) return ready;
        const int k = p_query.GetResultNum();
        std::vector<std::int32_t> ids((size_t)k);
        std::vector<float> dists((size_t)k);
        int rc = sptag_b200_refine_search(m_handle, p_query.GetTarget(), 1, k, p_searchDeleted ? 1 : 0, ids.data(), dists.data());
        if (rc != 0) return static_cast<ErrorCode>(rc);
        Scatter(ids.data(), dists.data(), (size_t)k, p_query.GetResults());
        return ErrorCode::Success;
    }

    // BKTIndex.cpp:650-657: the reference's own ResultIterator, driving the overrides below
    std::shared_ptr<ResultIterator> GetIterator(const void* p_target, bool p_searchDeleted = false) const override {
        if (!m_cpu->IsReady() || GetIndexAlgoType() != IndexAlgoType::BKT) return m_cpu->GetIterator(p_target, p_searchDeleted);
        return std::make_shared<ResultIterator>((const void*)static_cast<const VectorIndex*>(this), p_target, p_searchDeleted, 1);
    }

    // The rented WorkSpace is the caller's ticket: the device keeps the query's real work space (visited set,
    // NGQueue, SPTQueue) in HBM, keyed by this object (BKTIndex.cpp:686-696)
    std::unique_ptr<COMMON::WorkSpace> RentWorkSpace(int batch) const override { return m_cpu->RentWorkSpace(batch); }

    ErrorCode SearchIndexIterativeNext(QueryResult& p_query, COMMON::WorkSpace* workSpace, int p_batch, int& resultCount,
                                       bool p_isFirst, bool p_searchDeleted) const override {
        resultCount = 0;
        if (!m_cpu->IsReady()) return ErrorCode::EmptyIndex;
        sptag_b200_iter it = nullptr;
        const ErrorCode opened = DeviceIterator(workSpace, p_query.GetTarget(), p_isFirst, p_searchDeleted, it);
        if (opened != ErrorCode::Success) return opened;
        std::vector<std::int32_t> ids((size_t)p_batch);
        std::vector<float> dists((size_t)p_batch);
        std::int32_t count = 0;
        std::uint8_t relaxed = 0;
        int rc = sptag_b200_iterator_next(it, p_batch, ids.data(), dists.data(), &count, &relaxed);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        Scatter(ids.data(), dists.data(), (size_t)count, p_query.GetResults());
        workSpace->m_relaxedMono = relaxed != 0;  // what ResultIterator::Next reads back (ResultIterator.cpp:47-50)
        resultCount = count;
        FillMeta(p_query, count);
        return ErrorCode::Success;
    }

    ErrorCode SearchIndexIterativeEnd(std::unique_ptr<COMMON::WorkSpace> workSpace) const override {
        if (workSpace) {
            std::lock_guard<std::mutex> lock(m_iterLock);
            auto f = m_iters.find(workSpace.get());
            if (f != m_iters.end()) {
                sptag_b200_iterator_close(f->second);
                m_iters.erase(f);
            }
        }
        return m_cpu->SearchIndexIterativeEnd(std::move(workSpace));
    }

    // BKTIndex.cpp:543-595 (SPANN's head-index call, SPANNIndex.cpp:259-285)
    bool SearchIndexIterativeFromNeareast(QueryResult& p_query, COMMON::WorkSpace* p_space, bool p_isFirst,
                                          bool p_searchDeleted = false) const override {
        if (!m_cpu->IsReady()) return false;
        sptag_b200_iter it = nullptr;
        if (DeviceIterator(p_space, p_query.GetTarget(), p_isFirst, p_searchDeleted, it) != ErrorCode::Success) return false;
        const int k = p_query.GetResultNum();
        std::vector<std::int32_t> ids((size_t)k);
        std::vector<float> dists((size_t)k);
        std::uint8_t found = 0;
        if (sptag_b200_iterator_next_from_nearest(it, k, ids.data(), dists.data(), &found) != 0) return false;
        // the reference leaves slots it does not fill as the caller Reset() them: (-1, MaxDist) -- what the device returns
        Scatter(ids.data(), dists.data(), (size_t)k, p_query.GetResults());
        return found != 0;
    }

    // ------------------------------------------------------------------------------------------------
    // everything else: the wrapped index
    // ------------------------------------------------------------------------------------------------
    ErrorCode BuildIndex(const void* p_data, SizeType p_vectorNum, DimensionType p_dimension, bool p_normalized = false,
                         bool p_shareOwnership = false) override {
        Dirty();
        return m_cpu->BuildIndex(p_data, p_vectorNum, p_dimension, p_normalized, p_shareOwnership);
    }
    ErrorCode BuildIndex(std::shared_ptr<VectorSet> p_vectorSet, std::shared_ptr<MetadataSet> p_metadataSet,
                         bool p_withMetaIndex = false, bool p_normalized = false, bool p_shareOwnership = false) override {
        Dirty();
        return m_cpu->BuildIndex(p_vectorSet, p_metadataSet, p_withMetaIndex, p_normalized, p_shareOwnership);
    }
    ErrorCode BuildIndex(bool p_normalized = false) override {
        Dirty();
        return m_cpu->BuildIndex(p_normalized);
    }
    ErrorCode AddIndex(const void* p_data, SizeType p_vectorNum, DimensionType p_dimension, std::shared_ptr<MetadataSet> p_metadataSet,
                       bool p_withMetaIndex = false, bool p_normalized = false) override {
        Dirty();
        return m_cpu->AddIndex(p_data, p_vectorNum, p_dimension, p_metadataSet, p_withMetaIndex, p_normalized);
    }
    ErrorCode AddIndex(std::shared_ptr<VectorSet> p_vectorSet, std::shared_ptr<MetadataSet> p_metadataSet,
                       bool p_withMetaIndex = false, bool p_normalized = false) override {
        Dirty();
        return m_cpu->AddIndex(p_vectorSet, p_metadataSet, p_withMetaIndex, p_normalized);
    }
    ErrorCode DeleteIndex(const void* p_vectors, SizeType p_vectorNum) override {
        Dirty();
        return m_cpu->DeleteIndex(p_vectors, p_vectorNum);
    }
    ErrorCode DeleteIndex(ByteArray p_meta) override {
        Dirty();
        return m_cpu->DeleteIndex(p_meta);
    }
    ErrorCode DeleteIndex(const SizeType& p_id) override {
        Dirty();
        return m_cpu->DeleteIndex(p_id);
    }
    ErrorCode MergeIndex(VectorIndex* p_addindex, int p_threadnum, IAbortOperation* p_abort) override {
        Dirty();
        return m_cpu->MergeIndex(p_addindex, p_threadnum, p_abort);
    }
    ErrorCode RefineIndex(std::shared_ptr<VectorIndex>& p_newIndex) override { return m_cpu->RefineIndex(p_newIndex); }
    ErrorCode RefineIndex(const std::vector<std::shared_ptr<Helper::DiskIO>>& p_indexStreams, IAbortOperation* p_abort) override {
        return m_cpu->RefineIndex(p_indexStreams, p_abort);
    }
    ErrorCode UpdateIndex() override {
        Dirty();
        return m_cpu->UpdateIndex();
    }
    ErrorCode SearchTree(QueryResult& p_query) const override { return m_cpu->SearchTree(p_query); }

    float AccurateDistance(const void* pX, const void* pY) const override { return m_cpu->AccurateDistance(pX, pY); }
    float ComputeDistance(const void* pX, const void* pY) const override { return m_cpu->ComputeDistance(pX, pY); }
    float GetDistance(const void* target, const SizeType idx) const override { return m_cpu->GetDistance(target, idx); }
    const void* GetSample(const SizeType idx) const override { return m_cpu->GetSample(idx); }
    const void* GetSample(ByteArray p_meta, bool& deleteFlag) override { return m_cpu->GetSample(p_meta, deleteFlag); }
    bool ContainSample(const SizeType idx) const override { return m_cpu->ContainSample(idx); }
    bool NeedRefine() const override { return m_cpu->NeedRefine(); }
    DimensionType GetFeatureDim() const override { return m_cpu->GetFeatureDim(); }
    SizeType GetNumSamples() const override { return m_cpu->GetNumSamples(); }
    SizeType GetNumDeleted() const override { return m_cpu->GetNumDeleted(); }
    DistCalcMethod GetDistCalcMethod() const override { return m_cpu->GetDistCalcMethod(); }
    IndexAlgoType GetIndexAlgoType() const override { return m_cpu->GetIndexAlgoType(); }
    VectorValueType GetVectorValueType() const override { return m_cpu->GetVectorValueType(); }

    std::string GetParameter(const char* p_param, const char* p_section = nullptr) const override {
        if (p_param && std::strncmp(p_param, "B200.", 5) == 0 && m_handle) {
            char buf[64] = {0};
            return sptag_b200_get_param(m_handle, p_param, buf, sizeof(buf)) == 0 ? std::string(buf) : std::string();
        }
        return m_cpu->GetParameter(p_param, p_section);
    }
    // search-time parameters go to both sides (BKTIndex.cpp:980-1025); "B200.*" tuning knobs only to the device
    ErrorCode SetParameter(const char* p_param, const char* p_value, const char* p_section = nullptr) override {
        if (p_param && std::strncmp(p_param, "B200.", 5) == 0)
            return m_handle ? static_cast<ErrorCode>(sptag_b200_set_param(m_handle, p_param, p_value)) : ErrorCode::EmptyIndex;
        ErrorCode ec = m_cpu->SetParameter(p_param, p_value, p_section);
        if (ec == ErrorCode::Success && m_handle) PushSearchParameters();
        return ec;
    }
    std::string GetParameter(const std::string& p_param, const std::string& p_section = "Index") const override {
        return GetParameter(p_param.c_str(), p_section.c_str());
    }
    ErrorCode SetParameter(const std::string& p_param, const std::string& p_value, const std::string& p_section = "Index") override {
        return SetParameter(p_param.c_str(), p_value.c_str(), p_section.c_str());
    }

    bool IsReady() const override { return m_cpu->IsReady(); }
    void SetReady(bool p_ready) override { m_cpu->SetReady(p_ready); }
    std::shared_ptr<std::vector<std::uint64_t>> CalculateBufferSize() const override { return m_cpu->CalculateBufferSize(); }
    ErrorCode SaveIndex(std::string& p_config, const std::vector<ByteArray>& p_indexBlobs) override { return m_cpu->SaveIndex(p_config, p_indexBlobs); }
    ErrorCode SaveIndex(const std::string& p_folderPath) override { return m_cpu->SaveIndex(p_folderPath); }
    ErrorCode SaveIndexToFile(const std::string& p_file, IAbortOperation* p_abort = nullptr) override { return m_cpu->SaveIndexToFile(p_file, p_abort); }
    void ApproximateRNG(std::shared_ptr<VectorSet>& fullVectors, std::unordered_set<SizeType>& exceptIDS, int candidateNum, Edge* selections,
                        int replicaCount, int numThreads, int numTrees, int leafSize, float RNGFactor, int numGPUs) override {
        m_cpu->ApproximateRNG(fullVectors, exceptIDS, candidateNum, selections, replicaCount, numThreads, numTrees, leafSize, RNGFactor, numGPUs);
    }
    ByteArray GetMetadata(SizeType p_vectorID) const override { return m_cpu->GetMetadata(p_vectorID); }
    MetadataSet* GetMetadata() const override { return m_cpu->GetMetadata(); }
    void SetMetadata(MetadataSet* p_new) override { m_cpu->SetMetadata(p_new); }
    std::string GetIndexName() const override { return m_cpu->GetIndexName(); }
    void SetIndexName(std::string p_name) override { m_cpu->SetIndexName(p_name); }
    void SetQuantizerFileName(std::string p_QuantizerFileName) override { m_cpu->SetQuantizerFileName(p_QuantizerFileName); }
    void SetQuantizerADC(bool enableADC) override {
        m_cpu->SetQuantizerADC(enableADC);
        if (m_handle) sptag_b200_set_param(m_handle, "EnableADC", enableADC ? "1" : "0");
    }
    void SetQuantizer(std::shared_ptr<SPTAG::COMMON::IQuantizer> quantizer) override {
        Dirty();
        m_cpu->SetQuantizer(quantizer);
        m_pQuantizer = quantizer;
    }
    ErrorCode LoadQuantizer(std::string p_quantizerFile) override {
        Dirty();
        ErrorCode ec = m_cpu->LoadQuantizer(p_quantizerFile);
        m_pQuantizer = m_cpu->m_pQuantizer;
        return ec;
    }
    std::shared_ptr<SPTAG::COMMON::IQuantizer> GetQuantizer() override { return m_cpu->GetQuantizer(); }
    ErrorCode QuantizeVector(const void* p_data, SizeType p_num, ByteArray p_out) override { return m_cpu->QuantizeVector(p_data, p_num, p_out); }
    ErrorCode ReconstructVector(const void* p_data, SizeType p_num, ByteArray p_out) override { return m_cpu->ReconstructVector(p_data, p_num, p_out); }

    std::shared_ptr<std::vector<std::uint64_t>> BufferSize() const override { return m_cpu->BufferSize(); }
    std::shared_ptr<std::vector<std::string>> GetIndexFiles() const override { return m_cpu->GetIndexFiles(); }
    ErrorCode SaveConfig(std::shared_ptr<Helper::DiskIO> p_configout) override { return m_cpu->SaveConfig(p_configout); }
    ErrorCode SaveIndexData(const std::vector<std::shared_ptr<Helper::DiskIO>>& p_indexStreams) override { return m_cpu->SaveIndexData(p_indexStreams); }
    ErrorCode LoadConfig(Helper::IniReader& p_reader) override {
        Dirty();
        return m_cpu->LoadConfig(p_reader);
    }
    ErrorCode LoadIndexData(const std::vector<std::shared_ptr<Helper::DiskIO>>& p_indexStreams) override {
        Dirty();
        return m_cpu->LoadIndexData(p_indexStreams);
    }
    ErrorCode LoadIndexDataFromMemory(const std::vector<ByteArray>& p_indexBlobs) override {
        Dirty();
        return m_cpu->LoadIndexDataFromMemory(p_indexBlobs);
    }
    ErrorCode SetWorkSpaceFactory(std::unique_ptr<SPTAG::COMMON::IWorkSpaceFactory<SPTAG::COMMON::IWorkSpace>> up_workSpaceFactory) override {
        return m_cpu->SetWorkSpaceFactory(std::move(up_workSpaceFactory));
    }

private:
    Index(std::shared_ptr<VectorIndex> p_cpu, int p_device, SizeType p_idOffset)
        : m_cpu(std::move(p_cpu)), m_device(p_device), m_idOffset(p_idOffset) {
        m_pQuantizer = m_cpu->m_pQuantizer;
        m_bReady = true;
    }

    void Dirty() const { m_dirty = true; }

    SizeType Local(SizeType vid) const { return vid - m_idOffset; }

    ErrorCode Ready() const {
        if (!m_cpu->IsReady()) return ErrorCode::EmptyIndex;
        if (m_dirty || !m_handle) return Sync();
        return ErrorCode::Success;
    }

    static void Scatter(const std::int32_t* ids, const float* dists, size_t n, BasicResult* out) {
        for (size_t i = 0; i < n; ++i) {  // the C ABI returns POD SoA; BasicResult holds a ByteArray and cannot cross it
            out[i].VID = ids[i];
            out[i].Dist = dists[i];
        }
    }

    // BKTIndex.cpp:611-618
    void FillMeta(QueryResult& p_query, int count) const {
        MetadataSet* meta = p_query.WithMeta() ? m_cpu->GetMetadata() : nullptr;
        if (meta == nullptr) return;
        for (int i = 0; i < count; ++i) {
            const SizeType result = p_query.GetResult(i)->VID;
            p_query.SetMetadata(i, (result < 0) ? ByteArray::c_empty : meta->GetMetadataCopy(Local(result)));
        }
    }

    ErrorCode SearchBatch(const void* p_vectors, int p_count, int p_k, bool p_searchDeleted, int p_maxCheck,
                          const std::uint8_t* p_allowed, BasicResult* p_results) const {
        const ErrorCode ready = Ready();
        if (ready != ErrorCode::Success) return ready;
        const size_t n = (size_t)p_count * p_k;
        std::vector<std::int32_t> ids(n);
        std::vector<float> dists(n);
        sptag_b200_search_options o;
        std::memset(&o, 0, sizeof(o));
        o.struct_size = (std::int32_t)sizeof(o);
        o.search_deleted = p_searchDeleted ? 1 : 0;
        o.max_check = p_maxCheck;
        o.allowed = p_allowed;
        int rc = sptag_b200_search_ex(m_handle, p_vectors, p_count, p_k, &o, ids.data(), dists.data(), nullptr);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        Scatter(ids.data(), dists.data(), n, p_results);
        return ErrorCode::Success;
    }

    // one device iterator per rented WorkSpace; a first call on a reused WorkSpace starts over
    ErrorCode DeviceIterator(COMMON::WorkSpace* ws, const void* target, bool isFirst, bool searchDeleted, sptag_b200_iter& out) const {
        const ErrorCode ready = Ready();
        if (ready != ErrorCode::Success) return ready;
        std::lock_guard<std::mutex> lock(m_iterLock);
        auto f = m_iters.find(ws);
        if (isFirst && f != m_iters.end()) {
            sptag_b200_iterator_close(f->second);
            m_iters.erase(f);
            f = m_iters.end();
        }
        if (f == m_iters.end()) {
            if (!isFirst) return ErrorCode::Fail;
            sptag_b200_iter it = nullptr;
            int rc = sptag_b200_iterator_open_ex(m_handle, target, 1, searchDeleted ? 1 : 0, &it);
            if (rc != 0) return static_cast<ErrorCode>(rc);
            f = m_iters.emplace(ws, it).first;
        }
        out = f->second;
        return ErrorCode::Success;
    }

    void CloseAllIterators() const {
        std::lock_guard<std::mutex> lock(m_iterLock);
        for (auto& kv : m_iters) sptag_b200_iterator_close(kv.second);
        m_iters.clear();
    }

    void PushSearchParameters() const {
        // (EnableBfs: BKT only -- a KDT index has no such parameter, and the device refuses it there)
        static const char* names[] = {"MaxCheck", "MaxCheckForRefineGraph", "NumberOfInitialDynamicPivots", "NumberOfOtherDynamicPivots",
                                      "ThresholdOfNumberOfContinuousNoBetterPropagation", "EnableBfs"};
        for (const char* nm : names) {
            const std::string v = m_cpu->GetParameter(nm, "Index");
            if (!v.empty()) sptag_b200_set_param(m_handle, nm, v.c_str());
        }
    }

    // VectorIndex::SaveIndexData into memory (the blobs are exactly the files SaveIndex writes: Dataset.h:146-180,
    // BKTree.h:635-645 / KDTree.h:123-133, NeighborhoodGraph.h:606-615, Labelset.h:78-83) -> sptag_b200_create
    ErrorCode SyncLocked() const {
        const IndexAlgoType algo = m_cpu->GetIndexAlgoType();
        if (algo != IndexAlgoType::BKT && algo != IndexAlgoType::KDT) return ErrorCode::LackOfInputs;
        if (!m_cpu->IsReady() || m_cpu->GetNumSamples() <= 0) return ErrorCode::EmptyIndex;
        std::shared_ptr<std::vector<std::uint64_t>> sizes = m_cpu->BufferSize();
        if (!sizes || sizes->size() < 4) return ErrorCode::Fail;
        std::vector<std::vector<char>> blobs(4);
        std::vector<std::shared_ptr<Helper::DiskIO>> streams;
        for (int i = 0; i < 4; ++i) {
            blobs[i].resize((size_t)(*sizes)[i]);
            auto io = std::make_shared<Helper::SimpleBufferIO>();
            io->Initialize(blobs[i].data(), std::ios::binary | std::ios::out, (*sizes)[i]);
            streams.push_back(io);
        }
        const ErrorCode saved = m_cpu->SaveIndexData(streams);
        if (saved != ErrorCode::Success) return saved;

        sptag_b200_index_desc d;
        std::memset(&d, 0, sizeof(d));
        d.struct_size = (std::int32_t)sizeof(d);
        d.device = m_device;
        d.algo = (algo == IndexAlgoType::BKT) ? SPTAG_B200_ALGO_BKT : SPTAG_B200_ALGO_KDT;
        d.value_type = (std::int32_t)m_cpu->GetVectorValueType();
        d.metric = (std::int32_t)m_cpu->GetDistCalcMethod();
        const std::int32_t* vh = (const std::int32_t*)blobs[0].data();
        d.num_vectors = vh[0];
        d.dim = vh[1];
        d.vectors = blobs[0].data() + 8;
        const std::int32_t* th = (const std::int32_t*)blobs[1].data();
        d.tree_num = th[0];
        d.tree_starts = th + 1;
        d.node_count = th[1 + d.tree_num];
        d.tree_nodes = th + 2 + d.tree_num;
        const std::int32_t* gh = (const std::int32_t*)blobs[2].data();
        if (gh[0] != d.num_vectors) return ErrorCode::Fail;
        d.graph_degree = gh[1];
        d.graph = gh + 2;
        const std::int32_t* dh = (const std::int32_t*)blobs[3].data();
        d.num_deleted = dh[0];
        d.deleted = (d.num_deleted > 0) ? (const std::int8_t*)(blobs[3].data() + 12) : nullptr;
        d.id_offset = m_idOffset;

        sptag_b200_handle fresh = nullptr;
        int rc = sptag_b200_create(&d, &fresh);
        if (rc != 0) return static_cast<ErrorCode>(rc);
        if (m_cpu->m_pQuantizer) {  // IQuantizer::SaveQuantizer blob (PQQuantizer.h:226-239, OPQQuantizer.h:133-147)
            std::vector<char> qb((size_t)m_cpu->m_pQuantizer->BufferSize());
            auto io = std::make_shared<Helper::SimpleBufferIO>();
            io->Initialize(qb.data(), std::ios::binary | std::ios::out, qb.size());
            if (m_cpu->m_pQuantizer->SaveQuantizer(io) != ErrorCode::Success ||
                (rc = sptag_b200_set_quantizer(fresh, qb.data(), (std::int64_t)qb.size())) != 0) {
                sptag_b200_destroy(fresh);
                return rc != 0 ? static_cast<ErrorCode>(rc) : ErrorCode::Fail;
            }
            sptag_b200_set_param(fresh, "EnableADC", m_cpu->m_pQuantizer->GetEnableADC() ? "1" : "0");
        }
        CloseAllIterators();
        if (m_handle) sptag_b200_destroy(m_handle);
        m_handle = fresh;
        PushSearchParameters();
        m_dirty = false;
        return ErrorCode::Success;
    }

    std::shared_ptr<VectorIndex> m_cpu;
    int m_device;
    SizeType m_idOffset;
    mutable sptag_b200_handle m_handle = nullptr;
    mutable bool m_dirty = true;
    mutable std::mutex m_syncLock, m_iterLock;
    mutable std::map<COMMON::WorkSpace*, sptag_b200_iter> m_iters;
};

}  // namespace B200
}  // namespace SPTAG
