// TEST INFRASTRUCTURE.  Runs SPANN's build with the unmodified reference, so that tests/golden/make_golden_spann_build.py
// and tools/spann_build_bench.py can compare the device's posting-list build (sptag_b200_spann_build) against it.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage:
//   spann_build_ref full <folder> <Float|Int8|Int16> <L2|Cosine> <n> <dim> <data file> <threads> [Section.Name=Value ...]
//       SelectHead -> BuildHead -> BuildSSDIndex (SPANNIndex.cpp:818-951) on the rows, then SaveIndex(folder).
//   spann_build_ref head <folder> <Float|Int8|Int16> <L2|Cosine> <n> <dim> <data file> <threads> [Section.Name=Value ...]
//       SelectHead -> BuildHead only (BuildSsdIndex false), then indexloader.ini as SaveIndex writes it ([Index], then
//       SPANN::Index::SaveConfig): a folder that holds a head and its head-id file, for the SSD stage to run on.
//   spann_build_ref ssd <folder> <Float|Int8|Int16> <L2|Cosine> <n> <dim> <data file> <threads> [Section.Name=Value ...]
//       the same BuildIndex with SelectHead and BuildHead off: the SSD stage alone, from the head and the head-id file
//       already in <folder>.  Writes the posting files (and, with ExcludeHead false, the head-id file); <folder>/rng.txt
//       gets the RNG failed count ApproximateRNG logs (VectorIndex.cpp:984) and the stage's wall time in ms.
//   spann_build_ref heads <folder> <Float|Int8|Int16> <n> <dim> <data file> <K> <MaxCheck> <normalize 0/1> <out prefix>
//       VectorIndex::LoadIndex(<folder>/HeadIndex), MaxCheck set as SPANNIndex.cpp:901 sets it, then per row (normalised
//       first, as BasicVectorSet::Normalize does, when asked) the head's SearchIndex at K: <out>.ids / <out>.dists [n x K].
// The rows are raw row-major arrays of the value type.  Exit code 0 = every call succeeded.
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/Common/QueryResultSet.h"
#include "inc/Core/VectorIndex.h"
#include "inc/Helper/CommonHelper.h"
#include "inc/Helper/DiskIO.h"
#include "inc/Helper/Logging.h"

using namespace SPTAG;

static unsigned long long g_rng_failed = 0;

class QuietLogger : public Helper::Logger {
public:
    void Logging(const char*, Helper::LogLevel level, const char*, int, const char*, const char* format, ...) override {
        char buf[1024];
        va_list args;
        va_start(args, format);
        std::vsnprintf(buf, sizeof(buf), format, args);
        va_end(args);
        unsigned long long c = 0;
        if (std::sscanf(buf, "Searching replicas ended. RNG failed count: %llu", &c) == 1) g_rng_failed += c;
        if (level >= Helper::LogLevel::LL_Error) std::fputs(buf, stderr);
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
    if (vt == "Int8") return VectorValueType::Int8;
    if (vt == "Int16") return VectorValueType::Int16;
    return VectorValueType::Float;
}

static int build(int argc, char** argv, const std::string& mode) {
    const bool full = mode != "ssd";
    if (argc < 9) return 100;
    const std::string folder = argv[2], metric = argv[4], threads = argv[8];
    const VectorValueType type = value_type(argv[3]);
    const SizeType n = std::atoi(argv[5]);
    const DimensionType dim = std::atoi(argv[6]);
    const size_t bytes = (size_t)n * dim * GetValueTypeSize(type);
    std::vector<char> data;
    if (!read_all(argv[7], data, bytes)) return 101;
    std::shared_ptr<VectorIndex> idx = VectorIndex::CreateInstance(IndexAlgoType::SPANN, type);
    if (!idx) return 102;
    idx->SetParameter("IndexAlgoType", "BKT", "Base");
    idx->SetParameter("IndexDirectory", folder.c_str(), "Base");
    idx->SetParameter("DistCalcMethod", metric.c_str(), "Base");
    idx->SetParameter("isExecute", full ? "true" : "false", "SelectHead");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "SelectHead");
    idx->SetParameter("Ratio", "0.1", "SelectHead");
    idx->SetParameter("isExecute", full ? "true" : "false", "BuildHead");
    idx->SetParameter("RefineIterations", "3", "BuildHead");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "BuildHead");
    idx->SetParameter("isExecute", "true", "BuildSSDIndex");
    idx->SetParameter("BuildSsdIndex", "true", "BuildSSDIndex");
    idx->SetParameter("NumberOfThreads", threads.c_str(), "BuildSSDIndex");
    if (mode == "head") idx->SetParameter("BuildSsdIndex", "false", "BuildSSDIndex");
    for (int i = 9; i < argc; ++i) {
        const std::string kv = argv[i];
        const size_t dot = kv.find('.'), eq = kv.find('=');
        if (dot == std::string::npos || eq == std::string::npos || eq < dot) return 105;
        idx->SetParameter(kv.substr(dot + 1, eq - dot - 1).c_str(), kv.substr(eq + 1).c_str(), kv.substr(0, dot).c_str());
    }
    ByteArray arr = ByteArray::Alloc(bytes);
    std::memcpy(arr.Data(), data.data(), bytes);
    std::shared_ptr<VectorSet> vec(new BasicVectorSet(arr, type, dim, n));
    std::shared_ptr<MetadataSet> meta;
    const auto t0 = std::chrono::steady_clock::now();
    if (idx->BuildIndex(vec, meta) != ErrorCode::Success) return 103;
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (mode == "head") {
        auto ptr = f_createIO();
        if (!ptr || !ptr->Initialize((folder + "/indexloader.ini").c_str(), std::ios::out)) return 104;
        const std::string index = "[Index]\nIndexAlgoType=SPANN\nValueType=" + Helper::Convert::ConvertToString(type) + "\n\n";
        if (ptr->WriteString(index.c_str()) != index.size()) return 104;
        return idx->SaveConfig(ptr) == ErrorCode::Success ? 0 : 104;
    }
    if (full) return idx->SaveIndex(folder) == ErrorCode::Success ? 0 : 104;
    const std::string text = std::to_string(g_rng_failed) + " " + std::to_string(ms) + "\n";
    return write_all(folder + "/rng.txt", text.data(), text.size()) ? 0 : 106;
}

template <typename T>
static int heads_t(VectorIndex* head, std::vector<char>& data, SizeType n, DimensionType dim, int k, bool normalize,
                   const std::string& out) {
    T* rows = reinterpret_cast<T*>(data.data());
    if (normalize) {
        ByteArray arr((std::uint8_t*)rows, data.size(), false);
        BasicVectorSet(arr, GetEnumValueType<T>(), dim, n).Normalize(1);
    }
    std::vector<int> ids((size_t)n * k);
    std::vector<float> dists((size_t)n * k);
    for (SizeType i = 0; i < n; ++i) {
        QueryResult r(rows + (size_t)i * dim, k, false);
        if (head->SearchIndex(r) != ErrorCode::Success) return 112;
        for (int j = 0; j < k; ++j) {
            ids[(size_t)i * k + j] = r.GetResult(j)->VID;
            dists[(size_t)i * k + j] = r.GetResult(j)->Dist;
        }
    }
    return write_all(out + ".ids", ids.data(), ids.size() * 4) && write_all(out + ".dists", dists.data(), dists.size() * 4)
               ? 0
               : 113;
}

static int heads(int argc, char** argv) {
    if (argc < 11) return 100;
    const VectorValueType type = value_type(argv[3]);
    const SizeType n = std::atoi(argv[4]);
    const DimensionType dim = std::atoi(argv[5]);
    const int k = std::atoi(argv[7]);
    std::vector<char> data;
    if (!read_all(argv[6], data, (size_t)n * dim * GetValueTypeSize(type))) return 101;
    std::shared_ptr<VectorIndex> head;
    if (VectorIndex::LoadIndex(std::string(argv[2]) + "/HeadIndex", head) != ErrorCode::Success || !head) return 110;
    head->SetParameter("MaxCheck", argv[8]);
    const bool normalize = std::atoi(argv[9]) != 0;
    switch (type) {
    case VectorValueType::Int8: return heads_t<std::int8_t>(head.get(), data, n, dim, k, normalize, argv[10]);
    case VectorValueType::Int16: return heads_t<std::int16_t>(head.get(), data, n, dim, k, normalize, argv[10]);
    default: return heads_t<float>(head.get(), data, n, dim, k, normalize, argv[10]);
    }
}

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
    if (argc < 2) return 100;
    const std::string op = argv[1];
    if (op == "full" || op == "head" || op == "ssd") return build(argc, argv, op);
    if (op == "heads") return heads(argc, argv);
    return 100;
}
