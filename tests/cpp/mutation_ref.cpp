// TEST INFRASTRUCTURE.  Runs the unmodified reference's mutation calls on an index folder, so that
// tests/golden/make_golden_mutation.py can record what AddIndex / DeleteIndex produce.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage: mutation_ref <index folder> op...
//   set <Name> <Value>           VectorIndex::SetParameter
//   add <file> <num> <norm>      AddIndex(data, num, dim, nullptr, false, norm != 0)     (BKTIndex.cpp:902-970)
//   del <ids file> <num> <out>   DeleteIndex(id) per id; <out> gets one int32 ErrorCode per id (BKTIndex.cpp:893-899)
//   delvec <file> <num>          DeleteIndex(vectors, num) with one OpenMP thread           (BKTIndex.cpp:876-890)
//   save <folder>                SaveIndex(folder)
// Files are raw row-major arrays of the index's value type (ids: int32).  Exit code 0 = every call succeeded
// (del may return VectorNotFound; that is recorded, not an error).
#include <omp.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

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

static bool read_all(const char* path, std::vector<char>& out, size_t bytes) {
    out.resize(bytes);
    FILE* f = std::fopen(path, "rb");
    if (!f) return false;
    const bool ok = std::fread(out.data(), 1, bytes, f) == bytes;
    std::fclose(f);
    return ok;
}

int main(int argc, char** argv) {
    if (argc < 2) {
        std::fprintf(stderr, "usage: %s folder op...\n", argv[0]);
        return 100;
    }
    omp_set_num_threads(1);  // DeleteIndex(vectors): the single-thread order is the only one that is a function of the input
    SetLogger(std::make_shared<QuietLogger>());
    std::shared_ptr<VectorIndex> idx;
    if (VectorIndex::LoadIndex(argv[1], idx) != ErrorCode::Success || !idx) {
        std::fprintf(stderr, "reference LoadIndex failed\n");
        return 101;
    }
    const size_t row = GetValueTypeSize(idx->GetVectorValueType()) * (size_t)idx->GetFeatureDim();
    for (int a = 2; a < argc;) {
        const std::string op(argv[a]);
        if (op == "set" && a + 2 < argc) {
            if (idx->SetParameter(argv[a + 1], argv[a + 2]) != ErrorCode::Success) return 102;
            a += 3;
        } else if (op == "add" && a + 3 < argc) {
            const int num = std::atoi(argv[a + 2]);
            std::vector<char> data;
            if (!read_all(argv[a + 1], data, (size_t)num * row)) return 103;
            const ErrorCode rc = idx->AddIndex(data.data(), num, idx->GetFeatureDim(), nullptr, false, std::atoi(argv[a + 3]) != 0);
            if (rc != ErrorCode::Success) return 104;
            a += 4;
        } else if (op == "del" && a + 3 < argc) {
            const int num = std::atoi(argv[a + 2]);
            std::vector<char> data;
            if (!read_all(argv[a + 1], data, (size_t)num * 4)) return 105;
            std::vector<int> codes((size_t)num);
            for (int i = 0; i < num; ++i) {
                int id;
                std::memcpy(&id, data.data() + (size_t)i * 4, 4);
                codes[(size_t)i] = (int)idx->DeleteIndex((SizeType)id);
            }
            FILE* f = std::fopen(argv[a + 3], "wb");
            if (!f || std::fwrite(codes.data(), 4, codes.size(), f) != codes.size()) return 106;
            std::fclose(f);
            a += 4;
        } else if (op == "delvec" && a + 2 < argc) {
            const int num = std::atoi(argv[a + 2]);
            std::vector<char> data;
            if (!read_all(argv[a + 1], data, (size_t)num * row)) return 107;
            if (idx->DeleteIndex(data.data(), num) != ErrorCode::Success) return 108;
            a += 3;
        } else if (op == "save" && a + 1 < argc) {
            if (idx->SaveIndex(std::string(argv[a + 1])) != ErrorCode::Success) return 109;
            a += 2;
        } else {
            std::fprintf(stderr, "bad op %s\n", op.c_str());
            return 110;
        }
    }
    return 0;
}
