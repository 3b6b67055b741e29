// TEST INFRASTRUCTURE.  Runs SPANN iterators with the unmodified reference, so that
// tests/golden/make_golden_spann_iterator.py can record what SPANN::Index<T>::GetIterator + ResultIterator::Next return.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage:
//   spann_iter_ref <folder> <queries file> <nq> <out prefix> <b0,b1,...> [<threads>]
//       VectorIndex::LoadIndex(folder) (every parameter comes from the folder's indexloader.ini), then per query
//       GetIterator and Next(b) for each b of the schedule (SPANNResultIterator.h:37-63):
//         <out>.counts [calls x nq] int32 resultNum, <out>.relaxed [calls x nq] uint8 GetRelaxedMono(),
//         <out>.ids / .dists: per call c one [nq x b_c] block, the first resultNum results then (-1, MaxDist).
//       threads > 1 runs the queries in parallel (tools/spann_iterator_bench.py); <out>.ms gets the wall time of that loop.
// Queries are raw row-major arrays of the index's value type.  Exit code 0 = every call succeeded.
#include <omp.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/ResultIterator.h"
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

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
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
    const int threads = argc > 6 ? std::atoi(argv[6]) : 1;
    const size_t row = (size_t)index->GetFeatureDim() * (index->GetVectorValueType() == VectorValueType::Int8 ? 1 : 4);
    std::vector<char> qbuf;
    if (!read_all(argv[2], qbuf, (size_t)nq * row)) return 101;
    std::vector<size_t> at(schedule.size() + 1, 0);  // where call c's [nq x b_c] block starts
    for (size_t c = 0; c < schedule.size(); ++c) at[c + 1] = at[c] + (size_t)nq * schedule[c];
    std::vector<int> ids(at.back()), counts(schedule.size() * nq);
    std::vector<float> dists(at.back());
    std::vector<unsigned char> relaxed(schedule.size() * nq);
    int bad = 0;
    omp_set_num_threads(threads > 1 ? threads : 1);
    const auto t0 = std::chrono::steady_clock::now();
#pragma omp parallel for schedule(dynamic, 16) reduction(+ : bad)
    for (int i = 0; i < nq; ++i) {
        std::shared_ptr<ResultIterator> it = index->GetIterator(qbuf.data() + (size_t)i * row);
        if (!it) {
            ++bad;
            continue;
        }
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
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (bad) return 112;
    const bool ok = write_all(out + ".ids", ids.data(), ids.size() * 4) && write_all(out + ".dists", dists.data(), dists.size() * 4) &&
                    write_all(out + ".counts", counts.data(), counts.size() * 4) &&
                    write_all(out + ".relaxed", relaxed.data(), relaxed.size()) && write_all(out + ".ms", &ms, sizeof(ms));
    return ok ? 0 : 113;
}
