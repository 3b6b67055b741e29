// TEST INFRASTRUCTURE.  Runs MultiIndexScan with the unmodified reference, so that tests/golden/make_golden_multi_scan.py
// can record what Init + Next return, and tools/multi_scan_bench.py can time it.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so only.
// usage:
//   multi_scan_ref <nq> <out prefix> <k> <term_cond> <search_limit> <weights> <stream_len> <threads>
//                  <folder_0> <queries_0> [<folder_1> <queries_1> ...]
//       VectorIndex::LoadIndex(folder_i) for every index; per query a fresh MultiIndexScan, Init(indexes, targets,
//       weights, k, useTimer = false, term_cond, search_limit) -- or, with weights "sum", the constructor with the
//       reference's rankFunc -- then Next until it returns false:
//         <out>.ids [nq x k] int32, <out>.scores [nq x k] float32 (unfilled: -1, MaxDist), <out>.counts [nq] int32.
//       weights: comma-separated floats, one per index.  stream_len > 0 also records each index's own iterator
//       (GetIterator(target, true), Next(1) up to stream_len times, stopping at the first empty call):
//         <out>.sids / <out>.sdists [indexes x nq x stream_len] (-1, MaxDist after the end), <out>.slen [indexes x nq].
//       threads > 1 runs the queries in parallel; <out>.ms gets the wall time of the scan loop.
// Queries are raw row-major arrays of the index's value type.  Exit code 0 = success.
#include <omp.h>

#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/MultiIndexScan.h"
#include "inc/Core/ResultIterator.h"
#include "inc/Core/SearchQuery.h"
#include "inc/Core/VectorIndex.h"
#include "inc/Helper/Logging.h"

using namespace SPTAG;

namespace SPTAG {
float rankFunc(std::vector<float> in);  // MultiIndexScan.cpp:37-39, the constructor's sum
}

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

static size_t value_bytes(VectorValueType t) {
    switch (t) {
    case VectorValueType::Int8:
    case VectorValueType::UInt8: return 1;
    case VectorValueType::Int16: return 2;
    default: return 4;
    }
}

int main(int argc, char** argv) {
    SetLogger(std::make_shared<QuietLogger>());
    if (argc < 11 || (argc - 9) % 2 != 0) return 100;
    // MultiIndexScan prints its progress with printf
    if (!std::freopen("/dev/null", "w", stdout)) return 100;
    const int nq = std::atoi(argv[1]);
    const std::string out = argv[2];
    const int k = std::atoi(argv[3]);
    const int term_cond = std::atoi(argv[4]);
    const int search_limit = std::atoi(argv[5]);
    const std::string wspec = argv[6];
    const int stream_len = std::atoi(argv[7]);
    const int threads = std::atoi(argv[8]);
    const int n = (argc - 9) / 2;
    std::vector<std::shared_ptr<VectorIndex>> indexes(n);
    std::vector<std::vector<char>> qbuf(n);
    std::vector<size_t> row(n);
    for (int i = 0; i < n; ++i) {
        if (VectorIndex::LoadIndex(argv[9 + 2 * i], indexes[i]) != ErrorCode::Success || !indexes[i]) return 110;
        row[i] = (size_t)indexes[i]->GetFeatureDim() * value_bytes(indexes[i]->GetVectorValueType());
        if (!read_all(argv[10 + 2 * i], qbuf[i], (size_t)nq * row[i])) return 101;
    }
    const bool sum = wspec == "sum";
    std::vector<float> weights;
    if (!sum)
        for (const char* c = wspec.c_str(); *c;) {
            weights.push_back((float)std::atof(c));
            while (*c && *c != ',') ++c;
            if (*c == ',') ++c;
        }
    if (!sum && (int)weights.size() != n) return 102;
    std::vector<int> ids((size_t)nq * k, -1), counts(nq, 0);
    std::vector<float> scores((size_t)nq * k, MaxDist);
    omp_set_num_threads(threads > 1 ? threads : 1);
    const auto t0 = std::chrono::steady_clock::now();
#pragma omp parallel for schedule(dynamic, 4)
    for (int q = 0; q < nq; ++q) {
        std::unique_ptr<MultiIndexScan> scan;
        if (sum) {
            std::vector<void*> targets(n);
            for (int i = 0; i < n; ++i) targets[i] = qbuf[i].data() + (size_t)q * row[i];
            scan.reset(new MultiIndexScan(indexes, targets, (unsigned)k, rankFunc, false, term_cond, search_limit));
        } else {
            std::vector<ByteArray> targets;
            for (int i = 0; i < n; ++i)
                targets.push_back(ByteArray((std::uint8_t*)qbuf[i].data() + (size_t)q * row[i], row[i], false));
            scan.reset(new MultiIndexScan());
            scan->Init(indexes, targets, weights, (unsigned)k, false, term_cond, search_limit);
        }
        BasicResult r;
        int c = 0;
        while (c < k && scan->Next(r)) {
            ids[(size_t)q * k + c] = r.VID;
            scores[(size_t)q * k + c] = r.Dist;
            ++c;
        }
        counts[q] = c;
    }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    bool ok = write_all(out + ".ids", ids.data(), ids.size() * 4) && write_all(out + ".scores", scores.data(), scores.size() * 4) &&
              write_all(out + ".counts", counts.data(), counts.size() * 4) && write_all(out + ".ms", &ms, sizeof(ms));
    if (ok && stream_len > 0) {
        const size_t total = (size_t)n * nq * stream_len;
        std::vector<int> sids(total, -1), slen((size_t)n * nq, 0);
        std::vector<float> sdists(total, MaxDist);
#pragma omp parallel for schedule(dynamic, 4)
        for (int q = 0; q < nq; ++q)
            for (int i = 0; i < n; ++i) {
                std::shared_ptr<ResultIterator> it = indexes[i]->GetIterator(qbuf[i].data() + (size_t)q * row[i], true);
                const size_t at = ((size_t)i * nq + q) * stream_len;
                int c = 0;
                for (; c < stream_len; ++c) {
                    std::shared_ptr<QueryResult> res = it->Next(1);
                    if (res->GetResultNum() == 0) break;
                    sids[at + c] = res->GetResult(0)->VID;
                    sdists[at + c] = res->GetResult(0)->Dist;
                }
                slen[(size_t)i * nq + q] = c;
                it->Close();
            }
        ok = write_all(out + ".sids", sids.data(), total * 4) && write_all(out + ".sdists", sdists.data(), total * 4) &&
             write_all(out + ".slen", slen.data(), slen.size() * 4);
    }
    return ok ? 0 : 113;
}
