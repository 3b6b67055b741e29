// TEST INFRASTRUCTURE.  EnableBfs through the drop-in SPTAG::B200::Index (sptag_b200/csrc/sptag_vector_index.hpp): a
// reference index with SetParameter("EnableBfs", ...) is wrapped by B200::Index::Attach, and its SearchIndex and
// ResultIterator results are compared bit for bit with an untouched reference index loaded from the same folder, before
// and after a SetParameter made through the wrapper after Attach.
//   compiled against /root/reference/AnnService headers, linked with oracle/_ref/libsptag_ref.so and
//   sptag_b200/lib/libsptag_b200.so (built like tests/cpp/vector_index_dropin).
// usage: bfs_dropin <index folder> <queries.bin> <nq> <k> <maxcheck>
// Exit code = number of failed checks; one line per check on stdout.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "inc/Core/VectorIndex.h"
#include "inc/Helper/Logging.h"
#include "inc/Core/ResultIterator.h"
#include "inc/Core/Common/QueryResultSet.h"

#include "../../sptag_b200/csrc/sptag_vector_index.hpp"

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

static int g_failed = 0;

static void report(const std::string& name, bool ok, const std::string& detail = "") {
    std::printf("%s %s %s\n", ok ? "PASS" : "FAIL", name.c_str(), detail.c_str());
    if (!ok) ++g_failed;
}

static bool same_result(const BasicResult& a, const BasicResult& b) {
    return a.VID == b.VID && std::memcmp(&a.Dist, &b.Dist, 4) == 0;
}

static size_t count_diff(const std::vector<BasicResult>& a, const std::vector<BasicResult>& b) {
    size_t d = 0;
    for (size_t i = 0; i < a.size(); ++i) d += same_result(a[i], b[i]) ? 0 : 1;
    return d;
}

// SearchIndex(batch) and ResultIterator::Next batches of `ref` and `gpu`; `tag` names the EnableBfs value
static void compare(VectorIndex* ref, VectorIndex* gpu, const std::vector<char>& q, size_t qsize, int nq, int k,
                    const std::string& tag) {
    const size_t n = (size_t)nq * k;
    std::vector<BasicResult> a(n), b(n);
    ref->SearchIndex(q.data(), nq, k, false, a.data());
    const ErrorCode ec = gpu->SearchIndex(q.data(), nq, k, false, b.data());
    report("SearchIndex(batch) " + tag, ec == ErrorCode::Success && count_diff(a, b) == 0,
           std::to_string(count_diff(a, b)) + " of " + std::to_string(n) + " results differ");
    size_t bad = 0;
    bool shape = true;
    for (int i = 0; i < nq && i < 24; ++i) {
        std::shared_ptr<ResultIterator> ia = ref->GetIterator(q.data() + (size_t)i * qsize, false);
        std::shared_ptr<ResultIterator> ib = gpu->GetIterator(q.data() + (size_t)i * qsize, false);
        if (!ia || !ib) {
            shape = false;
            continue;
        }
        const int batches[3] = {7, 7, 5};
        for (int r = 0; r < 3; ++r) {
            std::shared_ptr<QueryResult> ra = ia->Next(batches[r]), rb = ib->Next(batches[r]);
            if (ra->GetResultNum() != rb->GetResultNum() || ia->GetRelaxedMono() != ib->GetRelaxedMono()) {
                shape = false;
                continue;
            }
            for (int j = 0; j < ra->GetResultNum(); ++j) bad += same_result(*ra->GetResult(j), *rb->GetResult(j)) ? 0 : 1;
        }
        ia->Close();
        ib->Close();
    }
    report("ResultIterator::Next " + tag, shape && bad == 0, std::to_string(bad) + " results differ");
}

int main(int argc, char** argv) {
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s folder queries.bin nq k maxcheck\n", argv[0]);
        return 100;
    }
    const int nq = std::atoi(argv[3]), k = std::atoi(argv[4]);
    SetLogger(std::make_shared<QuietLogger>());
    std::shared_ptr<VectorIndex> cpu, ref, plain;
    if (VectorIndex::LoadIndex(argv[1], cpu) != ErrorCode::Success || !cpu) return 101;
    if (VectorIndex::LoadIndex(argv[1], ref) != ErrorCode::Success || !ref) return 101;
    if (VectorIndex::LoadIndex(argv[1], plain) != ErrorCode::Success || !plain) return 101;
    const size_t qsize = GetValueTypeSize(cpu->GetVectorValueType()) * (size_t)cpu->GetFeatureDim();
    std::vector<char> q((size_t)nq * qsize);
    FILE* f = std::fopen(argv[2], "rb");
    if (!f || std::fread(q.data(), 1, q.size(), f) != q.size()) return 102;
    std::fclose(f);

    // EnableBfs set on the reference index BEFORE it is wrapped: Attach must carry it to the device
    for (VectorIndex* x : {cpu.get(), ref.get(), plain.get()}) x->SetParameter("MaxCheck", argv[5]);
    cpu->SetParameter("EnableBfs", "2");
    ref->SetParameter("EnableBfs", "2");
    std::shared_ptr<VectorIndex> gpu = B200::Index::Attach(cpu, 0);
    if (!gpu) {
        std::fprintf(stderr, "B200::Index::Attach failed: %s\n", sptag_b200_last_error());
        return 104;
    }
    {   // the queries make the parameter matter: the default seeding gives other results at this budget
        const size_t n = (size_t)nq * k;
        std::vector<BasicResult> a(n), b(n);
        ref->SearchIndex(q.data(), nq, k, false, a.data());
        plain->SearchIndex(q.data(), nq, k, false, b.data());
        report("EnableBfs=2 changes the reference's results", count_diff(a, b) > 0,
               std::to_string(count_diff(a, b)) + " results differ from EnableBfs=0");
    }
    compare(ref.get(), gpu.get(), q, qsize, nq, k, "EnableBfs=2 (set before Attach)");
    // ... and set through the wrapper after Attach
    ref->SetParameter("EnableBfs", "-1");
    gpu->SetParameter("EnableBfs", "-1");
    compare(ref.get(), gpu.get(), q, qsize, nq, k, "EnableBfs=-1 (set after Attach)");
    ref->SetParameter("EnableBfs", "8");
    gpu->SetParameter("EnableBfs", "8");
    compare(ref.get(), gpu.get(), q, qsize, nq, k, "EnableBfs=8 (set after Attach)");
    std::printf("%d check(s) failed\n", g_failed);
    return g_failed;
}
