// The host-side rules of symphonia_b200/csrc/batch_call.h on the CPU, driven by tests/test_batch_call.py.
// One command per input line, one answer line each:
//   ranges <n_jobs> <k> (<first> <n>) x k     -> status of check_job_ranges
//   slots <n_allocated> <k> <slot> x k        -> status of check_slots
//   region <out_offset> <region> <out_samples> -> status of check_region
//   jobs <n_bytes> <k> (<offset> <len>) x k   -> 1 if jobs_in_bytes, else 0
//   merge <k> (<begin> <end>) x k             -> m, then (<begin> <end>) x m of merge_ranges
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "batch_call.h"

using namespace symgpu_detail;

namespace {

struct Job {
    uint64_t offset;
    uint32_t len;
};

uint64_t next() {
    unsigned long long v = 0;
    if (std::scanf("%llu", &v) != 1) std::exit(2);
    return v;
}

}  // namespace

int main() {
    char cmd[16];
    while (std::scanf("%15s", cmd) == 1) {
        if (!std::strcmp(cmd, "ranges")) {
            const uint64_t n_jobs = next(), k = next();
            std::vector<JobRange> r(k);
            for (JobRange& x : r) x.first = next(), x.n = next();
            std::printf("%d\n", int(check_job_ranges(r, n_jobs)));
        } else if (!std::strcmp(cmd, "slots")) {
            const uint64_t n = next(), k = next();
            std::vector<uint32_t> s(k);
            for (uint32_t& x : s) x = uint32_t(next());
            std::printf("%d\n", int(check_slots(s, n)));
        } else if (!std::strcmp(cmd, "region")) {
            const uint64_t off = next(), region = next(), cap = next();
            std::printf("%d\n", int(check_region(off, region, cap)));
        } else if (!std::strcmp(cmd, "jobs")) {
            const uint64_t n_bytes = next(), k = next();
            std::vector<Job> j(k);
            for (Job& x : j) x.offset = next(), x.len = uint32_t(next());
            std::printf("%d\n", int(jobs_in_bytes(j.data(), j.size(), n_bytes)));
        } else if (!std::strcmp(cmd, "merge")) {
            const uint64_t k = next();
            std::vector<ByteRange> r(k);
            for (ByteRange& x : r) x.begin = next(), x.end = next();
            const std::vector<ByteRange> m = merge_ranges(r);
            std::printf("%zu", m.size());
            for (const ByteRange& x : m) std::printf(" %zu %zu", x.begin, x.end);
            std::printf("\n");
        } else {
            return 2;
        }
    }
    return 0;
}
