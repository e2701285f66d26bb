// Host-side pieces of the many-files-per-call device decoders (symgpu_<codec>_decode_host / _dev in *_decode_kernel.cu): the
// scratch carver, the argument and group rules they share, and the host variant's stage -> decode -> copy-back sequence
// (DESIGN §3b "The many-file calls").  Each codec keeps its own field checks, region formula, scratch and kernels.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <vector>

#include "ctx.h"

namespace symgpu_detail {

inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// Consecutive 256-byte aligned regions of a buffer: take(bytes) returns the next region's offset, `at` is the end so far.
struct Carver {
    size_t at = 0;
    size_t take(size_t bytes) {
        const size_t here = at;
        at += align256(bytes);
        return here;
    }
};

// The null / size rules every call shares (each codec adds its own): a non-empty array needs a pointer, and n_jobs <= max_jobs.
inline bool bad_batch_args(const symgpu_ctx* ctx, const void* bytes, size_t n_bytes, const void* jobs, size_t n_jobs, const void* groups, size_t n_groups,
                           const void* out, size_t out_bytes, const void* results, const void* status, size_t max_jobs) {
    return !ctx || (n_bytes && !bytes) || (n_jobs && (!jobs || !status)) || (n_groups && (!groups || !results)) || (out_bytes && !out) || n_jobs > max_jobs;
}

// Every job inside `bytes` (job records start with uint64 offset, uint32 len).
template <class Job>
bool jobs_in_bytes(const Job* jobs, size_t n_jobs, size_t n_bytes) {
    for (size_t k = 0; k < n_jobs; ++k)
        if (jobs[k].offset > n_bytes || jobs[k].len > n_bytes - jobs[k].offset) return false;
    return true;
}

struct JobRange {
    uint64_t first, n;
};

// SYMGPU_ERR_ARG unless every group's jobs lie inside the job table and no two non-empty groups share a job.
inline symgpu_status check_job_ranges(const std::vector<JobRange>& ranges, uint64_t n_jobs) {
    std::vector<JobRange> used;
    for (const JobRange& r : ranges) {
        if (r.first + r.n > n_jobs) return SYMGPU_ERR_ARG;
        if (r.n) used.push_back(r);
    }
    std::sort(used.begin(), used.end(), [](const JobRange& a, const JobRange& b) { return a.first < b.first; });
    for (size_t i = 1; i < used.size(); ++i)
        if (used[i - 1].first + used[i - 1].n > used[i].first) return SYMGPU_ERR_ARG;
    return SYMGPU_OK;
}

// State slots: SYMGPU_ERR_ARG when two groups name the same slot, else SYMGPU_ERR_LIMIT when one is not below n_allocated.
inline symgpu_status check_slots(std::vector<uint32_t> slots, uint64_t n_allocated) {
    std::sort(slots.begin(), slots.end());
    if (std::adjacent_find(slots.begin(), slots.end()) != slots.end()) return SYMGPU_ERR_ARG;
    if (!slots.empty() && slots.back() >= n_allocated) return SYMGPU_ERR_LIMIT;
    return SYMGPU_OK;
}

// SYMGPU_ERR_LIMIT unless samples [out_offset, out_offset + region) fit in out_samples (no overflow for any uint64 inputs).
inline symgpu_status check_region(uint64_t out_offset, uint64_t region, uint64_t out_samples) {
    return out_offset > out_samples || region > out_samples - out_offset ? SYMGPU_ERR_LIMIT : SYMGPU_OK;
}

struct ByteRange {
    size_t begin, end;
};

// The written ranges sorted, with empty ones dropped and ranges that touch or overlap merged: the fewest copies of their union.
inline std::vector<ByteRange> merge_ranges(std::vector<ByteRange> r) {
    r.erase(std::remove_if(r.begin(), r.end(), [](const ByteRange& x) { return x.end <= x.begin; }), r.end());
    std::sort(r.begin(), r.end(), [](const ByteRange& a, const ByteRange& b) { return a.begin < b.begin || (a.begin == b.begin && a.end < b.end); });
    std::vector<ByteRange> m;
    for (const ByteRange& x : r) {
        if (!m.empty() && x.begin <= m.back().end) m.back().end = std::max(m.back().end, x.end);
        else m.push_back(x);
    }
    return m;
}

// Each group's samples [out_offset, out_offset + frames * channels), in bytes, for result records with frames and channels.
template <class Group, class Result>
std::vector<ByteRange> written_by_results(const Group* groups, const Result* results, size_t n_groups, size_t sample_bytes) {
    std::vector<ByteRange> w;
    for (size_t g = 0; g < n_groups; ++g)
        w.push_back({size_t(groups[g].out_offset) * sample_bytes, size_t(groups[g].out_offset + results[g].frames * results[g].channels) * sample_bytes});
    return w;
}

struct HostIn {
    const void* p;
    size_t bytes;
};
struct HostOut {
    void* p;
    size_t bytes;
};

// The host variant after its checks: the stage holds the codec's scratch (scratch_bytes), then the inputs, `out` and the outputs,
// each 256-byte aligned.  The inputs are copied in, decode(d_in, d_out, d_back) runs on their device copies, the outputs come back
// into `back` (their host pointers), and after one wait only the byte ranges written(), computed from them, are copied into `out`.
template <size_t NI, size_t NB, class Decode, class Written>
symgpu_status decode_from_host(symgpu_ctx* ctx, size_t scratch_bytes, const std::array<HostIn, NI>& in, void* out, size_t out_bytes,
                               const std::array<HostOut, NB>& back, Decode&& decode, Written&& written) {
    Carver c{scratch_bytes};
    std::array<size_t, NI> o_in;
    std::array<size_t, NB> o_back;
    for (size_t i = 0; i < NI; ++i) o_in[i] = c.take(in[i].bytes);
    const size_t o_out = c.take(out_bytes);
    for (size_t i = 0; i < NB; ++i) o_back[i] = c.take(back[i].bytes);
    const symgpu_status e = ensure_stage(ctx, c.at);
    if (e != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    std::array<void*, NI> d_in;
    std::array<void*, NB> d_back;
    for (size_t i = 0; i < NI; ++i) {
        d_in[i] = stage + o_in[i];
        if (in[i].bytes) CU(ctx, cudaMemcpyAsync(d_in[i], in[i].p, in[i].bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    for (size_t i = 0; i < NB; ++i) d_back[i] = stage + o_back[i];
    char* d_out = stage + o_out;
    const symgpu_status d = decode(d_in, static_cast<void*>(d_out), d_back);
    if (d != SYMGPU_OK) return d;
    for (size_t i = 0; i < NB; ++i)
        if (back[i].bytes) CU(ctx, cudaMemcpyAsync(back[i].p, d_back[i], back[i].bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (const ByteRange& r : merge_ranges(written()))
        CU(ctx, cudaMemcpyAsync(static_cast<char*>(out) + r.begin, d_out + r.begin, r.end - r.begin, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return SYMGPU_OK;
}

}  // namespace symgpu_detail
