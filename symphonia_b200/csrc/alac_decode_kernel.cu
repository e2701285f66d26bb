// ALAC decoded on the device, many files per call (include/symgpu.h "ALAC"; DESIGN §5h).
//
//   alac_slot_kernel      per job: checks its byte range and group, and its slot size (channels x slot samples)
//   scan                  slot sizes -> each job's place in the scratch planes and tail planes
//   alac_decode_kernel    one thread per packet: alac_entropy.h's decode_packet, the function the CPU front-end runs.  A
//                         packet's bitstream is serial (a CPE's second channel starts where the first one's residuals end),
//                         so one thread reads it all and writes each channel's record, residuals and tail bits
//   alac_predict_kernel   one thread per channel of a packet: predict_channel over its plane, coefficients in registers
//   scan by group         accepted frame counts -> each packet's first output frame within its file
//   alac_finish_kernel    one CTA per packet: finish_sample (mid/side, tail bits, the scale to 32 bits) for every sample,
//                         written as [frames][channels] of the caller's sample format in the file's region
//
// Only decode_packet can refuse a packet; a refused packet writes no frame.  One thread decodes a whole packet and one thread
// predicts a whole channel: latency-bound work, hidden by having many packets in flight -- the case this path is for.
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>
#include <type_traits>
#include <vector>

#include "alac_entropy.h"
#include "batch_call.h"
#include "int_sample.cuh"

using namespace symgpu_detail;
using symgpu::alac::Channel;

namespace {

__host__ __device__ inline bool group_ok(const symgpu_alac_group& g) {
    return g.channels >= 1 && g.channels <= 8 && g.bit_depth <= 32 && g.frame_length <= 65536;
}

__device__ __forceinline__ bool job_in_range(const symgpu_alac_job& j, const symgpu_alac_group* groups, size_t n_groups, size_t n_bytes,
                                             symgpu_alac_group& g) {
    if (j.offset > n_bytes || j.len > n_bytes - j.offset || j.group >= n_groups) return false;
    g = groups[j.group];
    return group_ok(g);
}

__global__ void __launch_bounds__(256) alac_slot_kernel(const symgpu_alac_job* __restrict__ jobs, uint32_t n_jobs, const symgpu_alac_group* __restrict__ groups,
                                                        size_t n_groups, size_t n_bytes, unsigned long long* __restrict__ sizes, uint32_t* __restrict__ keys) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const symgpu_alac_job j = jobs[k];
    symgpu_alac_group g;
    sizes[k] = job_in_range(j, groups, n_groups, n_bytes, g) ? (unsigned long long)g.channels * j.slot : 0;
    keys[k] = j.group;
}

__global__ void __launch_bounds__(128) alac_decode_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_alac_job* __restrict__ jobs, uint32_t n_jobs,
                                                          const symgpu_alac_group* __restrict__ groups, size_t n_groups, const unsigned long long* __restrict__ base,
                                                          Channel* __restrict__ recs, int32_t* __restrict__ samples, uint16_t* __restrict__ tails,
                                                          unsigned long long samples_cap, unsigned long long* __restrict__ accepted, uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const symgpu_alac_job j = jobs[k];
    symgpu_alac_group g;
    uint8_t st = SYMGPU_FLAC_JOB_INVALID;
    uint32_t frames = 0;
    if (job_in_range(j, groups, n_groups, n_bytes, g)) {
        const unsigned long long b = base[k], room = (unsigned long long)g.channels * j.slot;
        if (b <= samples_cap && room <= samples_cap - b) {
            const symgpu::alac::Config cfg{g.frame_length, g.bit_depth, g.pb, g.mb, g.kb, g.channels};
            const int r = symgpu::alac::decode_packet(bytes + j.offset, j.len, cfg, recs + size_t(k) * 8, samples + b, tails + b, j.slot, &frames);
            st = uint8_t(r);
            if (r != symgpu::alac::kDecoded) frames = 0;
        }
    }
    accepted[k] = frames;
    status[k] = st;
}

__global__ void __launch_bounds__(128) alac_predict_kernel(const symgpu_alac_job* __restrict__ jobs, uint32_t n_jobs, const symgpu_alac_group* __restrict__ groups,
                                                           const unsigned long long* __restrict__ base, const Channel* __restrict__ recs,
                                                           int32_t* __restrict__ samples, const uint8_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t k = i >> 3, c = i & 7;
    if (k >= n_jobs || status[k] != SYMGPU_FLAC_JOB_DECODED) return;
    const symgpu_alac_job j = jobs[k];
    if (c >= groups[j.group].channels) return;
    symgpu::alac::predict_channel(recs[size_t(k) * 8 + c], samples + base[k] + size_t(c) * j.slot);
}

template <int Format>
__global__ void __launch_bounds__(256) alac_finish_kernel(const symgpu_alac_job* __restrict__ jobs, uint32_t n_jobs, const symgpu_alac_group* __restrict__ groups,
                                                          size_t n_groups, const unsigned long long* __restrict__ base, const Channel* __restrict__ recs,
                                                          const int32_t* __restrict__ samples, const uint16_t* __restrict__ tails,
                                                          const uint8_t* __restrict__ status, const unsigned long long* __restrict__ accepted,
                                                          const unsigned long long* __restrict__ first, typename FlacSample<Format>::type* __restrict__ out,
                                                          unsigned long long out_cap, uint64_t* __restrict__ group_frames) {
    __shared__ Channel rec_s[8];
    const uint32_t k = blockIdx.x;
    const symgpu_alac_job j = jobs[k];
    const uint32_t gi = j.group;
    if (gi >= n_groups) return;
    // the last job of a group's run knows the group's frame count
    if (threadIdx.x == 0 && (k + 1 == n_jobs || jobs[k + 1].group != gi)) group_frames[gi] = first[k] + accepted[k];
    if (status[k] != SYMGPU_FLAC_JOB_DECODED) return;
    const symgpu_alac_group g = groups[gi];
    const unsigned ch = g.channels;
    const unsigned long long n = accepted[k], at = g.out_offset + first[k] * ch, count = n * ch;
    if (g.out_offset > out_cap || at > out_cap || count > out_cap - at) return;
    if (threadIdx.x < ch) rec_s[threadIdx.x] = recs[size_t(k) * 8 + threadIdx.x];
    __syncthreads();
    const int32_t* planes = samples + base[k];
    const uint16_t* tail = tails + base[k];
    // a packet has at most 65 536 frames of at most 8 channels: the element index and its divide fit 32 bits
    for (uint32_t i = threadIdx.x; i < uint32_t(count); i += blockDim.x) {
        const uint32_t t = i / ch;
        const unsigned c = i - t * ch;
        const Channel& r = rec_s[c];
        const int32_t s = symgpu::alac::finish_sample(r, planes + size_t(c) * j.slot, planes + size_t(r.partner) * j.slot, tail + size_t(c) * j.slot, t,
                                                      g.bit_depth);
        out[at + i] = FlacSample<Format>::from(s);
    }
}

cudaError_t scan_slots(void* temp, size_t& temp_bytes, const unsigned long long* sizes, unsigned long long* base, uint32_t n_jobs, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSum(temp, temp_bytes, sizes, base, int(n_jobs), st);
}
cudaError_t scan_first(void* temp, size_t& temp_bytes, const uint32_t* keys, const unsigned long long* accepted, unsigned long long* first, uint32_t n_jobs,
                       cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSumByKey(temp, temp_bytes, keys, accepted, first, int(n_jobs), cuda::std::equal_to<>(), st);
}

struct Scratch {
    size_t sizes, base, keys, accepted, first, recs, samples, tails, temp, total;
    size_t temp_bytes;
};

cudaError_t scratch_layout(uint32_t n_jobs, size_t out_cap, Scratch& s) {
    size_t t_slots = 0, t_first = 0;
    cudaError_t e = scan_slots(nullptr, t_slots, nullptr, nullptr, n_jobs, nullptr);
    if (e != cudaSuccess) return e;
    e = scan_first(nullptr, t_first, nullptr, nullptr, nullptr, n_jobs, nullptr);
    if (e != cudaSuccess) return e;
    s.temp_bytes = t_slots > t_first ? t_slots : t_first;
    Carver c;
    s.sizes = c.take(n_jobs * sizeof(unsigned long long));
    s.base = c.take(n_jobs * sizeof(unsigned long long));
    s.keys = c.take(n_jobs * sizeof(uint32_t));
    s.accepted = c.take(n_jobs * sizeof(unsigned long long));
    s.first = c.take(n_jobs * sizeof(unsigned long long));
    s.recs = c.take(size_t(n_jobs) * 8 * sizeof(Channel));
    s.samples = c.take(out_cap * sizeof(int32_t));
    s.tails = c.take(out_cap * sizeof(uint16_t));
    s.temp = c.take(s.temp_bytes);
    s.total = c.at;
    return cudaSuccess;
}

symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const uint8_t* bytes, size_t n_bytes, const symgpu_alac_job* jobs, uint32_t n_jobs,
                               const symgpu_alac_group* groups, size_t n_groups, int format, void* out, size_t out_cap, uint64_t* group_frames,
                               uint8_t* status) {
    char* stage = static_cast<char*>(ctx->d_stage);
    auto* sizes = reinterpret_cast<unsigned long long*>(stage + s.sizes);
    auto* base = reinterpret_cast<unsigned long long*>(stage + s.base);
    auto* keys = reinterpret_cast<uint32_t*>(stage + s.keys);
    auto* accepted = reinterpret_cast<unsigned long long*>(stage + s.accepted);
    auto* first = reinterpret_cast<unsigned long long*>(stage + s.first);
    auto* recs = reinterpret_cast<Channel*>(stage + s.recs);
    auto* samples = reinterpret_cast<int32_t*>(stage + s.samples);
    auto* tails = reinterpret_cast<uint16_t*>(stage + s.tails);
    void* temp = stage + s.temp;
    size_t temp_bytes = s.temp_bytes;
    cudaStream_t st = ctx->stream;
    alac_slot_kernel<<<(n_jobs + 255) / 256, 256, 0, st>>>(jobs, n_jobs, groups, n_groups, n_bytes, sizes, keys);
    CU(ctx, cudaGetLastError());
    CU(ctx, scan_slots(temp, temp_bytes, sizes, base, n_jobs, st));
    alac_decode_kernel<<<(n_jobs + 127) / 128, 128, 0, st>>>(bytes, n_bytes, jobs, n_jobs, groups, n_groups, base, recs, samples, tails, out_cap, accepted,
                                                             status);
    CU(ctx, cudaGetLastError());
    alac_predict_kernel<<<(n_jobs * 8 + 127) / 128, 128, 0, st>>>(jobs, n_jobs, groups, base, recs, samples, status);
    CU(ctx, cudaGetLastError());
    temp_bytes = s.temp_bytes;
    CU(ctx, scan_first(temp, temp_bytes, keys, accepted, first, n_jobs, st));
    auto finish = [&](auto fmt) {
        constexpr int F = decltype(fmt)::value;
        alac_finish_kernel<F><<<n_jobs, 256, 0, st>>>(jobs, n_jobs, groups, n_groups, base, recs, samples, tails, status, accepted, first,
                                                      static_cast<typename FlacSample<F>::type*>(out), out_cap, group_frames);
    };
    switch (format) {
    case SYMGPU_FMT_F32: finish(std::integral_constant<int, SYMGPU_FMT_F32>{}); break;
    case SYMGPU_FMT_S16: finish(std::integral_constant<int, SYMGPU_FMT_S16>{}); break;
    case SYMGPU_FMT_S24: finish(std::integral_constant<int, SYMGPU_FMT_S24>{}); break;
    case SYMGPU_FMT_S32: finish(std::integral_constant<int, SYMGPU_FMT_S32>{}); break;
    default: finish(std::integral_constant<int, SYMGPU_FMT_U8>{}); break;
    }
    CU(ctx, cudaGetLastError());
    ctx->launches += 8;  // four kernels and two per device-wide scan
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x0fffffff;  // eight channel records per job, and eight predict threads, are counted in 32 bits

}  // namespace

static_assert(sizeof(symgpu_alac_group) == 32 && sizeof(symgpu_alac_job) == 24, "record sizes are ABI");

extern "C" symgpu_status symgpu_alac_decode_fmt_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_alac_job* jobs, size_t n_jobs,
                                                    const symgpu_alac_group* groups, size_t n_groups, int format, void* out, size_t out_cap,
                                                    uint64_t* group_frames, uint8_t* status) {
    if (symgpu_sample_bytes(format) == 0) return SYMGPU_ERR_ARG;
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_cap, group_frames, status, kMaxJobs)) return SYMGPU_ERR_ARG;
    DeviceGuard guard(ctx->device);
    if (n_groups) CU(ctx, cudaMemsetAsync(group_frames, 0, n_groups * sizeof(uint64_t), ctx->stream));
    if (n_jobs == 0) return SYMGPU_OK;
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), out_cap, s));
    const symgpu_status e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    return decode_on_device(ctx, s, bytes, n_bytes, jobs, uint32_t(n_jobs), groups, n_groups, format, out, out_cap, group_frames, status);
}

extern "C" symgpu_status symgpu_alac_decode_fmt_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_alac_job* jobs, size_t n_jobs,
                                                     const symgpu_alac_group* groups, size_t n_groups, int format, void* out, size_t out_cap,
                                                     uint64_t* group_frames, uint8_t* status) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_cap, group_frames, status, kMaxJobs) ||
        !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    for (size_t g = 0; g < n_groups; ++g)
        if (!group_ok(groups[g]) || groups[g].out_offset > out_cap) return SYMGPU_ERR_ARG;
    std::vector<uint64_t> need(n_groups, 0);
    std::vector<uint8_t> seen(n_groups, 0);
    uint64_t total = 0;
    for (size_t k = 0; k < n_jobs; ++k) {
        const symgpu_alac_job& j = jobs[k];
        if (j.group >= n_groups) return SYMGPU_ERR_ARG;
        if (k == 0 || jobs[k - 1].group != j.group) {
            if (seen[j.group]) return SYMGPU_ERR_ARG;  // the group's jobs are not consecutive
            seen[j.group] = 1;
        }
        const uint64_t size = uint64_t(groups[j.group].channels) * j.slot;
        need[j.group] += size, total += size;
    }
    for (size_t g = 0; g < n_groups; ++g)
        if (check_region(groups[g].out_offset, need[g], out_cap) != SYMGPU_OK) return SYMGPU_ERR_LIMIT;
    if (total > out_cap) return SYMGPU_ERR_LIMIT;
    for (size_t g = 0; g < n_groups; ++g) group_frames[g] = 0;
    if (n_jobs == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), out_cap, s));
    return decode_from_host(
        ctx, s.total,
        std::array<HostIn, 3>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_alac_job)}, {groups, n_groups * sizeof(symgpu_alac_group)}}}, out,
        out_cap * sample, std::array<HostOut, 2>{{{status, n_jobs}, {group_frames, n_groups * sizeof(uint64_t)}}},
        [&](const std::array<void*, 3>& in, void* d_out, const std::array<void*, 2>& back) {
            uint64_t* d_frames = static_cast<uint64_t*>(back[1]);
            if (n_groups) CU(ctx, cudaMemsetAsync(d_frames, 0, n_groups * sizeof(uint64_t), ctx->stream));
            return decode_on_device(ctx, s, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_alac_job*>(in[1]), uint32_t(n_jobs),
                                    static_cast<const symgpu_alac_group*>(in[2]), n_groups, format, d_out, out_cap, d_frames,
                                    static_cast<uint8_t*>(back[0]));
        },
        [&] {
            std::vector<ByteRange> w;
            for (size_t g = 0; g < n_groups; ++g)
                w.push_back({size_t(groups[g].out_offset) * sample, size_t(groups[g].out_offset + group_frames[g] * groups[g].channels) * sample});
            return w;
        });
}
