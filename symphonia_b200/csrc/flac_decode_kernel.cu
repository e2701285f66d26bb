// FLAC decoded on the device, many files per launch (include/symgpu.h "FLAC decoded on the device"; DESIGN §5e).
//
//   flac_slot_kernel         per job: checks its byte range and group, and its slot size (channels x slot samples)
//   scan                     slot sizes -> each job's place in the scratch planes and in the sub-frame table
//   flac_decode_kernel       one thread per packet: flac_entropy.h's decode_packet, the very function the CPU front-end
//                            runs, writes the frame record, its sub-frame records and the warm-up samples / residuals
//   flac_launch              prediction + decorrelation + scaling (flac_kernel.cu, unchanged) over all jobs' records
//   scan by group            accepted block sizes -> each frame's first output frame within its file
//   flac_interleave_kernel   one CTA per packet: the restored planes -> [frames][channels] of the caller's sample format in
//                            the file's region (one instantiation per SYMGPU_FMT_*, chosen once on the host)
//
// A refused packet keeps neutral records: a frame with 0 channels (flac_finish_kernel returns at once) and sub-frames
// with n = 0 (flac_predict_kernel leaves them alone), so the restoration kernels run on every job unchanged.
//
// A frame carries no state into the next one, so a packet is an independent job.  One thread decodes one whole frame
// serially: latency-bound work, hidden by having many packets in flight -- the case this path is for (many files).
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>
#include <type_traits>
#include <vector>

#include "batch_call.h"
#include "flac_entropy.h"
#include "flac_kernel.h"
#include "int_sample.cuh"

using namespace symgpu_detail;

namespace {

struct Slot {
    unsigned long long samples, subs;
};
struct SlotSum {
    __host__ __device__ Slot operator()(const Slot& a, const Slot& b) const { return Slot{a.samples + b.samples, a.subs + b.subs}; }
};

__device__ __forceinline__ bool job_in_range(const symgpu_flac_job& j, const symgpu_flac_group* groups, size_t n_groups, size_t n_bytes,
                                             symgpu_flac_group& g) {
    if (j.offset > n_bytes || j.len > n_bytes - j.offset || j.group >= n_groups) return false;
    g = groups[j.group];
    return g.channels >= 1 && g.channels <= 8;
}

__global__ void __launch_bounds__(256) flac_slot_kernel(const symgpu_flac_job* __restrict__ jobs, uint32_t n_jobs, const symgpu_flac_group* __restrict__ groups,
                                                        size_t n_groups, size_t n_bytes, Slot* __restrict__ sizes, uint32_t* __restrict__ keys) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const symgpu_flac_job j = jobs[k];
    symgpu_flac_group g;
    const bool ok = job_in_range(j, groups, n_groups, n_bytes, g);
    sizes[k] = ok ? Slot{(unsigned long long)g.channels * j.slot, g.channels} : Slot{0, 0};
    keys[k] = j.group;
}

__global__ void __launch_bounds__(128) flac_decode_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_flac_job* __restrict__ jobs, uint32_t n_jobs,
                                                          const symgpu_flac_group* __restrict__ groups, size_t n_groups, const Slot* __restrict__ base,
                                                          symgpu_flac_frame* __restrict__ frames, symgpu_flac_subframe* __restrict__ subs,
                                                          int32_t* __restrict__ samples, unsigned long long samples_cap, unsigned long long* __restrict__ accepted,
                                                          uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const symgpu_flac_job j = jobs[k];
    symgpu_flac_group g;
    uint8_t st = SYMGPU_FLAC_JOB_INVALID;
    unsigned long long block = 0;
    symgpu_flac_frame fr{};
    if (job_in_range(j, groups, n_groups, n_bytes, g)) {
        const Slot b = base[k];
        const unsigned long long room = (unsigned long long)g.channels * j.slot;
        if (b.samples <= samples_cap && room <= samples_cap - b.samples) {
            symgpu_flac_frame_info info;
            const int r = symgpu::flace::decode_packet(bytes + j.offset, j.len, g.bits_per_sample, g.channels, g.max_block, uint32_t(b.subs), subs + b.subs,
                                                       g.channels, samples + b.samples, b.samples, room, j.slot, &fr, &info);
            if (r == symgpu::flace::kDecoded) {
                st = SYMGPU_FLAC_JOB_DECODED, block = info.block_size;
            } else {
                st = r == symgpu::flace::kNoRoom ? SYMGPU_FLAC_JOB_NO_ROOM : SYMGPU_FLAC_JOB_REFUSED;
                fr = symgpu_flac_frame{};
                for (uint32_t c = 0; c < g.channels; ++c) subs[b.subs + c].n = 0;  // what a refused packet read stays out of the restoration
            }
        }
    }
    frames[k] = fr;
    accepted[k] = block;
    status[k] = st;
}

template <int Format>
__global__ void __launch_bounds__(256) flac_interleave_kernel(const symgpu_flac_job* __restrict__ jobs, uint32_t n_jobs, const symgpu_flac_group* __restrict__ groups,
                                                              size_t n_groups, const symgpu_flac_frame* __restrict__ frames,
                                                              const symgpu_flac_subframe* __restrict__ subs, const int32_t* __restrict__ samples,
                                                              const uint8_t* __restrict__ status, const unsigned long long* __restrict__ accepted,
                                                              const unsigned long long* __restrict__ first, typename FlacSample<Format>::type* __restrict__ out,
                                                              unsigned long long out_cap, uint64_t* __restrict__ group_frames) {
    __shared__ unsigned long long plane_s[8];
    const uint32_t k = blockIdx.x;
    const uint32_t gi = jobs[k].group;
    if (gi >= n_groups) return;
    // the last job of a group's run knows the group's frame count
    if (threadIdx.x == 0 && (k + 1 == n_jobs || jobs[k + 1].group != gi)) group_frames[gi] = first[k] + accepted[k];
    if (status[k] != SYMGPU_FLAC_JOB_DECODED) return;
    const symgpu_flac_group g = groups[gi];
    const symgpu_flac_frame fr = frames[k];
    const unsigned ch = g.channels, have = fr.channels;
    const unsigned long long n = accepted[k], at = g.out_offset + first[k] * ch, count = n * ch;
    if (g.out_offset > out_cap || at > out_cap || count > out_cap - at) return;
    if (threadIdx.x < have) plane_s[threadIdx.x] = subs[fr.first_subframe + threadIdx.x].offset;
    __syncthreads();
    // a block has at most 65 536 samples in at most 8 channels: the element index and its divide fit 32 bits
    for (uint32_t i = threadIdx.x; i < uint32_t(count); i += blockDim.x) {
        const uint32_t t = i / ch;
        const unsigned c = i - t * ch;
        out[at + i] = FlacSample<Format>::from(c < have ? samples[plane_s[c] + t] : 0);
    }
}

// The two device-wide scans; the size query (temp == nullptr) and the run go through the same instantiation.
cudaError_t scan_slots(void* temp, size_t& temp_bytes, const Slot* sizes, Slot* base, uint32_t n_jobs, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveScan(temp, temp_bytes, sizes, base, SlotSum(), Slot{0, 0}, int(n_jobs), st);
}
cudaError_t scan_first(void* temp, size_t& temp_bytes, const uint32_t* keys, const unsigned long long* accepted, unsigned long long* first, uint32_t n_jobs,
                       cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSumByKey(temp, temp_bytes, keys, accepted, first, int(n_jobs), cuda::std::equal_to<>(), st);
}

// The device variant's scratch at the start of ctx->d_stage.
struct Scratch {
    size_t sizes, keys, accepted, first, base, frames, subs, samples, temp, total;
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
    s.sizes = c.take(n_jobs * sizeof(Slot));
    s.base = c.take(n_jobs * sizeof(Slot));
    s.keys = c.take(n_jobs * sizeof(uint32_t));
    s.accepted = c.take(n_jobs * sizeof(unsigned long long));
    s.first = c.take(n_jobs * sizeof(unsigned long long));
    s.frames = c.take(n_jobs * sizeof(symgpu_flac_frame));
    s.subs = c.take(size_t(n_jobs) * 8 * sizeof(symgpu_flac_subframe));
    s.samples = c.take(out_cap * sizeof(int32_t));
    s.temp = c.take(s.temp_bytes);
    s.total = c.at;
    return cudaSuccess;
}

// Everything after the staging: device pointers, n_jobs > 0, a format symgpu_sample_bytes knows, ctx->d_stage holds `s`.
symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const uint8_t* bytes, size_t n_bytes, const symgpu_flac_job* jobs, uint32_t n_jobs,
                               const symgpu_flac_group* groups, size_t n_groups, int format, void* out, size_t out_cap, uint64_t* group_frames,
                               uint8_t* status) {
    char* stage = static_cast<char*>(ctx->d_stage);
    Slot* sizes = reinterpret_cast<Slot*>(stage + s.sizes);
    Slot* base = reinterpret_cast<Slot*>(stage + s.base);
    uint32_t* keys = reinterpret_cast<uint32_t*>(stage + s.keys);
    unsigned long long* accepted = reinterpret_cast<unsigned long long*>(stage + s.accepted);
    unsigned long long* first = reinterpret_cast<unsigned long long*>(stage + s.first);
    symgpu_flac_frame* frames = reinterpret_cast<symgpu_flac_frame*>(stage + s.frames);
    symgpu_flac_subframe* subs = reinterpret_cast<symgpu_flac_subframe*>(stage + s.subs);
    int32_t* samples = reinterpret_cast<int32_t*>(stage + s.samples);
    void* temp = stage + s.temp;
    size_t temp_bytes = s.temp_bytes;
    cudaStream_t st = ctx->stream;
    const unsigned per = 256, grid = (n_jobs + per - 1) / per;
    CU(ctx, cudaMemsetAsync(subs, 0, size_t(n_jobs) * 8 * sizeof(symgpu_flac_subframe), st));  // records no packet claims stay neutral
    flac_slot_kernel<<<grid, per, 0, st>>>(jobs, n_jobs, groups, n_groups, n_bytes, sizes, keys);
    CU(ctx, cudaGetLastError());
    CU(ctx, scan_slots(temp, temp_bytes, sizes, base, n_jobs, st));
    flac_decode_kernel<<<(n_jobs + 127) / 128, 128, 0, st>>>(bytes, n_bytes, jobs, n_jobs, groups, n_groups, base, frames, subs, samples, out_cap, accepted, status);
    CU(ctx, cudaGetLastError());
    CU(ctx, symgpu::flac_launch(frames, n_jobs, subs, n_jobs * 8, samples, out_cap, st));
    temp_bytes = s.temp_bytes;
    CU(ctx, scan_first(temp, temp_bytes, keys, accepted, first, n_jobs, st));
    auto interleave = [&](auto fmt) {
        constexpr int F = decltype(fmt)::value;
        flac_interleave_kernel<F><<<n_jobs, 256, 0, st>>>(jobs, n_jobs, groups, n_groups, frames, subs, samples, status, accepted, first,
                                                          static_cast<typename FlacSample<F>::type*>(out), out_cap, group_frames);
    };
    switch (format) {
    case SYMGPU_FMT_F32: interleave(std::integral_constant<int, SYMGPU_FMT_F32>{}); break;
    case SYMGPU_FMT_S16: interleave(std::integral_constant<int, SYMGPU_FMT_S16>{}); break;
    case SYMGPU_FMT_S24: interleave(std::integral_constant<int, SYMGPU_FMT_S24>{}); break;
    case SYMGPU_FMT_S32: interleave(std::integral_constant<int, SYMGPU_FMT_S32>{}); break;
    default: interleave(std::integral_constant<int, SYMGPU_FMT_U8>{}); break;
    }
    CU(ctx, cudaGetLastError());
    ctx->launches += 9;  // three kernels here, predict + finish, and two per device-wide scan
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x1fffffff;  // eight sub-frame records per job are counted in 32 bits

}  // namespace

extern "C" symgpu_status symgpu_flac_decode_fmt_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_flac_job* jobs, size_t n_jobs,
                                                    const symgpu_flac_group* groups, size_t n_groups, int format, void* out, size_t out_cap,
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

extern "C" symgpu_status symgpu_flac_decode_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_flac_job* jobs, size_t n_jobs,
                                                const symgpu_flac_group* groups, size_t n_groups, int32_t* out, size_t out_cap, uint64_t* group_frames,
                                                uint8_t* status) {
    return symgpu_flac_decode_fmt_dev(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, SYMGPU_FMT_S32, out, out_cap, group_frames, status);
}

extern "C" symgpu_status symgpu_flac_decode_fmt_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_flac_job* jobs, size_t n_jobs,
                                                     const symgpu_flac_group* groups, size_t n_groups, int format, void* out, size_t out_cap,
                                                     uint64_t* group_frames, uint8_t* status) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_cap, group_frames, status, kMaxJobs) ||
        !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    for (size_t g = 0; g < n_groups; ++g)
        if (groups[g].channels < 1 || groups[g].channels > 8 || groups[g].bits_per_sample > 32 || groups[g].out_offset > out_cap) return SYMGPU_ERR_ARG;
    std::vector<uint64_t> need(n_groups, 0);
    std::vector<uint8_t> seen(n_groups, 0);
    uint64_t total = 0;
    for (size_t k = 0; k < n_jobs; ++k) {
        const symgpu_flac_job& j = jobs[k];
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
        std::array<HostIn, 3>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_flac_job)}, {groups, n_groups * sizeof(symgpu_flac_group)}}}, out,
        out_cap * sample, std::array<HostOut, 2>{{{status, n_jobs}, {group_frames, n_groups * sizeof(uint64_t)}}},
        [&](const std::array<void*, 3>& in, void* d_out, const std::array<void*, 2>& back) {
            uint64_t* d_frames = static_cast<uint64_t*>(back[1]);
            if (n_groups) CU(ctx, cudaMemsetAsync(d_frames, 0, n_groups * sizeof(uint64_t), ctx->stream));
            return decode_on_device(ctx, s, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_flac_job*>(in[1]), uint32_t(n_jobs),
                                    static_cast<const symgpu_flac_group*>(in[2]), n_groups, format, d_out, out_cap, d_frames,
                                    static_cast<uint8_t*>(back[0]));
        },
        [&] {
            std::vector<ByteRange> w;
            for (size_t g = 0; g < n_groups; ++g)
                w.push_back({size_t(groups[g].out_offset) * sample, size_t(groups[g].out_offset + group_frames[g] * groups[g].channels) * sample});
            return w;
        });
}

extern "C" symgpu_status symgpu_flac_decode_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_flac_job* jobs, size_t n_jobs,
                                                 const symgpu_flac_group* groups, size_t n_groups, int32_t* out, size_t out_cap, uint64_t* group_frames,
                                                 uint8_t* status) {
    return symgpu_flac_decode_fmt_host(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, SYMGPU_FMT_S32, out, out_cap, group_frames, status);
}
