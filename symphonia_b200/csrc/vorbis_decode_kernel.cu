// Ogg Vorbis decoded on the device, many files per call (include/symgpu.h "Ogg Vorbis decoded on the device"; DESIGN §5f).
// A file is a group, an audio packet is a job.  The packet rules are those of vorbis_entropy.h, the code the CPU front-end runs.
//
//   (host)                 every distinct setup built once (symgpu_vorbis_fe_create) and flattened; one stream per group and
//                          every setup's floors once registered with the context
//   vorbis_key_kernel      one CTA per group: names the group of each of its jobs
//   vorbis_packet_kernel   one thread per job: decode_packet with a fresh partition-class buffer -> the job's unit, floor_y
//                          [2][65], residue [2][row] (zeroed beforehand by one memset of all jobs' rows, so no thread clears
//                          a row the call's longest block size dictates); its status and block flag
//   scan by group          over (decoded, block flag): each decoded packet's rank among its file's decoded packets and the block
//                          flag of the decoded packet before it
//   vorbis_span_kernel     one thread per job: prev_block_flag, frames = (prev_n + n) / 4, the trims, the frames that survive
//   scan by group          exclusive sum of the surviving frames: the packet's first output frame
//   vorbis_place_kernel    one CTA per job: the decoded packets into their group's first frame slots in stream order, muted
//                          records into the slots behind them; pack spans, group results
//   symgpu_vorbis_synth_dev (every group one run of n_jobs packets), symgpu_pcm_pack_dev (mono, stereo)
//
// Frame slots: a group owns n_jobs consecutive slots.  A muted slot has both floors unused (0xffff), do_not_decode set and a
// zero residue; the synthesis runs those after the group's real packets and the pack stage writes nothing for them.
#include <cuda_runtime.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>
#include <vector>

#include "batch_call.h"
#include "pack_kernel.h"
#include "vorbis_entropy.h"

using namespace symgpu_detail;
namespace ve = symgpu::vorbise;

namespace {

constexpr uint32_t kNone = 0xffffffffu;

struct DevGroup {  // symgpu_vorbis_group + where its slots, class buffers and floors start
    uint64_t out_offset;
    uint64_t frame_base;
    uint64_t class_base;
    uint32_t first_job, n_jobs, setup, floor_base, channels, bs0_exp, bs1_exp, class_cap;
};

struct Acc {  // decoded packets so far, block flag of the last of them (-1: none)
    uint32_t count;
    int32_t flag;
};
struct AccOp {
    __host__ __device__ Acc operator()(const Acc& a, const Acc& b) const { return Acc{a.count + b.count, b.flag >= 0 ? b.flag : a.flag}; }
};

struct Span {  // what vorbis_span_kernel computes for a decoded packet
    uint32_t frames, trim_start, trim_end, reserved;
};

// Per-job scratch (one array each, indexed by job).
struct JobBufs {
    symgpu_vorbis_unit* units;
    uint16_t* floor_y;  // [130]
    float* residue;     // [2][row]
    uint8_t* classes;   // class_cap bytes per job, from the group's class_base
    Acc* acc_in;
    Acc* acc;
    Span* span;
    unsigned long long* left;
    unsigned long long* first;
};

__global__ void __launch_bounds__(128) vorbis_key_kernel(const DevGroup* __restrict__ groups, uint32_t* __restrict__ keys) {
    const DevGroup g = groups[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < g.n_jobs; i += blockDim.x) keys[g.first_job + i] = blockIdx.x;
}

__global__ void __launch_bounds__(128) vorbis_packet_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_vorbis_job* __restrict__ jobs,
                                                            uint32_t n_jobs, const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys,
                                                            const uint8_t* __restrict__ blob, const ve::SetupHead* __restrict__ heads, uint32_t row,
                                                            JobBufs B, uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    Acc a{0, -1};
    if (gi != kNone) {
        const symgpu_vorbis_job j = jobs[k];
        if (j.offset > n_bytes || j.len > n_bytes - j.offset) {
            status[k] = SYMGPU_VORBIS_JOB_INVALID;
        } else {
            const DevGroup g = groups[gi];
            const ve::Setup S = ve::view_of(blob, heads[g.setup]);
            ve::ClassBuf cls{B.classes + g.class_base + uint64_t(k - g.first_job) * g.class_cap, 0, g.class_cap};
            symgpu_vorbis_unit* u = B.units + k;
            const symgpu_status st = ve::decode_packet(S, bytes + j.offset, j.len, row, g.floor_base, -1, cls, u, B.floor_y + 130 * size_t(k),
                                                       B.residue + 2 * size_t(row) * k, true);
            status[k] = st == SYMGPU_OK ? SYMGPU_VORBIS_JOB_DECODED : SYMGPU_VORBIS_JOB_REFUSED;
            if (st == SYMGPU_OK) a = Acc{1, int32_t(u->block_flag)};
        }
    }
    B.acc_in[k] = a;
}

// The time line of ogg_vorbis_plan: frames from the previous decoded packet's block flag, the reader's trims clamped to them,
// and a file's first decoded packet silenced (codec-vorbis lib.rs:318-322).
__global__ void __launch_bounds__(128) vorbis_span_kernel(const symgpu_vorbis_job* __restrict__ jobs, uint32_t n_jobs, const DevGroup* __restrict__ groups,
                                                          const uint32_t* __restrict__ keys, JobBufs B) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    unsigned long long left = 0;
    if (gi != kNone && B.acc_in[k].count) {
        const DevGroup g = groups[gi];
        const Acc before = B.acc[k];
        symgpu_vorbis_unit& u = B.units[k];
        const uint32_t prev = before.flag >= 0 ? uint32_t(before.flag) : u.block_flag;
        u.prev_block_flag = uint8_t(prev);
        const uint32_t n0 = 1u << g.bs0_exp, n1 = 1u << g.bs1_exp;
        const uint32_t frames = ((prev ? n1 : n0) + (u.block_flag ? n1 : n0)) / 4;
        Span s{frames, 0, 0, 0};
        if (before.count == 0) {
            s.trim_start = frames;
        } else {
            const symgpu_vorbis_job j = jobs[k];
            s.trim_start = min(j.discard, frames);
            s.trim_end = min(j.trim_end, frames - s.trim_start);
        }
        B.span[k] = s;
        left = frames - s.trim_start - s.trim_end;
    }
    B.left[k] = left;
}

__global__ void __launch_bounds__(256) vorbis_place_kernel(const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys, uint32_t row, JobBufs B,
                                                           symgpu_vorbis_unit* __restrict__ units, uint16_t* __restrict__ floor_y,
                                                           float* __restrict__ residue, symgpu_pcm_span* __restrict__ spans1,
                                                           symgpu_pcm_span* __restrict__ spans2, symgpu_vorbis_group_result* __restrict__ results,
                                                           const uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x;
    const uint32_t gi = keys[k];
    if (gi == kNone) return;
    const DevGroup g = groups[gi];
    const uint32_t rank = B.acc[k].count;
    const bool decoded = B.acc_in[k].count != 0;
    // decoded packets first in stream order, the others' slots from the back
    const uint64_t slot = g.frame_base + (decoded ? rank : g.n_jobs - 1 - ((k - g.first_job) - rank));
    float4* dst = reinterpret_cast<float4*>(residue + 2 * size_t(row) * slot);
    const float4* src = reinterpret_cast<const float4*>(B.residue + 2 * size_t(row) * k);
    for (uint32_t i = threadIdx.x; i < row / 2; i += blockDim.x) dst[i] = decoded ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t i = threadIdx.x; i < 130; i += blockDim.x) floor_y[130 * slot + i] = decoded ? B.floor_y[130 * size_t(k) + i] : uint16_t(0);
    if (threadIdx.x == 0) {
        symgpu_vorbis_unit u{};
        if (decoded) {
            u = B.units[k];
        } else {
            u.do_not_decode[0] = u.do_not_decode[1] = 1;
            u.floor[0] = u.floor[1] = 0xffff;
        }
        units[slot] = u;
        symgpu_pcm_span span{};
        const unsigned long long first = B.first[k];
        if (decoded) {
            const Span s = B.span[k];
            span = symgpu_pcm_span{slot * 2ull * row, row, s.frames, s.trim_start, s.trim_end, g.out_offset / g.channels + first};
        }
        spans1[k] = g.channels == 1 ? span : symgpu_pcm_span{};
        spans2[k] = g.channels == 2 ? span : symgpu_pcm_span{};
        if (k == g.first_job + g.n_jobs - 1) {  // the group's last job knows its totals
            symgpu_vorbis_group_result& r = results[gi];
            r.frames = first + B.left[k];
            r.packets = rank + (decoded ? 1u : 0u);
        }
    }
}

cudaError_t scan_acc(void* temp, size_t& temp_bytes, const uint32_t* keys, const Acc* in, Acc* out, uint32_t n_jobs, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveScanByKey(temp, temp_bytes, keys, in, out, AccOp(), Acc{0, -1}, int(n_jobs), cuda::std::equal_to<>(), st);
}
cudaError_t scan_first(void* temp, size_t& temp_bytes, const uint32_t* keys, const unsigned long long* left, unsigned long long* first, uint32_t n_jobs,
                       cudaStream_t st) {
    return cub::DeviceScan::ExclusiveSumByKey(temp, temp_bytes, keys, left, first, int(n_jobs), cuda::std::equal_to<>(), st);
}

// The distinct setups, built on the host.
struct Setups {
    std::vector<uint8_t> blob;
    std::vector<ve::SetupHead> heads;
    std::vector<symgpu_vorbis_stream> streams;
    std::vector<uint32_t> floor_base;
    std::vector<symgpu_vorbis_floor1> floors;
};

symgpu_status build_setups(const uint8_t* headers, size_t n_headers, const symgpu_vorbis_setup_ref* setups, size_t n_setups, Setups& out) {
    std::vector<symgpu_vorbis_floor1> fl(64);
    for (size_t i = 0; i < n_setups; ++i) {
        const symgpu_vorbis_setup_ref& r = setups[i];
        if (r.ident_offset > n_headers || r.ident_len > n_headers - r.ident_offset || r.setup_offset > n_headers || r.setup_len > n_headers - r.setup_offset)
            return SYMGPU_ERR_ARG;
        symgpu_vorbis_fe* fe = nullptr;
        symgpu_status e = symgpu_vorbis_fe_create(headers + r.ident_offset, r.ident_len, headers + r.setup_offset, r.setup_len, &fe);
        if (e != SYMGPU_OK) return e;
        ve::SetupHead h;
        ve::setup_export(fe, out.blob, h);
        symgpu_vorbis_stream s{};
        uint32_t n_fl = 0;
        e = symgpu_vorbis_fe_config(fe, &s, fl.data(), &n_fl);  // (a setup has at most 64 floors)
        symgpu_vorbis_fe_destroy(fe);
        if (e != SYMGPU_OK) return e;
        out.heads.push_back(h);
        out.streams.push_back(s);
        out.floor_base.push_back(uint32_t(out.floors.size()));
        out.floors.insert(out.floors.end(), fl.begin(), fl.begin() + n_fl);
    }
    if (out.floors.size() >= 0xffff) return SYMGPU_ERR_LIMIT;  // unit->floor is 16 bits, 0xffff = unused
    return SYMGPU_OK;
}

struct Layout {
    std::vector<DevGroup> dev;
    std::vector<symgpu_vorbis_run> runs;
    std::vector<symgpu_vorbis_stream> streams;  // one per group
    std::vector<symgpu_vorbis_group_result> empty;
    uint64_t n_frames = 0, class_bytes = 0;
    uint32_t row = 0;
};

symgpu_status check_groups(size_t n_jobs, const symgpu_vorbis_group* groups, size_t n_groups, const Setups& S, int format, size_t out_bytes, Layout& L) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    const uint64_t out_samples = out_bytes / sample;
    std::vector<JobRange> ranges;
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_vorbis_group& G = groups[g];
        if (G.setup >= S.heads.size() || G.out_offset % S.heads[G.setup].channels) return SYMGPU_ERR_ARG;
        ranges.push_back({G.first_job, G.n_jobs});
    }
    symgpu_status e = check_job_ranges(ranges, n_jobs);
    if (e != SYMGPU_OK) return e;
    if (n_groups > SYMGPU_VORBIS_MAX_FILES) return SYMGPU_ERR_LIMIT;
    for (size_t g = 0; g < n_groups; ++g) {
        const ve::SetupHead& h = S.heads[groups[g].setup];
        e = check_region(groups[g].out_offset, uint64_t(groups[g].n_jobs) * ((1u << h.bs1_exp) >> 1) * h.channels, out_samples);
        if (e != SYMGPU_OK) return e;
        L.row = std::max<uint32_t>(L.row, (1u << h.bs1_exp) >> 1);
    }
    L.dev.resize(n_groups);
    L.empty.resize(n_groups);
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_vorbis_group& G = groups[g];
        const ve::SetupHead& h = S.heads[G.setup];
        L.dev[g] = DevGroup{G.out_offset, L.n_frames, L.class_bytes, G.first_job, G.n_jobs, G.setup, S.floor_base[G.setup], h.channels, h.bs0_exp, h.bs1_exp,
                            h.class_cap};
        if (G.n_jobs) L.runs.push_back(symgpu_vorbis_run{uint32_t(g), uint32_t(L.n_frames), G.n_jobs, 0});
        L.streams.push_back(S.streams[G.setup]);
        L.empty[g] = symgpu_vorbis_group_result{};
        L.empty[g].sample_rate = h.sample_rate, L.empty[g].channels = h.channels;
        L.n_frames += G.n_jobs;
        L.class_bytes += uint64_t(G.n_jobs) * h.class_cap;
    }
    return SYMGPU_OK;
}

struct Scratch {
    size_t blob, heads, groups, keys, units, floor_y, residue, classes, acc_in, acc, span, left, first, p_units, p_floor_y, p_residue, pcm, spans1, spans2,
        temp, total;
    size_t temp_bytes;
};

cudaError_t scratch_layout(uint32_t n_jobs, const Setups& S, const Layout& L, Scratch& s) {
    size_t a = 0, b = 0;
    cudaError_t e = scan_acc(nullptr, a, nullptr, nullptr, nullptr, n_jobs, nullptr);
    if (e == cudaSuccess) e = scan_first(nullptr, b, nullptr, nullptr, nullptr, n_jobs, nullptr);
    if (e != cudaSuccess) return e;
    s.temp_bytes = std::max(a, b);
    Carver c;
    const size_t J = n_jobs, F = L.n_frames, R = L.row;
    s.blob = c.take(S.blob.size());
    s.heads = c.take(S.heads.size() * sizeof(ve::SetupHead));
    s.groups = c.take(L.dev.size() * sizeof(DevGroup));
    s.keys = c.take(J * sizeof(uint32_t));
    s.units = c.take(J * sizeof(symgpu_vorbis_unit));
    s.floor_y = c.take(J * 130 * sizeof(uint16_t));
    s.residue = c.take(J * 2 * R * sizeof(float));
    s.classes = c.take(L.class_bytes);
    s.acc_in = c.take(J * sizeof(Acc));
    s.acc = c.take(J * sizeof(Acc));
    s.span = c.take(J * sizeof(Span));
    s.left = c.take(J * sizeof(unsigned long long));
    s.first = c.take(J * sizeof(unsigned long long));
    s.p_units = c.take(F * sizeof(symgpu_vorbis_unit));
    s.p_floor_y = c.take(F * 130 * sizeof(uint16_t));
    s.p_residue = c.take(F * 2 * R * sizeof(float));
    s.pcm = c.take(F * 2 * R * sizeof(float));
    s.spans1 = c.take(J * sizeof(symgpu_pcm_span));
    s.spans2 = c.take(J * sizeof(symgpu_pcm_span));
    s.temp = c.take(s.temp_bytes);
    s.total = c.at;
    return cudaSuccess;
}

// The setups' floors and one stream per group, as symgpu_vorbis_floors_set / _streams_set register them (both wait for the stream).
symgpu_status register_streams(symgpu_ctx* ctx, const Setups& S, const Layout& L) {
    symgpu_status e = symgpu_vorbis_streams_set(ctx, L.streams.data(), uint32_t(L.streams.size()));
    if (e == SYMGPU_OK) e = symgpu_vorbis_floors_set(ctx, S.floors.data(), uint32_t(S.floors.size()));
    return e;
}

// Everything after the staging: device pointers, n_jobs > 0, n_groups > 0, ctx->d_stage holds `s`.
symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const Setups& S, const Layout& L, const uint8_t* bytes, size_t n_bytes,
                               const symgpu_vorbis_job* jobs, uint32_t n_jobs, int format, void* out, symgpu_vorbis_group_result* results, uint8_t* status) {
    char* stage = static_cast<char*>(ctx->d_stage);
    auto at = [&](size_t off) { return static_cast<void*>(stage + off); };
    uint8_t* blob = static_cast<uint8_t*>(at(s.blob));
    ve::SetupHead* heads = static_cast<ve::SetupHead*>(at(s.heads));
    DevGroup* groups = static_cast<DevGroup*>(at(s.groups));
    uint32_t* keys = static_cast<uint32_t*>(at(s.keys));
    JobBufs B{static_cast<symgpu_vorbis_unit*>(at(s.units)), static_cast<uint16_t*>(at(s.floor_y)), static_cast<float*>(at(s.residue)),
              static_cast<uint8_t*>(at(s.classes)),          static_cast<Acc*>(at(s.acc_in)),       static_cast<Acc*>(at(s.acc)),
              static_cast<Span*>(at(s.span)),                static_cast<unsigned long long*>(at(s.left)), static_cast<unsigned long long*>(at(s.first))};
    symgpu_vorbis_unit* p_units = static_cast<symgpu_vorbis_unit*>(at(s.p_units));
    uint16_t* p_floor_y = static_cast<uint16_t*>(at(s.p_floor_y));
    float* p_residue = static_cast<float*>(at(s.p_residue));
    float* pcm = static_cast<float*>(at(s.pcm));
    symgpu_pcm_span* spans1 = static_cast<symgpu_pcm_span*>(at(s.spans1));
    symgpu_pcm_span* spans2 = static_cast<symgpu_pcm_span*>(at(s.spans2));
    void* temp = at(s.temp);
    size_t temp_bytes = s.temp_bytes;
    const uint32_t n_groups = uint32_t(L.dev.size());
    const uint32_t job_blocks = (n_jobs + 127) / 128;
    cudaStream_t st = ctx->stream;
    // (copies from pageable memory return once the source is staged, so the host vectors may go out of scope without a wait)
    CU(ctx, cudaMemcpyAsync(blob, S.blob.data(), S.blob.size(), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(heads, S.heads.data(), S.heads.size() * sizeof(ve::SetupHead), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(groups, L.dev.data(), n_groups * sizeof(DevGroup), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemcpyAsync(results, L.empty.data(), n_groups * sizeof(symgpu_vorbis_group_result), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemsetAsync(keys, 0xff, n_jobs * sizeof(uint32_t), st));  // jobs no group names
    CU(ctx, cudaMemsetAsync(status, SYMGPU_VORBIS_JOB_REFUSED, n_jobs, st));
    CU(ctx, cudaMemsetAsync(spans1, 0, n_jobs * sizeof(symgpu_pcm_span), st));
    CU(ctx, cudaMemsetAsync(spans2, 0, n_jobs * sizeof(symgpu_pcm_span), st));
    CU(ctx, cudaMemsetAsync(B.residue, 0, size_t(n_jobs) * 2 * L.row * sizeof(float), st));  // decode_packet only adds into the rows
    vorbis_key_kernel<<<n_groups, 128, 0, st>>>(groups, keys);
    CU(ctx, cudaGetLastError());
    vorbis_packet_kernel<<<job_blocks, 128, 0, st>>>(bytes, n_bytes, jobs, n_jobs, groups, keys, blob, heads, L.row, B, status);
    CU(ctx, cudaGetLastError());
    CU(ctx, scan_acc(temp, temp_bytes, keys, B.acc_in, B.acc, n_jobs, st));
    vorbis_span_kernel<<<job_blocks, 128, 0, st>>>(jobs, n_jobs, groups, keys, B);
    CU(ctx, cudaGetLastError());
    temp_bytes = s.temp_bytes;
    CU(ctx, scan_first(temp, temp_bytes, keys, B.left, B.first, n_jobs, st));
    vorbis_place_kernel<<<n_jobs, 256, 0, st>>>(groups, keys, L.row, B, p_units, p_floor_y, p_residue, spans1, spans2, results, status);
    CU(ctx, cudaGetLastError());
    ctx->launches += 8;  // four kernels here, two for each device-wide scan
    if (!L.runs.empty()) {
        const symgpu_status e = symgpu_vorbis_synth_dev(ctx, p_units, p_floor_y, p_residue, L.runs.data(), uint32_t(L.runs.size()), uint32_t(L.n_frames),
                                                        L.row, pcm);
        if (e != SYMGPU_OK) return e;
    }
    for (uint32_t ch = 1; ch <= 2; ++ch) {
        const symgpu_status e = symgpu_pcm_pack_dev(ctx, pcm, ch == 1 ? spans1 : spans2, n_jobs, ch, L.row, L.row, format, out);
        if (e != SYMGPU_OK) return e;
    }
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x7fffffff;  // the device-wide scans count items in an int

// Host-side preparation shared by both variants: setups, groups, registration and the staging buffer's size.
symgpu_status prepare(symgpu_ctx* ctx, const uint8_t* headers, size_t n_headers, const symgpu_vorbis_setup_ref* setups, size_t n_setups, size_t n_jobs,
                      const symgpu_vorbis_group* groups, size_t n_groups, int format, size_t out_bytes, Setups& S, Layout& L) {
    symgpu_status e = build_setups(headers, n_headers, setups, n_setups, S);
    if (e == SYMGPU_OK) e = check_groups(n_jobs, groups, n_groups, S, format, out_bytes, L);
    return e;
}

}  // namespace

extern "C" symgpu_status symgpu_vorbis_decode_dev(symgpu_ctx* ctx, const uint8_t* headers, size_t n_headers, const symgpu_vorbis_setup_ref* setups,
                                                  size_t n_setups, const uint8_t* bytes, size_t n_bytes, const symgpu_vorbis_job* jobs, size_t n_jobs,
                                                  const symgpu_vorbis_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                  symgpu_vorbis_group_result* results, uint8_t* status) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || (n_headers && !headers) ||
        (n_setups && !setups))
        return SYMGPU_ERR_ARG;
    Setups S;
    Layout L;
    symgpu_status e = prepare(ctx, headers, n_headers, setups, n_setups, n_jobs, groups, n_groups, format, out_bytes, S, L);
    if (e != SYMGPU_OK) return e;
    DeviceGuard guard(ctx->device);
    if (n_jobs == 0 || n_groups == 0) {  // what a call with jobs reports for a group without any
        if (n_groups) {
            CU(ctx, cudaMemcpyAsync(results, L.empty.data(), n_groups * sizeof(symgpu_vorbis_group_result), cudaMemcpyHostToDevice, ctx->stream));
            CU(ctx, cudaStreamSynchronize(ctx->stream));  // `L` is pageable and local
        }
        if (n_jobs) CU(ctx, cudaMemsetAsync(status, SYMGPU_VORBIS_JOB_REFUSED, n_jobs, ctx->stream));
        return SYMGPU_OK;
    }
    e = register_streams(ctx, S, L);
    if (e != SYMGPU_OK) return e;
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), S, L, s));
    e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    return decode_on_device(ctx, s, S, L, bytes, n_bytes, jobs, uint32_t(n_jobs), format, out, results, status);
}

extern "C" symgpu_status symgpu_vorbis_decode_host(symgpu_ctx* ctx, const uint8_t* headers, size_t n_headers, const symgpu_vorbis_setup_ref* setups,
                                                   size_t n_setups, const uint8_t* bytes, size_t n_bytes, const symgpu_vorbis_job* jobs, size_t n_jobs,
                                                   const symgpu_vorbis_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                   symgpu_vorbis_group_result* results, uint8_t* status) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || (n_headers && !headers) ||
        (n_setups && !setups) || !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    Setups S;
    Layout L;
    symgpu_status e = prepare(ctx, headers, n_headers, setups, n_setups, n_jobs, groups, n_groups, format, out_bytes, S, L);
    if (e != SYMGPU_OK) return e;
    for (size_t g = 0; g < n_groups; ++g) results[g] = L.empty[g];
    for (size_t k = 0; k < n_jobs; ++k) status[k] = SYMGPU_VORBIS_JOB_REFUSED;
    if (n_jobs == 0 || n_groups == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    e = register_streams(ctx, S, L);
    if (e != SYMGPU_OK) return e;
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), S, L, s));
    return decode_from_host(
        ctx, s.total, std::array<HostIn, 2>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_vorbis_job)}}}, out, out_bytes,
        std::array<HostOut, 2>{{{status, n_jobs}, {results, n_groups * sizeof(symgpu_vorbis_group_result)}}},
        [&](const std::array<void*, 2>& in, void* d_out, const std::array<void*, 2>& back) {
            return decode_on_device(ctx, s, S, L, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_vorbis_job*>(in[1]), uint32_t(n_jobs),
                                    format, d_out, static_cast<symgpu_vorbis_group_result*>(back[1]), static_cast<uint8_t*>(back[0]));
        },
        [&] { return written_by_results(groups, results, n_groups, symgpu_sample_bytes(format)); });
}
