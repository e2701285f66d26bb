// ADTS AAC-LC decoded on the device, many files per call (include/symgpu.h "AAC-LC decoded on the device"; DESIGN §3, §5g).
// A file is a group, a packet (one raw_data_block) is a job.  The packet rules are those of aac_entropy.h, the code the CPU
// front-end runs.
//
//   aac_setup_kernel    one CTA per group: resets the group's synthesis state slot, names the group of each of its jobs
//   aac_pass_kernel A   one thread per job: decode_job from a fresh state -> the job's units, TNS records, coefficients,
//                       pulse lines, group-0 scale factors and the JobRec of what it does to the state that carries
//   aac_walk_kernel     one thread per group: walk_step over the group's records in stream order -> each packet's status in
//                       context, its generators' start states, previous window shapes and the packets whose scale factors its
//                       pulse lines read; frame slots, spans, the result
//   aac_pass_kernel B   one thread per job that is decoded in context and drew noise: decode_job again from its real
//                       generator states (noise changes values, never control flow)
//   aac_pulse_kernel    one thread per job: every pulsed channel of a decoded packet -> a PulseFix record with the line values
//                       and the scale factors the walk named for them
//   -- one 8-byte readback (records, pass-B packets); when records exist, they come back, the host runs pulse_apply (the C
//      library's powf) on them, and they go back --
//   aac_pulse_write_kernel  one thread per record: the at most 4 new line values
//   aac_place_kernel    one CTA per frame slot: coefficients, units (prev_window_shape, tns_first) and TNS records into place;
//                       muted slots and channels a file does not have become zeros
//   symgpu_aac_synth_dev (every group one run of n_jobs frames), symgpu_pcm_pack_dev (mono, stereo)
//
// Frame slots: a group owns n_jobs consecutive slots.  Its decoded packets take the first ones in stream order, the others
// the slots behind them, muted; the synthesis runs those after the group's real frames, and the state slot's contents after
// the call are unspecified.  Each slot has room for 16 TNS records (8 per channel), so no scan places them.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "aac_entropy.h"
#include "batch_call.h"
#include "pack_kernel.h"

using namespace symgpu_detail;
namespace ae = symgpu::aace;

namespace {

constexpr uint32_t kNone = 0xffffffffu;
constexpr int8_t kOutside = -128;  // JobRec::status of a job outside `bytes`

struct DevGroup {  // symgpu_aac_group + the group's first frame slot and rate index
    uint64_t out_offset;
    uint64_t frame_base;
    uint32_t first_job, n_jobs, slot, sample_rate, rate_idx, channels;
};

struct PulseFix {  // one pulsed channel of a decoded packet
    uint32_t job, ch;
    ae::PulseLines p;
    float value[4], scale[4];
};

// Per-job scratch (one array each, indexed by job).
struct JobBufs {
    ae::JobState* state;
    symgpu_aac_unit* units;   // [2]
    symgpu_aac_tns* tns;      // [16]
    float* coeffs;            // [2048]
    ae::PulseLines* pulse;    // [2]
    float* scales0;           // [128]
    ae::WalkOut* walk;
};

__device__ __forceinline__ ae::JobOut out_of(const JobBufs& B, uint32_t k) {
    return ae::JobOut{B.units + 2 * size_t(k), B.tns + 16 * size_t(k), B.coeffs + 2048 * size_t(k), B.pulse + 2 * size_t(k), B.scales0 + 128 * size_t(k)};
}

__global__ void __launch_bounds__(128) aac_setup_kernel(const DevGroup* __restrict__ groups, uint32_t* __restrict__ keys, float* __restrict__ states) {
    const DevGroup g = groups[blockIdx.x];
    float4* st = reinterpret_cast<float4*>(states + size_t(g.slot) * 4096);  // what symgpu_aac_stream_reset does
    for (uint32_t i = threadIdx.x; i < 1024; i += blockDim.x) st[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t i = threadIdx.x; i < g.n_jobs; i += blockDim.x) keys[g.first_job + i] = blockIdx.x;
}

__global__ void __launch_bounds__(128) aac_pass_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_piece* __restrict__ jobs,
                                                       uint32_t n_jobs, const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys,
                                                       const ae::Tables* __restrict__ T, JobBufs B, uint32_t* __restrict__ n_redo) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    if (gi == kNone) return;
    ae::JobState& S = B.state[k];
    uint32_t start[2] = {ae::kLcgSeed, ae::kLcgSeed};
    if (n_redo) {  // pass B
        const ae::WalkOut w = B.walk[k];
        if (w.status != SYMGPU_OK || (S.rec.draws[0] == 0 && S.rec.draws[1] == 0)) return;
        start[0] = w.lcg_start[0], start[1] = w.lcg_start[1];
        atomicAdd(n_redo, 1u);
    }
    const symgpu_piece j = jobs[k];
    if (j.offset > n_bytes || j.len > n_bytes - j.offset) {
        S.rec = ae::JobRec{};
        S.rec.status = kOutside;
        return;
    }
    const DevGroup g = groups[gi];
    ae::decode_job(bytes + j.offset, j.len, *T, g.rate_idx, g.channels, start, n_redo == nullptr, S, out_of(B, k));
}

__global__ void __launch_bounds__(128) aac_walk_kernel(const DevGroup* __restrict__ groups, uint32_t n_groups, JobBufs B, uint32_t* __restrict__ slot_job,
                                                       symgpu_pcm_span* __restrict__ spans1, symgpu_pcm_span* __restrict__ spans2,
                                                       symgpu_aac_group_result* __restrict__ results, uint8_t* __restrict__ status) {
    const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n_groups) return;
    const DevGroup g = groups[gi];
    const uint64_t frame0 = g.out_offset / g.channels;
    ae::WalkState w;
    ae::walk_begin(w);
    uint32_t good = 0, back = 0;
    for (uint32_t i = 0; i < g.n_jobs; ++i) {
        const uint32_t k = g.first_job + i;
        const ae::JobRec r = B.state[k].rec;
        ae::WalkOut o{};
        uint8_t result;
        if (r.status == kOutside) {  // no packet: the state is untouched
            o.status = kOutside;
            result = SYMGPU_AAC_JOB_INVALID;
        } else {
            o = ae::walk_step(w, r, k, B.pulse + 2 * size_t(k));
            result = o.status == SYMGPU_OK ? SYMGPU_AAC_JOB_DECODED : o.status == SYMGPU_ERR_UNSUPPORTED ? SYMGPU_AAC_JOB_UNSUPPORTED : SYMGPU_AAC_JOB_REFUSED;
        }
        const bool decoded = result == SYMGPU_AAC_JOB_DECODED;
        const uint64_t slot = g.frame_base + (decoded ? good : g.n_jobs - 1 - back++);
        B.walk[k] = o;
        slot_job[slot] = decoded ? k : kNone;
        symgpu_pcm_span span{};
        if (decoded) span = symgpu_pcm_span{slot * 2048ull, 1024u, 1024u, 0u, 0u, frame0 + 1024ull * good++};
        spans1[k] = g.channels == 1 ? span : symgpu_pcm_span{};
        spans2[k] = g.channels == 2 ? span : symgpu_pcm_span{};
        status[k] = result;
    }
    symgpu_aac_group_result res{};
    res.frames = 1024ull * good, res.packets = good, res.sample_rate = g.sample_rate, res.channels = uint8_t(g.channels);
    results[gi] = res;
}

// Each line reads the group-0 scale factor the walk names (the packet's own, or the one an earlier packet left behind in a band
// at or above this packet's max_sfb; 0.0 when no packet wrote that band: a new element's scale factors are zero).
__global__ void __launch_bounds__(128) aac_pulse_kernel(const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys, uint32_t n_jobs,
                                                        JobBufs B, PulseFix* __restrict__ fixes, uint32_t* __restrict__ n_fixes) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    if (gi == kNone || B.walk[k].status != SYMGPU_OK) return;
    const uint32_t channels = groups[gi].channels;
    for (uint32_t c = 0; c < channels; ++c) {
        const ae::PulseLines p = B.pulse[2 * size_t(k) + c];
        if (p.n == 0) continue;
        PulseFix f;
        f.job = k, f.ch = c, f.p = p;
        for (uint32_t i = 0; i < p.n; ++i) {
            const uint32_t src = B.walk[k].scale_src[c][i];
            f.value[i] = B.coeffs[2048 * size_t(k) + 1024 * c + p.line[i]];
            f.scale[i] = src == ae::kNoJob ? 0.0f : B.scales0[128 * size_t(src) + 64 * c + p.band[i]];
        }
        fixes[atomicAdd(n_fixes, 1u)] = f;
    }
}

__global__ void __launch_bounds__(128) aac_pulse_write_kernel(const PulseFix* __restrict__ fixes, uint32_t n, float* __restrict__ coeffs) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const PulseFix f = fixes[t];
    for (uint32_t i = 0; i < f.p.n; ++i) coeffs[2048 * size_t(f.job) + 1024 * f.ch + f.p.line[i]] = f.value[i];  // in order: a line's last pulse wins
}

__global__ void __launch_bounds__(256) aac_place_kernel(const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys,
                                                        const uint32_t* __restrict__ slot_job, JobBufs B, symgpu_aac_unit* __restrict__ units,
                                                        symgpu_aac_tns* __restrict__ tns, float* __restrict__ coeffs) {
    const uint32_t f = blockIdx.x;
    const uint32_t k = slot_job[f];
    const uint32_t channels = k == kNone ? 0 : groups[keys[k]].channels;
    float4* dst = reinterpret_cast<float4*>(coeffs + 2048 * size_t(f));
    const float4* src = reinterpret_cast<const float4*>(B.coeffs + 2048 * size_t(k == kNone ? 0 : k));
    for (uint32_t i = threadIdx.x; i < 512; i += blockDim.x) dst[i] = (i >> 8) < channels ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const symgpu_aac_unit* ju = B.units + 2 * size_t(k == kNone ? 0 : k);
    if (threadIdx.x < 2) {
        const uint32_t c = threadIdx.x;
        symgpu_aac_unit u{};
        if (c < channels) {
            u = ju[c];
            u.prev_window_shape = uint8_t(B.walk[k].prev_shape >> c & 1);
            u.tns_first = u.n_tns ? uint32_t(16 * f + 8 * c) : 0;
        }
        units[2 * size_t(f) + c] = u;
    }
    // 16 records of 22 words: referenced ones copied, the rest zero
    uint32_t* tw = reinterpret_cast<uint32_t*>(tns + 16 * size_t(f));
    const uint32_t* jt = reinterpret_cast<const uint32_t*>(B.tns + 16 * size_t(k == kNone ? 0 : k));
    constexpr uint32_t kWords = sizeof(symgpu_aac_tns) / 4;
    for (uint32_t i = threadIdx.x; i < 16 * kWords; i += blockDim.x) {
        const uint32_t rec = i / kWords, c = rec / 8;
        const bool used = c < channels && rec % 8 < ju[c].n_tns;
        tw[i] = used ? jt[i] : 0u;
    }
}

struct Layout {
    std::vector<DevGroup> dev;
    std::vector<symgpu_aac_run> runs;
    uint64_t n_frames = 0;
};

symgpu_status check_groups(const symgpu_ctx* ctx, size_t n_jobs, const symgpu_aac_group* groups, size_t n_groups, int format, size_t out_bytes, Layout& L) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    const uint64_t out_samples = out_bytes / sample;
    std::vector<JobRange> ranges;
    std::vector<uint32_t> slots;
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_aac_group& G = groups[g];
        if ((G.channels != 1 && G.channels != 2) || G.sample_rate == 0 || G.out_offset % G.channels) return SYMGPU_ERR_ARG;
        ranges.push_back({G.first_job, G.n_jobs});
        slots.push_back(G.slot);
    }
    symgpu_status e = check_job_ranges(ranges, n_jobs);
    if (e == SYMGPU_OK) e = check_slots(slots, ctx->n_aac_streams);
    for (size_t g = 0; g < n_groups && e == SYMGPU_OK; ++g) e = check_region(groups[g].out_offset, uint64_t(groups[g].n_jobs) * 1024u * groups[g].channels, out_samples);
    if (e != SYMGPU_OK) return e;
    L.dev.resize(n_groups);
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_aac_group& G = groups[g];
        L.dev[g] = DevGroup{G.out_offset, L.n_frames, G.first_job, G.n_jobs, uint32_t(G.slot), G.sample_rate, symgpu::aac_rate_index(G.sample_rate), G.channels};
        if (G.n_jobs) L.runs.push_back(symgpu_aac_run{uint32_t(G.slot), uint32_t(L.n_frames), G.n_jobs, G.channels, {0, 0, 0}});
        L.n_frames += G.n_jobs;
    }
    return SYMGPU_OK;
}

struct Scratch {
    size_t groups, keys, state, units, tns, coeffs, pulse, scales0, walk, frame, slot_job, spans1, spans2, counts, fixes, p_units, p_tns, p_coeffs, pcm,
        total;
};

Scratch scratch_layout(uint32_t n_jobs, size_t n_groups, const Layout& L) {
    Scratch s;
    Carver c;
    const size_t J = n_jobs, F = L.n_frames;
    s.groups = c.take(n_groups * sizeof(DevGroup));
    s.keys = c.take(J * sizeof(uint32_t));
    s.state = c.take(J * sizeof(ae::JobState));
    s.units = c.take(J * 2 * sizeof(symgpu_aac_unit));
    s.tns = c.take(J * 16 * sizeof(symgpu_aac_tns));
    s.coeffs = c.take(J * 2048 * sizeof(float));
    s.pulse = c.take(J * 2 * sizeof(ae::PulseLines));
    s.scales0 = c.take(J * 128 * sizeof(float));
    s.walk = c.take(J * sizeof(ae::WalkOut));
    s.slot_job = c.take(F * sizeof(uint32_t));
    s.spans1 = c.take(J * sizeof(symgpu_pcm_span));
    s.spans2 = c.take(J * sizeof(symgpu_pcm_span));
    s.counts = c.take(2 * sizeof(uint32_t));
    s.fixes = c.take(J * 2 * sizeof(PulseFix));
    s.p_units = c.take(F * 2 * sizeof(symgpu_aac_unit));
    s.p_tns = c.take(F * 16 * sizeof(symgpu_aac_tns));
    s.p_coeffs = c.take(F * 2048 * sizeof(float));
    s.pcm = c.take(F * 2048 * sizeof(float));
    s.total = c.at;
    return s;
}

// Everything after the staging: device pointers, n_jobs > 0, n_groups > 0, ctx->d_stage holds `s`.
symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const Layout& L, const uint8_t* bytes, size_t n_bytes, const symgpu_piece* jobs,
                               uint32_t n_jobs, int format, void* out, symgpu_aac_group_result* results, uint8_t* status, uint32_t* n_redecoded) {
    char* stage = static_cast<char*>(ctx->d_stage);
    auto at = [&](size_t off) { return static_cast<void*>(stage + off); };
    DevGroup* groups = static_cast<DevGroup*>(at(s.groups));
    uint32_t* keys = static_cast<uint32_t*>(at(s.keys));
    JobBufs B{static_cast<ae::JobState*>(at(s.state)),   static_cast<symgpu_aac_unit*>(at(s.units)), static_cast<symgpu_aac_tns*>(at(s.tns)),
              static_cast<float*>(at(s.coeffs)),         static_cast<ae::PulseLines*>(at(s.pulse)),  static_cast<float*>(at(s.scales0)),
              static_cast<ae::WalkOut*>(at(s.walk))};
    uint32_t* slot_job = static_cast<uint32_t*>(at(s.slot_job));
    symgpu_pcm_span* spans1 = static_cast<symgpu_pcm_span*>(at(s.spans1));
    symgpu_pcm_span* spans2 = static_cast<symgpu_pcm_span*>(at(s.spans2));
    uint32_t* counts = static_cast<uint32_t*>(at(s.counts));  // pulse records, pass-B packets
    PulseFix* fixes = static_cast<PulseFix*>(at(s.fixes));
    symgpu_aac_unit* p_units = static_cast<symgpu_aac_unit*>(at(s.p_units));
    symgpu_aac_tns* p_tns = static_cast<symgpu_aac_tns*>(at(s.p_tns));
    float* p_coeffs = static_cast<float*>(at(s.p_coeffs));
    float* pcm = static_cast<float*>(at(s.pcm));
    const uint32_t n_groups = uint32_t(L.dev.size());
    const uint32_t job_blocks = (n_jobs + 127) / 128;
    cudaStream_t st = ctx->stream;
    if (!ctx->d_aac_fe_tab) {  // the packet rules' tables, uploaded once per context and freed with it
        void* p = nullptr;
        CU(ctx, cudaMalloc(&p, sizeof(ae::Tables)));
        const cudaError_t e = cudaMemcpy(p, &symgpu::aac_tables_host(), sizeof(ae::Tables), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) return cudaFree(p), cuda_fail(ctx, e, "cudaMemcpy(aac tables)");
        ctx->d_aac_fe_tab = p;
    }
    const ae::Tables* T = static_cast<const ae::Tables*>(ctx->d_aac_fe_tab);
    CU(ctx, cudaMemcpyAsync(groups, L.dev.data(), n_groups * sizeof(DevGroup), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemsetAsync(keys, 0xff, n_jobs * sizeof(uint32_t), st));  // jobs no group names
    CU(ctx, cudaMemsetAsync(status, SYMGPU_AAC_JOB_REFUSED, n_jobs, st));
    CU(ctx, cudaMemsetAsync(spans1, 0, n_jobs * sizeof(symgpu_pcm_span), st));
    CU(ctx, cudaMemsetAsync(spans2, 0, n_jobs * sizeof(symgpu_pcm_span), st));
    CU(ctx, cudaMemsetAsync(counts, 0, 2 * sizeof(uint32_t), st));
    CU(ctx, cudaMemsetAsync(B.coeffs, 0, size_t(n_jobs) * 2048 * sizeof(float), st));  // pass A writes only coded lines
    aac_setup_kernel<<<n_groups, 128, 0, st>>>(groups, keys, ctx->d_aac_states);
    CU(ctx, cudaGetLastError());
    aac_pass_kernel<<<job_blocks, 128, 0, st>>>(bytes, n_bytes, jobs, n_jobs, groups, keys, T, B, nullptr);
    CU(ctx, cudaGetLastError());
    aac_walk_kernel<<<(n_groups + 127) / 128, 128, 0, st>>>(groups, n_groups, B, slot_job, spans1, spans2, results, status);
    CU(ctx, cudaGetLastError());
    aac_pass_kernel<<<job_blocks, 128, 0, st>>>(bytes, n_bytes, jobs, n_jobs, groups, keys, T, B, counts + 1);
    CU(ctx, cudaGetLastError());
    aac_pulse_kernel<<<job_blocks, 128, 0, st>>>(groups, keys, n_jobs, B, fixes, counts);
    CU(ctx, cudaGetLastError());
    ctx->launches += 5;
    // Pulse::synth on the host: one 8-byte readback (with the pass-B count), the records only when there are any
    uint32_t h_counts[2] = {0, 0};
    CU(ctx, cudaMemcpyAsync(h_counts, counts, sizeof h_counts, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    const uint32_t n_fix = h_counts[0];
    if (n_redecoded) *n_redecoded = h_counts[1];
    if (n_fix) {
        std::vector<PulseFix> h(n_fix);
        CU(ctx, cudaMemcpyAsync(h.data(), fixes, n_fix * sizeof(PulseFix), cudaMemcpyDeviceToHost, st));
        CU(ctx, cudaStreamSynchronize(st));
        for (PulseFix& f : h) ae::pulse_apply(f.p, f.scale, f.value);
        CU(ctx, cudaMemcpyAsync(fixes, h.data(), n_fix * sizeof(PulseFix), cudaMemcpyHostToDevice, st));
        // (a copy from pageable memory returns once `h` is staged, so `h` may go out of scope without a wait)
        aac_pulse_write_kernel<<<(n_fix + 127) / 128, 128, 0, st>>>(fixes, n_fix, B.coeffs);
        CU(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    if (L.n_frames) {
        aac_place_kernel<<<uint32_t(L.n_frames), 256, 0, st>>>(groups, keys, slot_job, B, p_units, p_tns, p_coeffs);
        CU(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    if (!L.runs.empty()) {
        const symgpu_status e = symgpu_aac_synth_dev(ctx, p_units, p_tns, uint32_t(L.n_frames * 16), p_coeffs, L.runs.data(), uint32_t(L.runs.size()),
                                                     uint32_t(L.n_frames), pcm);
        if (e != SYMGPU_OK) return e;
    }
    for (uint32_t ch = 1; ch <= 2; ++ch) {
        const symgpu_status e = symgpu_pcm_pack_dev(ctx, pcm, ch == 1 ? spans1 : spans2, n_jobs, ch, 1024, 1024, format, out);
        if (e != SYMGPU_OK) return e;
    }
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x0fffffff;  // 16 TNS records per frame slot are counted in 32 bits

symgpu_aac_group_result empty_result(const symgpu_aac_group& G) {
    symgpu_aac_group_result r{};
    r.sample_rate = G.sample_rate, r.channels = G.channels;
    return r;
}

}  // namespace

extern "C" symgpu_status symgpu_aac_decode_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_piece* jobs, size_t n_jobs,
                                               const symgpu_aac_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                               symgpu_aac_group_result* results, uint8_t* status, uint32_t* n_redecoded) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff)
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    if (n_redecoded) *n_redecoded = 0;
    DeviceGuard guard(ctx->device);
    if (n_jobs == 0 || n_groups == 0) {  // what a call with jobs reports for a group without any
        if (n_groups) {
            std::vector<symgpu_aac_group_result> r(n_groups);
            for (size_t g = 0; g < n_groups; ++g) r[g] = empty_result(groups[g]);
            CU(ctx, cudaMemcpyAsync(results, r.data(), n_groups * sizeof(symgpu_aac_group_result), cudaMemcpyHostToDevice, ctx->stream));
            CU(ctx, cudaStreamSynchronize(ctx->stream));  // `r` is pageable and local
        }
        if (n_jobs) CU(ctx, cudaMemsetAsync(status, SYMGPU_AAC_JOB_REFUSED, n_jobs, ctx->stream));
        return SYMGPU_OK;
    }
    const Scratch s = scratch_layout(uint32_t(n_jobs), n_groups, L);
    e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    return decode_on_device(ctx, s, L, bytes, n_bytes, jobs, uint32_t(n_jobs), format, out, results, status, n_redecoded);
}

extern "C" symgpu_status symgpu_aac_decode_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_piece* jobs, size_t n_jobs,
                                                const symgpu_aac_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                symgpu_aac_group_result* results, uint8_t* status, uint32_t* n_redecoded) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff ||
        !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    for (size_t g = 0; g < n_groups; ++g) results[g] = empty_result(groups[g]);
    for (size_t k = 0; k < n_jobs; ++k) status[k] = SYMGPU_AAC_JOB_REFUSED;
    if (n_redecoded) *n_redecoded = 0;
    if (n_jobs == 0 || n_groups == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const Scratch s = scratch_layout(uint32_t(n_jobs), n_groups, L);
    return decode_from_host(
        ctx, s.total, std::array<HostIn, 2>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_piece)}}}, out, out_bytes,
        std::array<HostOut, 2>{{{status, n_jobs}, {results, n_groups * sizeof(symgpu_aac_group_result)}}},
        [&](const std::array<void*, 2>& in, void* d_out, const std::array<void*, 2>& back) {
            return decode_on_device(ctx, s, L, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_piece*>(in[1]), uint32_t(n_jobs), format,
                                    d_out, static_cast<symgpu_aac_group_result*>(back[1]), static_cast<uint8_t*>(back[0]), n_redecoded);
        },
        [&] { return written_by_results(groups, results, n_groups, symgpu_sample_bytes(format)); });
}
