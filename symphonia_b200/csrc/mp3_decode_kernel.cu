// MPEG Layer III decoded on the device, many files per call (include/symgpu.h "MPEG Layer III decoded on the device";
// DESIGN §3).  A file is a group, a packet is a job.
//
//   mp3_head_kernel     one CTA per group: resets the group's synthesis state slot; one thread per job runs the packet
//                       prologue (sync search, header, length); the group's first job that passes fixes the specification
//   mp3_side_kernel     one thread per job: the specification, the group's granules / channels, the layer check and the
//                       side read of mp3_entropy.h -> the job's FrameSide record
//   -- rounds --
//   mp3_walk_kernel     one thread per group: the reservoir step of mp3_entropy.h over the group's records in order ->
//                       four GcJobs per frame, each frame's slot and main-data place, the output spans, the group's result
//   mp3_gather_kernel   one warp per job: the frame's main data into the compacted stream md
//   mp3_huffman_kernel  one thread per granule-channel: decode_gc_job; a failure records the frame (atomicMin per group)
//   -- until no group fails; then --
//   dequant_launch, symgpu_mp3_synth_dev (every group one run of n_jobs frames), symgpu_pcm_pack_dev (mono, stereo)
//
// Frame slots: a group owns n_jobs consecutive slots.  Its decoded frames take the first ones in stream order; a left-out
// frame takes a slot from the back with its real granule-channels (their over-read is still a failure, as in the
// reference), the slots of refused packets come behind, muted.  None of those has a span, and the synthesis runs them
// after the group's real frames.  A group's region of md is 2048 bytes per slot, the most main data an accepted frame can
// add (main_data_begin + slot <= 2048), so no device-wide scan places it.
//
// Only a group's first failed frame is certain: the frames behind it were walked with a reservoir the reference empties.
// So a round ends with one 4-byte readback; when a group failed, the next walk marks that frame bad (bad = 1) and re-runs
// the group, and the gather and Huffman kernels skip the groups that did not.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "batch_call.h"
#include "mp3_entropy.h"
#include "mp3_kernel.h"
#include "pack_kernel.h"

using namespace symgpu_detail;
namespace me = symgpu::mp3e;

namespace {

constexpr uint32_t kNone = 0xffffffffu;     // no group / no packet fixed the specification / the header was refused
constexpr uint32_t kOutside = 0xfffffffeu;  // Head::q of a job outside `bytes`
constexpr uint32_t kMdPerSlot = 2048;
constexpr int kWarpsPerCta = 4;

struct DevGroup {  // 32 bytes: symgpu_mp3_group + the group's first frame slot
    uint64_t out_offset;
    uint64_t frame_base;
    uint32_t first_job, n_jobs, slot;
    uint8_t granules, channels, reserved[2];
};
struct Spec {
    uint32_t job, rate, channels, granules;
};
struct Head {
    uint32_t q;     // the header's byte offset in the packet; kNone: refused by the prologue, kOutside: outside `bytes`
    uint32_t word;  // the header word
};
struct Copy {       // what the gather moves for a job: nothing when len == 0
    uint64_t dst;   // in md
    uint32_t src;   // from the packet's first byte
    uint32_t len;
};

__device__ __forceinline__ bool job_in_range(const symgpu_mp3_job& j, size_t n_bytes) { return j.offset <= n_bytes && j.len <= n_bytes - j.offset; }

__global__ void __launch_bounds__(128) mp3_head_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_mp3_job* __restrict__ jobs,
                                                       const DevGroup* __restrict__ groups, Head* __restrict__ heads, uint32_t* __restrict__ keys,
                                                       Spec* __restrict__ spec, symgpu::Mp3StreamState* __restrict__ states) {
    __shared__ uint32_t first;
    const uint32_t gi = blockIdx.x;
    const DevGroup g = groups[gi];
    // the group's state slot starts from silence (what symgpu_mp3_stream_reset does), in this same launch for every group
    float4* st = reinterpret_cast<float4*>(states + size_t(g.slot) * 2);
    for (uint32_t i = threadIdx.x; i < 2 * sizeof(symgpu::Mp3StreamState) / sizeof(float4); i += blockDim.x) st[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (threadIdx.x == 0) first = kNone;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < g.n_jobs; i += blockDim.x) {
        const uint32_t k = g.first_job + i;
        const symgpu_mp3_job j = jobs[k];
        Head hd{kOutside, 0};
        if (job_in_range(j, n_bytes)) {
            symgpu::packet::MpaHeader h;
            size_t q;
            hd.q = kNone;
            if (me::read_header(bytes + j.offset, j.len, h, q) == me::kDecoded) {
                hd = Head{uint32_t(q), symgpu::packet::detail::be32(bytes + j.offset + q)};
                atomicMin(&first, k);
            }
        }
        heads[k] = hd;
        keys[k] = gi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Spec sp{first, 0, 0, 0};
        symgpu::packet::MpaHeader h;
        if (first != kNone && symgpu::packet::mpa_parse_header(heads[first].word, h) == symgpu::packet::Status::Ok)
            sp.rate = h.sample_rate, sp.channels = uint32_t(h.n_channels()), sp.granules = uint32_t(h.n_granules());
        spec[gi] = sp;
    }
}

__global__ void __launch_bounds__(128) mp3_side_kernel(const uint8_t* __restrict__ bytes, const symgpu_mp3_job* __restrict__ jobs, uint32_t n_jobs,
                                                       const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys,
                                                       const Head* __restrict__ heads, const Spec* __restrict__ spec,
                                                       const __grid_constant__ me::LongEdges E, me::FrameSide* __restrict__ sides,
                                                       uint8_t* __restrict__ bad, symgpu_pcm_span* __restrict__ spans1,
                                                       symgpu_pcm_span* __restrict__ spans2, uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    me::FrameSide s{};
    s.state = me::kSideRefused;
    uint8_t result = SYMGPU_MP3_JOB_REFUSED;
    if (gi != kNone) {
        const Head hd = heads[k];
        if (hd.q == kOutside) {
            result = SYMGPU_MP3_JOB_INVALID;
        } else if (hd.q != kNone) {
            const symgpu_mp3_job j = jobs[k];
            const DevGroup g = groups[gi];
            const Spec sp = spec[gi];
            symgpu::packet::MpaHeader h;
            symgpu::packet::mpa_parse_header(hd.word, h);  // parsed once already: Ok
            uint32_t at, n;
            if (sp.channels == g.channels && sp.granules == g.granules && h.sample_rate == sp.rate && uint32_t(h.n_channels()) == sp.channels &&
                me::body_of(h, 3, j.len, hd.q, at, n))
                me::read_frame_side(bytes + j.offset + at, at, n, h, E, s);
        }
    }
    sides[k] = s;
    bad[k] = 0;
    spans1[k] = spans2[k] = symgpu_pcm_span{};  // the walk writes the spans of the jobs a group names
    status[k] = result;
}

// One thread per group.  Round 0 walks every group; a later round walks only the groups whose Huffman pass failed, with the
// failed frame marked bad.  redo[gi] tells the gather and Huffman kernels which groups this round is for.
__global__ void __launch_bounds__(128) mp3_walk_kernel(const symgpu_mp3_job* __restrict__ jobs, const DevGroup* __restrict__ groups, uint32_t n_groups,
                                                       const Spec* __restrict__ spec, const me::FrameSide* __restrict__ sides, uint8_t* __restrict__ bad,
                                                       uint32_t* __restrict__ fail_job, uint8_t* __restrict__ redo, int round, me::GcJob* __restrict__ gc,
                                                       Copy* __restrict__ copies, uint32_t* __restrict__ slot_group, uint32_t* __restrict__ slot_job,
                                                       symgpu_pcm_span* __restrict__ spans1, symgpu_pcm_span* __restrict__ spans2,
                                                       symgpu_mp3_group_result* __restrict__ results, uint8_t* __restrict__ status) {
    const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n_groups) return;
    if (round > 0) {
        const uint32_t f = fail_job[gi];
        redo[gi] = f != kNone;
        if (f == kNone) return;
        bad[f] = 1, fail_job[gi] = kNone;
    } else {
        redo[gi] = 1, fail_job[gi] = kNone;
    }
    const DevGroup g = groups[gi];
    const Spec sp = spec[gi];
    const uint32_t per = 576u * g.granules;
    const uint64_t frame0 = g.out_offset / g.channels;
    me::Reservoir r{0, 0, g.frame_base * kMdPerSlot};
    uint32_t good = 0, back = 0;
    uint64_t frames = 0;
    for (uint32_t i = 0; i < g.n_jobs; ++i) {
        const uint32_t k = g.first_job + i;
        const me::FrameSide s = sides[k];
        const uint8_t b = bad[k];
        me::GcJob four[4];
        me::StepOut o{};
        const int step = me::reservoir_step(r, s, b ? b : (s.mismatch ? 2 : 0), 0, four, o);
        const bool real = step == me::kStepDecoded || step == me::kStepLeftOut;
        const uint64_t slot = g.frame_base + (step == me::kStepDecoded ? good++ : g.n_jobs - 1 - back++);
        if (real) {
            for (int q = 0; q < 4; ++q) four[q].out_index = uint32_t(slot * 4 + q);
        } else {
            for (int q = 0; q < 4; ++q) {
                four[q] = me::GcJob{};
                four[q].kind = me::kJobMute, four[q].out_index = uint32_t(slot * 4 + q);
            }
        }
        for (int q = 0; q < 4; ++q) gc[slot * 4 + q] = four[q];
        slot_group[slot] = gi, slot_job[slot] = real ? k : kNone;
        copies[k] = real ? Copy{o.copy_at, s.body_at + s.side_len, o.slot} : Copy{0, 0, 0};
        symgpu_pcm_span span{};
        if (step == me::kStepDecoded) {
            const symgpu_mp3_job j = jobs[k];
            const uint32_t ts = min(j.trim_start, per), te = min(j.trim_end, per - ts);
            span = symgpu_pcm_span{slot * 2304ull, 1152u, per, ts, te, frame0 + frames};
            frames += per - ts - te;
        }
        spans1[k] = g.channels == 1 ? span : symgpu_pcm_span{};
        spans2[k] = g.channels == 2 ? span : symgpu_pcm_span{};
        if (status[k] != SYMGPU_MP3_JOB_INVALID)
            status[k] = uint8_t(step == me::kStepDecoded ? SYMGPU_MP3_JOB_DECODED : step == me::kStepFailed ? SYMGPU_MP3_JOB_FAILED
                                : step == me::kStepLeftOut ? SYMGPU_MP3_JOB_LEFT_OUT : SYMGPU_MP3_JOB_REFUSED);
    }
    symgpu_mp3_group_result res{};
    res.frames = frames, res.packets = good, res.sample_rate = sp.rate, res.channels = uint8_t(sp.channels);
    results[gi] = res;
}

__global__ void __launch_bounds__(32 * kWarpsPerCta) mp3_gather_kernel(const uint8_t* __restrict__ bytes, const symgpu_mp3_job* __restrict__ jobs,
                                                                       uint32_t n_jobs, const uint32_t* __restrict__ keys,
                                                                       const uint8_t* __restrict__ redo, const Copy* __restrict__ copies,
                                                                       uint8_t* __restrict__ md) {
    const unsigned lane = threadIdx.x & 31;
    const uint32_t k = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    if (gi == kNone || !redo[gi]) return;
    const Copy c = copies[k];
    const uint8_t* src = bytes + jobs[k].offset + c.src;
    for (uint32_t i = lane; i < c.len; i += 32) md[c.dst + i] = src[i];
}

__global__ void __launch_bounds__(128) mp3_huffman_kernel(const uint8_t* __restrict__ md, const me::GcJob* __restrict__ gc, uint32_t n_gc, me::HuffSet hs,
                                                          const uint32_t* __restrict__ slot_group, const uint32_t* __restrict__ slot_job,
                                                          const uint8_t* __restrict__ redo, symgpu_mp3_gc* __restrict__ units,
                                                          int16_t* __restrict__ quant, uint32_t* __restrict__ fail_job, uint32_t* __restrict__ any_failed) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_gc) return;
    const uint32_t gi = slot_group[t >> 2];
    if (gi == kNone || !redo[gi]) return;
    const me::GcJob j = gc[t];
    if (me::decode_gc_job(j, md, hs, units + t, quant + size_t(t) * 576)) {
        atomicMin(fail_job + gi, slot_job[t >> 2]);
        atomicOr(any_failed, 1u);
    }
}

// Everything the host knows from the group table: the device records, the synthesis runs.
struct Layout {
    std::vector<DevGroup> dev;
    std::vector<symgpu_mp3_run> runs;
    uint64_t n_frames = 0;
};

symgpu_status check_groups(const symgpu_ctx* ctx, size_t n_jobs, const symgpu_mp3_group* groups, size_t n_groups, int format, size_t out_bytes, Layout& L) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    const uint64_t out_samples = out_bytes / sample;
    std::vector<JobRange> ranges;
    std::vector<uint32_t> slots;
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_mp3_group& G = groups[g];
        if ((G.granules != 1 && G.granules != 2) || (G.channels != 1 && G.channels != 2) || G.out_offset % G.channels) return SYMGPU_ERR_ARG;
        ranges.push_back({G.first_job, G.n_jobs});
        slots.push_back(G.slot);
    }
    symgpu_status e = check_job_ranges(ranges, n_jobs);
    if (e == SYMGPU_OK) e = check_slots(slots, ctx->n_mp3_streams);
    for (size_t g = 0; g < n_groups && e == SYMGPU_OK; ++g)
        e = check_region(groups[g].out_offset, uint64_t(groups[g].n_jobs) * groups[g].granules * 576u * groups[g].channels, out_samples);
    if (e != SYMGPU_OK) return e;
    L.dev.resize(n_groups);
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_mp3_group& G = groups[g];
        L.dev[g] = DevGroup{G.out_offset, L.n_frames, G.first_job, G.n_jobs, G.slot, G.granules, G.channels, {0, 0}};
        if (G.n_jobs) L.runs.push_back(symgpu_mp3_run{G.slot, uint32_t(L.n_frames), G.n_jobs, G.granules, G.channels, 0});
        L.n_frames += G.n_jobs;
    }
    return SYMGPU_OK;
}

// The device scratch at the start of ctx->d_stage.
struct Scratch {
    size_t groups, heads, keys, spec, sides, bad, copies, fail, redo, any, gc, slot_group, slot_job, md, units, quant, spectra, pcm, spans1, spans2, total;
};

Scratch scratch_layout(uint32_t n_jobs, size_t n_groups, const Layout& L) {
    Scratch s;
    Carver c;
    const size_t F = L.n_frames;
    s.groups = c.take(n_groups * sizeof(DevGroup));
    s.heads = c.take(n_jobs * sizeof(Head));
    s.keys = c.take(n_jobs * sizeof(uint32_t));
    s.spec = c.take(n_groups * sizeof(Spec));
    s.sides = c.take(n_jobs * sizeof(me::FrameSide));
    s.bad = c.take(n_jobs);
    s.copies = c.take(n_jobs * sizeof(Copy));
    s.fail = c.take(n_groups * sizeof(uint32_t));
    s.redo = c.take(n_groups);
    s.any = c.take(sizeof(uint32_t));
    s.gc = c.take(F * 4 * sizeof(me::GcJob));
    s.slot_group = c.take(F * sizeof(uint32_t));
    s.slot_job = c.take(F * sizeof(uint32_t));
    s.md = c.take(F * kMdPerSlot);
    s.units = c.take(F * 4 * sizeof(symgpu_mp3_gc));
    s.quant = c.take(F * SYMGPU_MP3_FRAME_FLOATS * sizeof(int16_t));
    s.spectra = c.take(F * SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
    s.pcm = c.take(F * SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
    s.spans1 = c.take(n_jobs * sizeof(symgpu_pcm_span));
    s.spans2 = c.take(n_jobs * sizeof(symgpu_pcm_span));
    s.total = c.at;
    return s;
}

// Everything after the staging: device pointers, n_jobs > 0, n_groups > 0, ctx->d_stage holds `s`.
symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const Layout& L, const uint8_t* bytes, size_t n_bytes, const symgpu_mp3_job* jobs,
                               uint32_t n_jobs, int format, void* out, symgpu_mp3_group_result* results, uint8_t* status, uint32_t* n_rounds) {
    char* stage = static_cast<char*>(ctx->d_stage);
    auto at = [&](size_t off) { return static_cast<void*>(stage + off); };
    DevGroup* groups = static_cast<DevGroup*>(at(s.groups));
    Head* heads = static_cast<Head*>(at(s.heads));
    uint32_t* keys = static_cast<uint32_t*>(at(s.keys));
    Spec* spec = static_cast<Spec*>(at(s.spec));
    me::FrameSide* sides = static_cast<me::FrameSide*>(at(s.sides));
    uint8_t* bad = static_cast<uint8_t*>(at(s.bad));
    Copy* copies = static_cast<Copy*>(at(s.copies));
    uint32_t* fail_job = static_cast<uint32_t*>(at(s.fail));
    uint8_t* redo = static_cast<uint8_t*>(at(s.redo));
    uint32_t* any = static_cast<uint32_t*>(at(s.any));
    me::GcJob* gc = static_cast<me::GcJob*>(at(s.gc));
    uint32_t* slot_group = static_cast<uint32_t*>(at(s.slot_group));
    uint32_t* slot_job = static_cast<uint32_t*>(at(s.slot_job));
    uint8_t* md = static_cast<uint8_t*>(at(s.md));
    symgpu_mp3_gc* units = static_cast<symgpu_mp3_gc*>(at(s.units));
    int16_t* quant = static_cast<int16_t*>(at(s.quant));
    float* spectra = static_cast<float*>(at(s.spectra));
    float* pcm = static_cast<float*>(at(s.pcm));
    symgpu_pcm_span* spans1 = static_cast<symgpu_pcm_span*>(at(s.spans1));
    symgpu_pcm_span* spans2 = static_cast<symgpu_pcm_span*>(at(s.spans2));
    const uint32_t n_groups = uint32_t(L.dev.size());
    const uint32_t n_gc = uint32_t(L.n_frames * 4);
    cudaStream_t st = ctx->stream;
    me::HuffSet hs;
    CU(ctx, symgpu::device_huffset(ctx->device, hs));
    CU(ctx, cudaMemcpyAsync(groups, L.dev.data(), n_groups * sizeof(DevGroup), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemsetAsync(keys, 0xff, n_jobs * sizeof(uint32_t), st));  // jobs no group names
    CU(ctx, cudaMemsetAsync(results, 0, n_groups * sizeof(symgpu_mp3_group_result), st));
    mp3_head_kernel<<<n_groups, 128, 0, st>>>(bytes, n_bytes, jobs, groups, heads, keys, spec, ctx->d_mp3_states);
    CU(ctx, cudaGetLastError());
    mp3_side_kernel<<<(n_jobs + 127) / 128, 128, 0, st>>>(bytes, jobs, n_jobs, groups, keys, heads, spec, symgpu::mp3_long_edges_host(), sides, bad, spans1, spans2,
                                                          status);
    CU(ctx, cudaGetLastError());
    ctx->launches += 2;
    uint32_t rounds = 0;
    for (;; ++rounds) {
        CU(ctx, cudaMemsetAsync(any, 0, sizeof(uint32_t), st));
        mp3_walk_kernel<<<(n_groups + 127) / 128, 128, 0, st>>>(jobs, groups, n_groups, spec, sides, bad, fail_job, redo, int(rounds), gc, copies,
                                                                slot_group, slot_job, spans1, spans2, results, status);
        CU(ctx, cudaGetLastError());
        mp3_gather_kernel<<<(n_jobs + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, st>>>(bytes, jobs, n_jobs, keys, redo, copies, md);
        CU(ctx, cudaGetLastError());
        mp3_huffman_kernel<<<(n_gc + 127) / 128, 128, 0, st>>>(md, gc, n_gc, hs, slot_group, slot_job, redo, units, quant, fail_job, any);
        CU(ctx, cudaGetLastError());
        ctx->launches += 3;
        uint32_t again = 0;
        CU(ctx, cudaMemcpyAsync(&again, any, sizeof again, cudaMemcpyDeviceToHost, st));
        CU(ctx, cudaStreamSynchronize(st));
        if (!again) break;
    }
    if (n_rounds) *n_rounds = rounds + 1;
    CU(ctx, symgpu::dequant_launch(quant, spectra, L.n_frames * SYMGPU_MP3_FRAME_FLOATS, ctx->d_mp3_tab->pow43, st));
    ctx->launches += 1;
    if (!L.runs.empty()) {
        const symgpu_status e = symgpu_mp3_synth_dev(ctx, units, spectra, L.runs.data(), uint32_t(L.runs.size()), uint32_t(L.n_frames), pcm);
        if (e != SYMGPU_OK) return e;
    }
    for (uint32_t ch = 1; ch <= 2; ++ch) {
        const symgpu_status e = symgpu_pcm_pack_dev(ctx, pcm, ch == 1 ? spans1 : spans2, n_jobs, ch, 1152, 1152, format, out);
        if (e != SYMGPU_OK) return e;
    }
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x3fffffff;  // four granule-channel indices per frame slot fit in 32 bits

}  // namespace

extern "C" symgpu_status symgpu_mp3_decode_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_mp3_job* jobs, size_t n_jobs,
                                               const symgpu_mp3_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                               symgpu_mp3_group_result* results, uint8_t* status, uint32_t* n_rounds) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff)
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    if (n_rounds) *n_rounds = 0;
    DeviceGuard guard(ctx->device);
    if (n_jobs == 0 || n_groups == 0) {
        if (n_groups) CU(ctx, cudaMemsetAsync(results, 0, n_groups * sizeof(symgpu_mp3_group_result), ctx->stream));
        if (n_jobs) CU(ctx, cudaMemsetAsync(status, SYMGPU_MP3_JOB_REFUSED, n_jobs, ctx->stream));
        return SYMGPU_OK;
    }
    const Scratch s = scratch_layout(uint32_t(n_jobs), n_groups, L);
    e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    return decode_on_device(ctx, s, L, bytes, n_bytes, jobs, uint32_t(n_jobs), format, out, results, status, n_rounds);
}

extern "C" symgpu_status symgpu_mp3_decode_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_mp3_job* jobs, size_t n_jobs,
                                                const symgpu_mp3_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                symgpu_mp3_group_result* results, uint8_t* status, uint32_t* n_rounds) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff ||
        !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    for (size_t g = 0; g < n_groups; ++g) results[g] = symgpu_mp3_group_result{};
    for (size_t k = 0; k < n_jobs; ++k) status[k] = SYMGPU_MP3_JOB_REFUSED;
    if (n_rounds) *n_rounds = 0;
    if (n_jobs == 0 || n_groups == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const Scratch s = scratch_layout(uint32_t(n_jobs), n_groups, L);
    return decode_from_host(
        ctx, s.total, std::array<HostIn, 2>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_mp3_job)}}}, out, out_bytes,
        std::array<HostOut, 2>{{{status, n_jobs}, {results, n_groups * sizeof(symgpu_mp3_group_result)}}},
        [&](const std::array<void*, 2>& in, void* d_out, const std::array<void*, 2>& back) {
            return decode_on_device(ctx, s, L, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_mp3_job*>(in[1]), uint32_t(n_jobs),
                                    format, d_out, static_cast<symgpu_mp3_group_result*>(back[1]), static_cast<uint8_t*>(back[0]), n_rounds);
        },
        [&] { return written_by_results(groups, results, n_groups, symgpu_sample_bytes(format)); });
}
