// MPEG Layer I / II decoded on the device, many files per call (include/symgpu.h "MPEG Layer I / II decoded on the device";
// DESIGN §5d).  A file is a group, a packet is a job.
//
//   mpa12_head_kernel     one CTA per group: resets the group's synthesis state slot; one thread per job runs the packet
//                         prologue (sync search, header, length); the group's first job that passes fixes (rate, channels)
//   mpa12_side_kernel     one thread per job: the signal specification, the layer check, the side read and the fit rule of
//                         mpa12_entropy.h -> the job's side record, accepted or not, and its frames after the trims
//   scan by group         accepted (count, frames) -> each frame's place in its group and its first output frame
//   mpa12_sample_kernel   one warp per job: the frame's sample codewords, each at its closed-form bit position, decoded by
//                         the lanes in parallel -> [frame][2][32][n_slots]; the output spans; the group's result
//   symgpu_mpa12_synth_dev   unchanged, once per layer present; every group is one run of n_jobs frames at 2 channels
//   symgpu_pcm_pack_dev      unchanged, once for the mono and once for the stereo groups
//
// Frame slots: a group owns n_jobs consecutive slots.  Its accepted frames take the first ones in stream order; the slots
// of refused packets come after them, zeroed, so they cannot change the PCM of the real frames (the synthesis runs them
// last).  The synthesis plan is built on the host from the group table alone, before anything is decoded, so the call
// makes no host round trip.  Layer I slots come first in the frame buffers, then Layer II slots.
#include <cuda_runtime.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>
#include <numeric>
#include <vector>

#include "batch_call.h"
#include "mp3_kernel.h"
#include "mpa12_entropy.h"

using namespace symgpu_detail;
namespace me = symgpu::mpa12e;

namespace {

constexpr uint32_t kNone = 0xffffffffu;      // no group / no packet fixed the specification / the header was refused
constexpr uint32_t kOutside = 0xfffffffeu;   // Head::q of a job outside `bytes`
constexpr int kWarpsPerCta = 4;

struct DevGroup {  // 32 bytes: symgpu_mpa12_group + the group's first frame slot
    uint64_t out_offset;
    uint64_t frame_base;
    uint32_t first_job, n_jobs, slot;
    uint8_t layer, reserved[3];
};
struct Spec {
    uint32_t job, rate, channels, reserved;
};
struct Head {
    uint32_t q;     // the header's byte offset in the packet; kNone: refused by the prologue, kOutside: outside `bytes`
    uint32_t word;  // the header word
};
struct Place {
    unsigned long long frames;  // frames after the trims
    unsigned long long count;   // accepted packets
};
struct PlaceSum {
    __host__ __device__ Place operator()(const Place& a, const Place& b) const { return Place{a.frames + b.frames, a.count + b.count}; }
};

__device__ __forceinline__ bool job_in_range(const symgpu_mpa12_job& j, size_t n_bytes) { return j.offset <= n_bytes && j.len <= n_bytes - j.offset; }

__global__ void __launch_bounds__(128) mpa12_head_kernel(const uint8_t* __restrict__ bytes, size_t n_bytes, const symgpu_mpa12_job* __restrict__ jobs,
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
        const symgpu_mpa12_job j = jobs[k];
        Head hd{kOutside, 0};
        if (job_in_range(j, n_bytes)) {
            me::MpaHeader h;
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
        me::MpaHeader h;
        if (first != kNone && symgpu::packet::mpa_parse_header(heads[first].word, h) == symgpu::packet::Status::Ok)
            sp.rate = h.sample_rate, sp.channels = uint32_t(h.n_channels());
        spec[gi] = sp;
    }
}

__global__ void __launch_bounds__(128) mpa12_side_kernel(const uint8_t* __restrict__ bytes, const symgpu_mpa12_job* __restrict__ jobs, uint32_t n_jobs,
                                                         const DevGroup* __restrict__ groups, const uint32_t* __restrict__ keys,
                                                         const Head* __restrict__ heads, const Spec* __restrict__ spec,
                                                         const __grid_constant__ me::Constants K, me::Side* __restrict__ sides,
                                                         Place* __restrict__ place_in, uint8_t* __restrict__ status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    Place p{0, 0};
    uint8_t result = SYMGPU_MPA12_JOB_REFUSED;
    if (gi != kNone) {
        const Head hd = heads[k];
        if (hd.q == kOutside) {
            result = SYMGPU_MPA12_JOB_INVALID;
        } else if (hd.q != kNone) {
            const symgpu_mpa12_job j = jobs[k];
            const DevGroup g = groups[gi];
            const Spec sp = spec[gi];
            me::MpaHeader h;
            symgpu::packet::mpa_parse_header(hd.word, h);  // parsed once already: Ok
            me::Side& s = sides[k];
            uint32_t at, n;
            if (h.sample_rate == sp.rate && uint32_t(h.n_channels()) == sp.channels && me::body_of(h, g.layer, j.len, hd.q, at, n)) {
                s.body_at = at, s.body_bytes = n;
                if (me::read_side(K, bytes + j.offset + at, h, s) && me::fits(s)) {
                    const uint32_t per = g.layer == 1 ? 384u : 1152u;
                    const uint32_t ts = min(j.trim_start, per), te = min(j.trim_end, per - ts);
                    p = Place{per - ts - te, 1};
                    result = SYMGPU_MPA12_JOB_DECODED;
                }
            }
        }
    }
    place_in[k] = p;
    status[k] = result;
}

__device__ __forceinline__ float* frame_ptr(float* sub, uint64_t f, uint64_t n_l1) {
    return f < n_l1 ? sub + f * (64 * 12) : sub + n_l1 * (64 * 12) + (f - n_l1) * (64 * 36);
}

__global__ void __launch_bounds__(32 * kWarpsPerCta) mpa12_sample_kernel(const uint8_t* __restrict__ bytes, const symgpu_mpa12_job* __restrict__ jobs,
                                                                         uint32_t n_jobs, const DevGroup* __restrict__ groups,
                                                                         const uint32_t* __restrict__ keys, const Spec* __restrict__ spec,
                                                                         const __grid_constant__ me::Constants K, const me::Side* __restrict__ sides,
                                                                         const Place* __restrict__ place, const uint8_t* __restrict__ status,
                                                                         float* __restrict__ sub, uint64_t n_l1, symgpu_pcm_span* __restrict__ spans1,
                                                                         symgpu_pcm_span* __restrict__ spans2, symgpu_mpa12_group_result* __restrict__ results) {
    __shared__ me::Side side_s[kWarpsPerCta];
    __shared__ __align__(16) float frame_s[kWarpsPerCta][64 * 36];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t k = blockIdx.x * kWarpsPerCta + warp;
    if (k >= n_jobs) return;
    const uint32_t gi = keys[k];
    if (gi == kNone) {
        if (lane == 0) spans1[k] = spans2[k] = symgpu_pcm_span{};
        return;
    }
    const DevGroup g = groups[gi];
    const Place pl = place[k];
    const bool accepted = status[k] == SYMGPU_MPA12_JOB_DECODED;
    const int n_slots = g.layer == 1 ? 12 : 36, per = g.layer == 1 ? 1 : 3;
    // accepted frames first in stream order, refused packets' slots from the back
    const uint64_t slot = g.frame_base + (accepted ? pl.count : g.n_jobs - 1 - ((k - g.first_job) - pl.count));
    float4* dst = reinterpret_cast<float4*>(frame_ptr(sub, slot, n_l1));
    const unsigned quads = 64 * n_slots / 4;
    if (!accepted) {
        for (unsigned i = lane; i < quads; i += 32) dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
        me::Side& s = side_s[warp];
        const uint32_t* from = reinterpret_cast<const uint32_t*>(sides + k);
        uint32_t* to = reinterpret_cast<uint32_t*>(&s);
        for (unsigned i = lane; i < sizeof(me::Side) / 4; i += 32) to[i] = from[i];
        __syncwarp();
        const uint8_t* body = bytes + jobs[k].offset + s.body_at;
        float* f = frame_s[warp];
        // 64 rows (channel, sub-band) x 12 granules, each item one codeword (Layer I one sample, Layer II three)
        for (unsigned i = lane; i < 64 * 12; i += 32) {
            const unsigned row = i / 12, gr = i - row * 12, c = row >> 5, sb = row & 31;
            float* o = f + row * n_slots + gr * per;
            if (c < s.n_ch) {
                me::decode_codeword(K, s, body, int(gr), int(sb), int(c), o);  // cannot fail: the side pass checked fits()
            } else {
                for (int t = 0; t < per; ++t) o[t] = 0.0f;
            }
        }
        __syncwarp();
        const float4* f4 = reinterpret_cast<const float4*>(f);
        for (unsigned i = lane; i < quads; i += 32) dst[i] = f4[i];
    }
    if (lane == 0) {
        const Spec sp = spec[gi];
        const symgpu_mpa12_job j = jobs[k];
        const uint32_t frames = g.layer == 1 ? 384u : 1152u;
        symgpu_pcm_span span{};
        if (accepted) {
            const uint32_t ts = min(j.trim_start, frames), te = min(j.trim_end, frames - ts);
            span = symgpu_pcm_span{slot * 2304ull, 1152u, frames, ts, te, g.out_offset / sp.channels + pl.frames};
        }
        spans1[k] = sp.channels == 1 ? span : symgpu_pcm_span{};
        spans2[k] = sp.channels == 2 ? span : symgpu_pcm_span{};
        if (k == g.first_job + g.n_jobs - 1) {  // the group's last job knows its totals
            const Place own = accepted ? Place{frames - span.trim_start - span.trim_end, 1} : Place{0, 0};
            symgpu_mpa12_group_result r{};
            r.frames = pl.frames + own.frames, r.packets = uint32_t(pl.count + own.count);
            r.sample_rate = sp.rate, r.channels = uint8_t(sp.channels);
            results[gi] = r;
        }
    }
}

cudaError_t scan_place(void* temp, size_t& temp_bytes, const uint32_t* keys, const Place* in, Place* out, uint32_t n_jobs, cudaStream_t st) {
    return cub::DeviceScan::ExclusiveScanByKey(temp, temp_bytes, keys, in, out, PlaceSum(), Place{0, 0}, int(n_jobs), cuda::std::equal_to<>(), st);
}

// Everything the host knows from the group table: the device records, the synthesis runs of each layer.
struct Layout {
    std::vector<DevGroup> dev;
    std::vector<symgpu_mpa12_run> runs[2];
    uint64_t n_frames[2] = {0, 0};
};

symgpu_status check_groups(const symgpu_ctx* ctx, size_t n_jobs, const symgpu_mpa12_group* groups, size_t n_groups, int format, size_t out_bytes,
                           Layout& L) {
    const size_t sample = symgpu_sample_bytes(format);
    if (sample == 0) return SYMGPU_ERR_ARG;
    const uint64_t out_samples = out_bytes / sample;
    std::vector<JobRange> ranges;
    std::vector<uint32_t> slots;
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_mpa12_group& G = groups[g];
        if ((G.layer != 1 && G.layer != 2) || (G.out_offset & 1)) return SYMGPU_ERR_ARG;
        ranges.push_back({G.first_job, G.n_jobs});
        slots.push_back(G.slot);
    }
    symgpu_status e = check_job_ranges(ranges, n_jobs);
    if (e == SYMGPU_OK) e = check_slots(slots, ctx->n_mp3_streams);
    for (size_t g = 0; g < n_groups && e == SYMGPU_OK; ++g)
        e = check_region(groups[g].out_offset, 2ull * groups[g].n_jobs * (groups[g].layer == 1 ? 384u : 1152u), out_samples);
    if (e != SYMGPU_OK) return e;
    for (size_t g = 0; g < n_groups; ++g) L.n_frames[groups[g].layer - 1] += groups[g].n_jobs;
    uint64_t base[2] = {0, L.n_frames[0]};
    L.dev.resize(n_groups);
    for (size_t g = 0; g < n_groups; ++g) {
        const symgpu_mpa12_group& G = groups[g];
        const int l = G.layer - 1;
        L.dev[g] = DevGroup{G.out_offset, base[l], G.first_job, G.n_jobs, G.slot, G.layer, {0, 0, 0}};
        if (G.n_jobs) L.runs[l].push_back(symgpu_mpa12_run{G.slot, uint32_t(base[l] - (l ? L.n_frames[0] : 0)), G.n_jobs, 2, {0, 0, 0}});
        base[l] += G.n_jobs;
    }
    return SYMGPU_OK;
}

// The device scratch at the start of ctx->d_stage.
struct Scratch {
    size_t groups, heads, keys, spec, sides, place_in, place, sub, pcm, spans1, spans2, temp, total;
    size_t temp_bytes;
};

cudaError_t scratch_layout(uint32_t n_jobs, size_t n_groups, const Layout& L, Scratch& s) {
    cudaError_t e = scan_place(nullptr, s.temp_bytes, nullptr, nullptr, nullptr, n_jobs, nullptr);
    if (e != cudaSuccess) return e;
    Carver c;
    s.groups = c.take(n_groups * sizeof(DevGroup));
    s.heads = c.take(n_jobs * sizeof(Head));
    s.keys = c.take(n_jobs * sizeof(uint32_t));
    s.spec = c.take(n_groups * sizeof(Spec));
    s.sides = c.take(n_jobs * sizeof(me::Side));
    s.place_in = c.take(n_jobs * sizeof(Place));
    s.place = c.take(n_jobs * sizeof(Place));
    s.sub = c.take((L.n_frames[0] * 64 * 12 + L.n_frames[1] * 64 * 36) * sizeof(float));
    s.pcm = c.take(size_t(L.n_frames[0] + L.n_frames[1]) * SYMGPU_MP3_FRAME_FLOATS * sizeof(float));
    s.spans1 = c.take(n_jobs * sizeof(symgpu_pcm_span));
    s.spans2 = c.take(n_jobs * sizeof(symgpu_pcm_span));
    s.temp = c.take(s.temp_bytes);
    s.total = c.at;
    return cudaSuccess;
}

// Everything after the staging: device pointers, n_jobs > 0, n_groups > 0, ctx->d_stage holds `s`.
symgpu_status decode_on_device(symgpu_ctx* ctx, const Scratch& s, const Layout& L, const uint8_t* bytes, size_t n_bytes, const symgpu_mpa12_job* jobs,
                               uint32_t n_jobs, int format, void* out, symgpu_mpa12_group_result* results, uint8_t* status) {
    char* stage = static_cast<char*>(ctx->d_stage);
    DevGroup* groups = reinterpret_cast<DevGroup*>(stage + s.groups);
    Head* heads = reinterpret_cast<Head*>(stage + s.heads);
    uint32_t* keys = reinterpret_cast<uint32_t*>(stage + s.keys);
    Spec* spec = reinterpret_cast<Spec*>(stage + s.spec);
    me::Side* sides = reinterpret_cast<me::Side*>(stage + s.sides);
    Place* place_in = reinterpret_cast<Place*>(stage + s.place_in);
    Place* place = reinterpret_cast<Place*>(stage + s.place);
    float* sub = reinterpret_cast<float*>(stage + s.sub);
    float* pcm = reinterpret_cast<float*>(stage + s.pcm);
    symgpu_pcm_span* spans1 = reinterpret_cast<symgpu_pcm_span*>(stage + s.spans1);
    symgpu_pcm_span* spans2 = reinterpret_cast<symgpu_pcm_span*>(stage + s.spans2);
    void* temp = stage + s.temp;
    size_t temp_bytes = s.temp_bytes;
    const size_t n_groups = L.dev.size();
    cudaStream_t st = ctx->stream;
    const me::Constants& K = me::host_constants();
    CU(ctx, cudaMemcpyAsync(groups, L.dev.data(), n_groups * sizeof(DevGroup), cudaMemcpyHostToDevice, st));
    CU(ctx, cudaMemsetAsync(keys, 0xff, n_jobs * sizeof(uint32_t), st));  // jobs no group names
    CU(ctx, cudaMemsetAsync(results, 0, n_groups * sizeof(symgpu_mpa12_group_result), st));
    mpa12_head_kernel<<<unsigned(n_groups), 128, 0, st>>>(bytes, n_bytes, jobs, groups, heads, keys, spec, ctx->d_mp3_states);
    CU(ctx, cudaGetLastError());
    mpa12_side_kernel<<<(n_jobs + 127) / 128, 128, 0, st>>>(bytes, jobs, n_jobs, groups, keys, heads, spec, K, sides, place_in, status);
    CU(ctx, cudaGetLastError());
    CU(ctx, scan_place(temp, temp_bytes, keys, place_in, place, n_jobs, st));
    mpa12_sample_kernel<<<(n_jobs + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, st>>>(bytes, jobs, n_jobs, groups, keys, spec, K, sides, place, status,
                                                                                                  sub, L.n_frames[0], spans1, spans2, results);
    CU(ctx, cudaGetLastError());
    ctx->launches += 5;  // three kernels here, two for the device-wide scan
    for (int l = 0; l < 2; ++l) {
        if (L.runs[l].empty()) continue;
        const uint32_t n_slots = l == 0 ? 12 : 36;
        const symgpu_status e = symgpu_mpa12_synth_dev(ctx, l == 0 ? sub : sub + L.n_frames[0] * 64 * 12, L.runs[l].data(), uint32_t(L.runs[l].size()),
                                                       uint32_t(L.n_frames[l]), n_slots, l == 0 ? pcm : pcm + L.n_frames[0] * SYMGPU_MP3_FRAME_FLOATS);
        if (e != SYMGPU_OK) return e;
    }
    for (uint32_t ch = 1; ch <= 2; ++ch) {
        const symgpu_status e = symgpu_pcm_pack_dev(ctx, pcm, ch == 1 ? spans1 : spans2, n_jobs, ch, 1152, 1152, format, out);
        if (e != SYMGPU_OK) return e;
    }
    return SYMGPU_OK;
}

constexpr size_t kMaxJobs = 0x7fffffff;  // the device-wide scan counts items in an int

}  // namespace

extern "C" symgpu_status symgpu_mpa12_decode_dev(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_mpa12_job* jobs, size_t n_jobs,
                                                 const symgpu_mpa12_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                 symgpu_mpa12_group_result* results, uint8_t* status) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff)
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    DeviceGuard guard(ctx->device);
    if (n_jobs == 0 || n_groups == 0) {
        if (n_groups) CU(ctx, cudaMemsetAsync(results, 0, n_groups * sizeof(symgpu_mpa12_group_result), ctx->stream));
        if (n_jobs) CU(ctx, cudaMemsetAsync(status, SYMGPU_MPA12_JOB_REFUSED, n_jobs, ctx->stream));
        return SYMGPU_OK;
    }
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), n_groups, L, s));
    e = ensure_stage(ctx, s.total);
    if (e != SYMGPU_OK) return e;
    return decode_on_device(ctx, s, L, bytes, n_bytes, jobs, uint32_t(n_jobs), format, out, results, status);
}

extern "C" symgpu_status symgpu_mpa12_decode_host(symgpu_ctx* ctx, const uint8_t* bytes, size_t n_bytes, const symgpu_mpa12_job* jobs, size_t n_jobs,
                                                  const symgpu_mpa12_group* groups, size_t n_groups, int format, void* out, size_t out_bytes,
                                                  symgpu_mpa12_group_result* results, uint8_t* status) {
    if (bad_batch_args(ctx, bytes, n_bytes, jobs, n_jobs, groups, n_groups, out, out_bytes, results, status, kMaxJobs) || n_groups > 0x7fffffff ||
        !jobs_in_bytes(jobs, n_jobs, n_bytes))
        return SYMGPU_ERR_ARG;
    Layout L;
    symgpu_status e = check_groups(ctx, n_jobs, groups, n_groups, format, out_bytes, L);
    if (e != SYMGPU_OK) return e;
    for (size_t g = 0; g < n_groups; ++g) results[g] = symgpu_mpa12_group_result{};
    for (size_t k = 0; k < n_jobs; ++k) status[k] = SYMGPU_MPA12_JOB_REFUSED;
    if (n_jobs == 0 || n_groups == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    Scratch s;
    CU(ctx, scratch_layout(uint32_t(n_jobs), n_groups, L, s));
    return decode_from_host(
        ctx, s.total, std::array<HostIn, 2>{{{bytes, n_bytes}, {jobs, n_jobs * sizeof(symgpu_mpa12_job)}}}, out, out_bytes,
        std::array<HostOut, 2>{{{status, n_jobs}, {results, n_groups * sizeof(symgpu_mpa12_group_result)}}},
        [&](const std::array<void*, 2>& in, void* d_out, const std::array<void*, 2>& back) {
            return decode_on_device(ctx, s, L, static_cast<const uint8_t*>(in[0]), n_bytes, static_cast<const symgpu_mpa12_job*>(in[1]), uint32_t(n_jobs),
                                    format, d_out, static_cast<symgpu_mpa12_group_result*>(back[1]), static_cast<uint8_t*>(back[0]));
        },
        [&] { return written_by_results(groups, results, n_groups, symgpu_sample_bytes(format)); });
}
