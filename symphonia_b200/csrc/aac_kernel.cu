// AAC-LC synthesis for sm_90a: TNS (aac/ics/tns.rs:149-199) then the filterbank of Dsp::synth
// (aac/dsp.rs:57-158): 1024-point or 8 x 128-point IMDCT, sine / KBD windows, the four window
// sequences, overlap-add through the per-channel `delay` line.
//
// Work decomposition (DESIGN.md §4): `delay` is overwritten from the current frame only, so a
// channel's frames are cut into chunks of consecutive frames; a persistent CTA walks chunks, one group of
// 64 threads per frame of the chunk plus one for the frame before it (whose IMDCT output is the delay
// line the chunk's first frame overlaps with; a run's first chunk takes it from the stream state).
// TNS is a serial recurrence along frequency: it runs in a pre-pass, one LANE per filter, on a scratch
// copy of the channel-frames that carry filters.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <type_traits>

#include "../../include/symgpu.h"
#include "codec_kernels.h"
#include "imdct.cuh"
#include "tables.h"

namespace symgpu {
namespace {

constexpr int P0 = 512 - 64, P1 = 512 + 64; // SHORT_WIN_POINT0/1, aac/dsp.rs:19-20

// ---- TNS ------------------------------------------------------------------------------------
// coeffs[i] -= coeffs[i -/+ (j+1)] * lpc[j], j ascending, in place (tns.rs:183-196): an all-pole recurrence
// along frequency, serial per filter (one product on the previous output, then ORDER dependent
// subtractions per line).  Filters are independent of each other, so the pre-pass packs one filter per LANE:
//   aac_tns_prepare  copies the spectra of the channel-frames that carry filters into the scratch buffer
//                    and records, for every filter, the channel-frame it belongs to;
//   aac_tns_sort     counting sort of the filter indices by order, so that the lanes of a warp run the
//                    same instantiation;
//   aac_tns_apply    lane = filter, in place in the scratch buffer.
// The filterbank kernel then reads those channel-frames from the scratch buffer.
// One line with the full history (GUARD = false) or, for the first lines of a filter, with the `order.min(m)`
// terms the reference uses (tns.rs:187, :193; subtracting a zero product instead would turn a -0.0 input into
// +0.0 when the coefficient is negative).  h[j] = the output j + 1 lines back.
template <int ORDER, bool GUARD>
__device__ __forceinline__ float tns_line(float v, int m, float (&h)[20], const float (&lpc)[20]) {
#pragma unroll
    for (int j = 0; j < ORDER; ++j)
        if (!GUARD || j < m) v -= h[j] * lpc[j];
#pragma unroll
    for (int j = ORDER - 1; j > 0; --j) h[j] = h[j - 1];
    h[0] = v;
    return v;
}

// `cnt` consecutive lines of one filter, held in a column of the warp's tile (row stride 33 floats).
template <int ORDER>
__device__ __forceinline__ void tns_lines(float* col, int cnt, int m0, float (&h)[20], const float (&lpc)[20], int stride = 33) {
    int k = 0;
    for (; k < cnt && m0 + k < ORDER; ++k) col[stride * k] = tns_line<ORDER, true>(col[stride * k], m0 + k, h, lpc);
    // Main part: trips of L lines (a multiple of ORDER) with the history in a ring of ORDER registers -- c[r % ORDER] is the
    // output of the trip's line r, so the output j + 1 lines back sits at c[(r - 1 - j) mod ORDER] with every index known at
    // compile time: no register moves between lines (the shifting form below spends ORDER of its ~3.3 ORDER instructions per
    // line on them).  Same operations on the same operands in the same order.
    constexpr int L = ORDER >= 4 ? ORDER : ORDER == 3 ? 6 : 4;
#ifndef SYMGPU_TNS_NO_RING // (A/B switch: TNS history in shared memory instead of the register ring)
    if (k + L <= cnt) {
        float c[ORDER];
#pragma unroll
        for (int j = 0; j < ORDER; ++j) c[ORDER - 1 - j] = h[j];
        for (; k + L <= cnt; k += L) {
            float x[L];
#pragma unroll
            for (int r = 0; r < L; ++r) x[r] = col[stride * (k + r)];
#pragma unroll
            for (int r = 0; r < L; ++r) {
                float v = x[r];
#pragma unroll
                for (int j = 0; j < ORDER; ++j) v -= c[(r + 2 * L - 1 - j) % ORDER] * lpc[j];
                c[r % ORDER] = v;
                x[r] = v;
            }
#pragma unroll
            for (int r = 0; r < L; ++r) col[stride * (k + r)] = x[r];
        }
#pragma unroll
        for (int j = 0; j < ORDER; ++j) h[j] = c[ORDER - 1 - j];
    }
#endif
    for (; k < cnt; ++k) col[stride * k] = tns_line<ORDER, false>(col[stride * k], 0, h, lpc);
}

// One whole filter by one thread, in place on a channel-frame's 1024 lines in shared memory (the Z kernel runs the filters of a
// frame on the lanes of the frame's own warp, one filter per lane, before its IMDCT).  Out of line: its twenty instantiations
// and their registers stay out of the filterbank's code.
// (TAG: one copy per calling kernel, so that the 64-register budget of the Z kernel does not bind the pre-pass kernel's copy.)
template <int TAG>
__device__ __noinline__ void tns_filter_in_place(float* lines, const symgpu_aac_tns* __restrict__ t) {
    int start = t->start, end = t->end;
    if (end > 1024) end = 1024; // a malformed filter must not leave its channel-frame
    const int order = t->order;
    if (!(start < end) || order < 1 || order > 20) return;
    const bool down = t->direction != 0;
    float lpc[20], h[20];
#pragma unroll
    for (int j = 0; j < 20; ++j) {
        h[j] = 0.0f;
        lpc[j] = j < order ? __ldg(t->lpc + j) : 0.0f;
    }
    float* first = lines + (down ? end - 1 : start);
    const int stride = down ? -1 : 1, len = end - start;
    switch (order) {
#define TNS_CASE(N) case N: tns_lines<N>(first, len, 0, h, lpc, stride); break;
        TNS_CASE(1) TNS_CASE(2) TNS_CASE(3) TNS_CASE(4) TNS_CASE(5) TNS_CASE(6) TNS_CASE(7) TNS_CASE(8) TNS_CASE(9)
        TNS_CASE(10) TNS_CASE(11) TNS_CASE(12) TNS_CASE(13) TNS_CASE(14) TNS_CASE(15) TNS_CASE(16) TNS_CASE(17)
        TNS_CASE(18) TNS_CASE(19) TNS_CASE(20)
#undef TNS_CASE
        default: break;
    }
}

// The pre-pass in ONE kernel (the default): a warp per channel-frame that carries filters moves the frame's 1024 lines into
// shared memory (coalesced), runs its filters there, one per lane -- a long frame has at most 3, eight short windows at most 8,
// and together they cover at most the frame's TNS band range, so a warp's serial work is bounded by ~670 lines -- and writes the
// lines to the scratch buffer (coalesced).  No sort, no owner table, no 32-line transposition rounds: the three-kernel pre-pass
// below spent three quarters of its apply kernel moving lines in and out of its tiles.
constexpr int kTnsFrameWarps = 8;
__global__ void __launch_bounds__(kTnsFrameWarps * 32) aac_tns_frames(const symgpu_aac_unit* __restrict__ units, const symgpu_aac_tns* __restrict__ tns,
                                                                     uint32_t n_tns, const float* __restrict__ coeffs, float* __restrict__ scratch,
                                                                     uint32_t n_units) {
    __shared__ __align__(16) float lines_s[kTnsFrameWarps][1024];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t u = blockIdx.x * kTnsFrameWarps + warp;
    if (u >= n_units) return;
    const symgpu_aac_unit unit = units[u];
    if (unit.n_tns == 0) return;
    float* lines = lines_s[warp];
    const float4* src = reinterpret_cast<const float4*>(coeffs + (size_t)u * 1024);
    float4* dst = reinterpret_cast<float4*>(scratch + (size_t)u * 1024);
#pragma unroll
    for (int i = 0; i < 8; ++i) reinterpret_cast<float4*>(lines)[lane + 32 * i] = __ldg(src + lane + 32 * i);
    __syncwarp();
    for (uint32_t f = lane; f < unit.n_tns; f += 32)
        if (unit.tns_first + f < n_tns) tns_filter_in_place<0>(lines, tns + unit.tns_first + f);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[lane + 32 * i] = reinterpret_cast<const float4*>(lines)[lane + 32 * i];
}

// ---- the three-kernel pre-pass of round 1 (SYMGPU_AAC_TNS=sorted) ----
// One warp per channel-frame: copy the spectra that carry filters, note the owner of each filter.
__global__ void __launch_bounds__(256) aac_tns_prepare(const symgpu_aac_unit* __restrict__ units, const float* __restrict__ coeffs,
                                                       float* __restrict__ scratch, uint32_t* __restrict__ owner, uint32_t n_units,
                                                       uint32_t n_tns) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t u = blockIdx.x * 8 + warp;
    if (u >= n_units) return;
    const symgpu_aac_unit unit = units[u];
    if (unit.n_tns == 0) return;
    const float4* src = reinterpret_cast<const float4*>(coeffs + (size_t)u * 1024);
    float4* dst = reinterpret_cast<float4*>(scratch + (size_t)u * 1024);
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[lane + 32 * i] = __ldg(src + lane + 32 * i);
    for (uint32_t f = lane; f < unit.n_tns; f += 32)
        if (unit.tns_first + f < n_tns) owner[unit.tns_first + f] = u;
}

// Counting sort of filter indices by order (one CTA; a batch holds a few thousand filters).  Lanes that hold
// the same order are found with match.any and send ONE shared-memory atomic per group; the orders are read
// eight at a time so that the strided global loads overlap.
__global__ void __launch_bounds__(1024) aac_tns_sort(const symgpu_aac_tns* __restrict__ tns, uint32_t n_tns, uint32_t* __restrict__ sorted) {
    __shared__ uint32_t bin[32];
    const unsigned lane = threadIdx.x & 31;
    if (threadIdx.x < 32) bin[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t n_pad = (n_tns + 31u) & ~31u; // whole warps enter the collectives
    // Batches of 8 * blockDim filters; the orders of a batch stay in registers between the two passes when the
    // whole list is one batch (the usual case), otherwise they are read again.
    const bool one_batch = n_pad <= 8 * blockDim.x;
    int keep[8];
    for (int pass = 0; pass < 2; ++pass) {
        for (uint32_t f0 = threadIdx.x; f0 < n_pad; f0 += 8 * blockDim.x) {
            int o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t f = f0 + k * blockDim.x;
                if (pass == 1 && one_batch) o[k] = keep[k];
                else o[k] = f < n_tns ? min((int)tns[f].order, 30) : 31;
                keep[k] = o[k];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t f = f0 + k * blockDim.x;
                if (f - lane >= n_pad) continue; // warp-uniform
                const unsigned peers = __match_any_sync(0xffffffffu, o[k]);
                const int leader = __ffs(peers) - 1;
                uint32_t base = 0;
                if ((int)lane == leader) base = atomicAdd(&bin[o[k]], (uint32_t)__popc(peers));
                if (pass == 1) {
                    base = __shfl_sync(0xffffffffu, base, leader);
                    if (f < n_tns) sorted[base + __popc(peers & ((1u << lane) - 1u))] = f;
                }
            }
        }
        __syncthreads();
        if (pass == 0 && threadIdx.x == 0) {
            uint32_t acc = 0;
            for (int b = 0; b < 32; ++b) {
                const uint32_t n = bin[b];
                bin[b] = acc;
                acc += n;
            }
        }
        __syncthreads();
    }
}

// A warp takes kTnsPerWarp consecutive entries of the order-sorted list, one filter per lane (the recurrence is
// serial, so a scheduler needs several such warps to stay busy: 8 filters per warp gives ~1.5 warps per
// scheduler on this batch), in place in the scratch buffer.  The lines are moved between global and shared
// memory by the whole warp, 32 lines of every filter per round: for filter j the lanes fetch 32 consecutive
// lines (one coalesced request), and the fetch of round r+1 overlaps the recurrences of round r.
constexpr int kTnsWarps = 4;
constexpr int kTnsPerWarp = 8;
__global__ void __launch_bounds__(kTnsWarps * 32) aac_tns_apply(const symgpu_aac_tns* __restrict__ tns, const uint32_t* __restrict__ sorted,
                                                                const uint32_t* __restrict__ owner, float* __restrict__ scratch,
                                                                uint32_t n_tns, uint32_t n_units) {
    __shared__ float tile_s[kTnsWarps][32 * 33];
    __shared__ float* first_s[kTnsWarps][kTnsPerWarp]; // address of each filter's first line (in processing order)
    __shared__ int len_s[kTnsWarps][kTnsPerWarp];      // lines, negated when the filter runs downwards
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* tile = tile_s[warp];
    const uint32_t i = (blockIdx.x * kTnsWarps + warp) * kTnsPerWarp + lane;
    int len = 0, order = 0;
    bool down = false;
    float* first = scratch;
    float lpc[20], h[20];
#pragma unroll
    for (int j = 0; j < 20; ++j) lpc[j] = h[j] = 0.0f;
    if (lane < kTnsPerWarp && i < n_tns) {
        const uint32_t f = sorted[i];
        const uint32_t u = owner[f];
        const symgpu_aac_tns* t = tns + f;
        int start = t->start, end = t->end;
        if (end > 1024) end = 1024; // a malformed filter must not leave its channel-frame
        order = t->order;
        if (u < n_units && start < end && order >= 1 && order <= 20) {
            len = end - start;
            down = t->direction != 0;
            first = scratch + (size_t)u * 1024 + (down ? end - 1 : start);
#pragma unroll
            for (int j = 0; j < 20; ++j)
                if (j < order) lpc[j] = __ldg(t->lpc + j);
        }
    }
    if (lane < kTnsPerWarp) {
        first_s[warp][lane] = first;
        len_s[warp][lane] = down ? -len : len;
    }
    int max_len = len;
#pragma unroll
    for (int d = 16; d; d >>= 1) max_len = max(max_len, __shfl_xor_sync(0xffffffffu, max_len, d));
    __syncwarp();

    float r[kTnsPerWarp]; // lines in flight: r[j] = line (round * 32 + lane) of filter j
    auto fetch = [&](int round) {
        const int m = round * 32 + lane;
#pragma unroll
        for (int j = 0; j < kTnsPerWarp; ++j) {
            const int lj = len_s[warp][j];
            r[j] = 0.0f;
            if (m < abs(lj)) r[j] = first_s[warp][j][lj < 0 ? -m : m];
        }
    };
    fetch(0);
    for (int round = 0; round * 32 < max_len; ++round) {
#pragma unroll
        for (int j = 0; j < kTnsPerWarp; ++j) tile[33 * lane + j] = r[j]; // row = line in the round, column = filter
        __syncwarp();
        if ((round + 1) * 32 < max_len) fetch(round + 1);
        const int m0 = round * 32;
        const int cnt = min(32, len - m0);
        if (cnt > 0) {
            float* col = tile + lane;
            switch (order) {
#define TNS_CASE(N) case N: tns_lines<N>(col, cnt, m0, h, lpc); break;
                TNS_CASE(1) TNS_CASE(2) TNS_CASE(3) TNS_CASE(4) TNS_CASE(5) TNS_CASE(6) TNS_CASE(7) TNS_CASE(8) TNS_CASE(9)
                TNS_CASE(10) TNS_CASE(11) TNS_CASE(12) TNS_CASE(13) TNS_CASE(14) TNS_CASE(15) TNS_CASE(16) TNS_CASE(17)
                TNS_CASE(18) TNS_CASE(19) TNS_CASE(20)
#undef TNS_CASE
                default: break;
            }
        }
        __syncwarp();
        const int m = m0 + lane;
#pragma unroll
        for (int j = 0; j < kTnsPerWarp; ++j) {
            const int lj = len_s[warp][j];
            if (m < abs(lj)) first_s[warp][j][lj < 0 ? -m : m] = tile[33 * lane + j];
        }
        __syncwarp();
    }
}

// ---- filterbank --------------------------------------------------------------------------------
// One CTA = one chunk of <= K consecutive frames of one channel, plus one slot for the frame before
// the chunk (its delay line).  Each frame has its own group of 64 threads and its own named barrier,
// so the K+1 IMDCTs proceed independently; the window / overlap step then reads the IMDCT output of
// frame f and of frame f-1 (the `delay` of the reference is a pure function of frame f-1's output).
constexpr int kAacK = kAacChunkFrames;     // frames per chunk, two warps per frame (named barriers)
constexpr int kAacKWarp = kAacChunkFramesWarp; // frames per chunk, ONE warp per frame (__syncwarp only)
#ifndef SYMGPU_AAC_PRE_UNROLL
#define SYMGPU_AAC_PRE_UNROLL 2
#endif
constexpr int kAacPreUnroll = SYMGPU_AAC_PRE_UNROLL; // pre-twiddle iterations (4 spectrum loads each) in flight per lane; 2 / 4 / 8
constexpr int kAacKZ = kAacChunkFramesZ;       // the same with frame slots in the Z layout
struct alignas(16) AacFrameSmem {
    float out[2048];          // spectrum (first 1024 floats) until the pre-twiddle has consumed it, then pcm_long
    float2 z[zpad_len(512)];
};
// Twiddle tables staged in shared memory once per CTA: the 200 KB of frame slots leave almost no L1,
// and the FFT passes read twiddles at lane-dependent indices (ncu: long_scoreboard 7.7 per issue with
// the tables in global memory).
struct alignas(16) AacTabSmem {
    float2 fft[8 + 16 + 480]; // FftTables prefix: lit16, lit32, merge tables of sizes 64..512
    float2 tw_long[512];
    float2 tw_short[64];
    float win_long[2][1024];  // [0] sine, [1] KBD (window_shape)
    float win_short[2][128];
};

// Two layouts of a frame slot.  Array: the 2048 IMDCT outputs as the reference stores them (12.8 KB with the FFT scratch).
// Z: only the 512 post-twiddled complex values (imdct_to_z, 4.6 KB); an output sample is looked up through imdct_out.
struct alignas(16) AacFrameZ { // 16: the in-kernel TNS moves a frame through these bytes as float4
    float2 z[zpad_len(512)];
};
struct OutArray {
    const float* p;
    __device__ __forceinline__ float lng(int j) const { return p[j]; }
    __device__ __forceinline__ float sht(int j) const { return p[j]; }     // eight short blocks: block j / 256, sample j % 256
    __device__ __forceinline__ float state(int i) const { return p[1024 + i]; } // slot 0 of a run start holds the delay line
};
struct OutZ {
    const float2* z;
    __device__ __forceinline__ float lng(int j) const { return imdct_out<9>(z, 0, j); }
    __device__ __forceinline__ float sht(int j) const { return imdct_out<6>(z, j >> 8, j & 255); }
    __device__ __forceinline__ float state(int i) const { return reinterpret_cast<const float*>(z)[i]; }
};

// pcm_short[x] of aac/dsp.rs:86-101, rebuilt per sample with the reference's operation order: the
// second half of window w-1 is written first (assignment for w-1 = 0, "0.0 +=" otherwise), then the
// first half of window w is added.
template <typename Out>
__device__ __forceinline__ float aac_pcm_short(const Out out, const float* __restrict__ sw, const float* __restrict__ psw, int x) {
    const int w = x >> 7, i = x & 127;
    if (w == 0) return out.sht(i) * psw[i];
    const float t2 = out.sht(256 * (w - 1) + 128 + i) * sw[127 - i];
    const float prev = (w == 1) ? t2 : 0.0f + t2;
    if (w == 8) return prev;
    return prev + out.sht(256 * w + i) * sw[i];
}

// delay[i] after a frame with IMDCT output `out` (aac/dsp.rs:131-157) -- what the NEXT frame overlaps with.
template <typename Out>
__device__ __forceinline__ float aac_new_delay(int seq, const Out out, const float* __restrict__ lw, const float* __restrict__ sw,
                                               const float* __restrict__ psw, int i) {
    switch (seq) {
        case SYMGPU_AAC_ONLY_LONG:
        case SYMGPU_AAC_LONG_STOP: return out.lng(i + 1024) * lw[1023 - i];
        case SYMGPU_AAC_EIGHT_SHORT: return i < P1 ? aac_pcm_short(out, sw, psw, i + 512 + 64) : 0.0f;
        default: // LONG_START
            return i < P0 ? out.lng(i + 1024) : i < P1 ? out.lng(i + 1024) * sw[127 - (i - P0)] : 0.0f;
    }
}

// Persistent: gridDim.x CTAs (two per SM) walk the chunks blockIdx.x, blockIdx.x + gridDim.x, ...; the twiddle
// and window tables are staged in shared memory once per CTA.
// GW = threads per frame: 64 (two warps, named barrier; K = 6 frames per chunk, two CTAs per SM) or 32 (one warp, __syncwarp
// only; K = 13 frames per chunk, one CTA per SM: half the warps, no hardware barrier inside the IMDCT, one halo frame in 14
// instead of one in 7).
//
// ZL (GW = 32 only): frame slots in the Z layout -- 14 slots are 65 KB instead of 180 KB, so two CTAs share an SM: 28 frames in
// flight per SM, one warp each, no hardware barrier inside an IMDCT.
template <int GW, int K, bool ZL>
__global__ void __launch_bounds__((K + 1) * GW, ZL ? (K >= 15 ? 2 : K >= 9 ? 3 : 4) : GW == 64 ? 2 : 1) aac_synth_kernel(AacArgs a) {
    static_assert(!ZL || GW == 32, "the Z layout is written for one warp per frame");
    extern __shared__ __align__(16) unsigned char aac_raw[];
    using Slot = typename std::conditional<ZL, AacFrameZ, AacFrameSmem>::type;
    using Out = typename std::conditional<ZL, OutZ, OutArray>::type;
    Slot* fs = reinterpret_cast<Slot*>(aac_raw);
    // the tables follow the slots at a 16-byte boundary
    AacTabSmem& ts = *reinterpret_cast<AacTabSmem*>(aac_raw + (((K + 1) * sizeof(Slot) + 15) & ~size_t(15)));
    auto out_of = [&](int slot) -> Out {
        if constexpr (ZL) return Out{fs[slot].z};
        else return Out{fs[slot].out};
    };
    __shared__ bool is_last;
    const int tid = threadIdx.x;
    const int slot = tid / GW, gt = tid % GW; // frame slot of this thread's group in the CTA, thread within the group
    const CodecTables* __restrict__ tab = a.tab;
    {
        const float2* g_fft = reinterpret_cast<const float2*>(tab->fft_lit16);
        const float2* g_twl = reinterpret_cast<const float2*>(tab->aac_tw_long);
        const float2* g_tws = reinterpret_cast<const float2*>(tab->aac_tw_short);
        for (int i = tid; i < 504; i += blockDim.x) ts.fft[i] = __ldg(g_fft + i);
        for (int i = tid; i < 512; i += blockDim.x) ts.tw_long[i] = __ldg(g_twl + i);
        if (tid < 64) ts.tw_short[tid] = __ldg(g_tws + tid);
        for (int i = tid; i < 1024; i += blockDim.x) {
            ts.win_long[0][i] = __ldg(tab->aac_sine_long + i);
            ts.win_long[1][i] = __ldg(tab->aac_kbd_long + i);
        }
        if (tid < 128) {
            ts.win_short[0][tid] = __ldg(tab->aac_sine_short + tid);
            ts.win_short[1][tid] = __ldg(tab->aac_kbd_short + tid);
        }
    }
    __syncthreads();
    const FftTables* ft = reinterpret_cast<const FftTables*>(ts.fft);

    const uint32_t* __restrict__ group_first = reinterpret_cast<const uint32_t*>(a.chunks + a.n_chunks);
    const int lane = tid & 31;
    // My chunk of group g and my slot inside it: the chunks of a group take count + 1 consecutive frame slots each.
    auto locate = [&](int g, int& grp) -> int {
        const uint32_t c0 = group_first[g], nc = group_first[g + 1] - c0;
        const int cnt = (uint32_t)lane < nc ? (int)a.chunks[c0 + lane].count + 1 : 0;
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        const unsigned mine = __ballot_sync(0xffffffffu, cnt > 0 && incl - cnt <= slot && slot < incl);
        if (!mine) {
            grp = 0;
            return -1;
        }
        const int j = __ffs(mine) - 1;
        grp = slot - __shfl_sync(0xffffffffu, incl - cnt, j);
        return (int)c0 + j;
    };

    for (int g = blockIdx.x; g < a.n_groups; g += gridDim.x) {
        int grp;
        const int cidx = locate(g, grp);
        const bool active = cidx >= 0;
        const CodecChunk ck = active ? a.chunks[cidx] : CodecChunk{};
        const int ch = ck.channel;
        const uint32_t gen = active ? a.gen[ck.stream] : 0u;
        const float* st_in = a.states + (((size_t)ck.stream * 2 + (gen & 1)) * 2 + ch) * 1024;
        float* st_out = a.states + (((size_t)ck.stream * 2 + ((gen + 1) & 1)) * 2 + ch) * 1024;
        const bool load_state = ck.flags & kChunkLoadState;
        const int count = active ? (int)ck.count : -1;

        // slot 0 of a chunk = the frame before it (or the stream state), slot k = chunk frame k-1
        const int f = (int)ck.first - 1 + grp;
        const bool have_frame = active && grp <= count && (grp > 0 || !load_state);
        symgpu_aac_unit u = {};
        if (have_frame) {
            const size_t unit_idx = 2 * (size_t)f + ch;
            u = a.units[unit_idx];
            const float* src = ((u.n_tns && !(ZL && a.tns_inline)) ? a.tns_scratch : a.coeffs) + unit_idx * 1024;
            if constexpr (ZL) {
                WarpSync sync;
                bool filtered = false;
                if (a.tns_inline && u.n_tns) {
                    // TNS here instead of in a pre-pass: the frame's lines into shared memory (the bytes z will take), one
                    // filter per lane in place (filters of a frame never read outside their own range, tns.rs:163-196), and
                    // out to the scratch buffer, where the pre-twiddle picks them up (through L2: they were written by this
                    // kernel).  The longest recurrence of a CTA pass delays its window phase; the SM's other CTA fills in.
                    float* lines = reinterpret_cast<float*>(fs[slot].z);
                    float* back = a.tns_scratch_rw + unit_idx * 1024;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        reinterpret_cast<float4*>(lines)[gt + 32 * i] = __ldg(reinterpret_cast<const float4*>(a.coeffs + unit_idx * 1024) + gt + 32 * i);
                    __syncwarp();
                    for (uint32_t f = gt; f < u.n_tns; f += 32)
                        if (u.tns_first + f < a.n_tns) tns_filter_in_place<1>(lines, a.tns + u.tns_first + f);
                    __syncwarp();
#pragma unroll
                    for (int i = 0; i < 8; ++i) reinterpret_cast<float4*>(back)[gt + 32 * i] = reinterpret_cast<const float4*>(lines)[gt + 32 * i];
                    __threadfence_block();
                    __syncwarp();
                    src = back;
                    filtered = true;
                }
                auto pair_long = [src, filtered](int, int l) {
                    const float2* q = reinterpret_cast<const float2*>(src + l);
                    return filtered ? __ldcg(q) : __ldg(q);
                };
                auto pair_short = [src, filtered](int b, int l) {
                    const float2* q = reinterpret_cast<const float2*>(src + (b << 7) + l);
                    return filtered ? __ldcg(q) : __ldg(q);
                };
                if (u.window_sequence != SYMGPU_AAC_EIGHT_SHORT)
                    imdct_to_z_from<9, kAacPreUnroll>(pair_long, fs[slot].z, 1, ts.tw_long, ft, gt, 32, sync);
                else
                    imdct_to_z_from<6, kAacPreUnroll>(pair_short, fs[slot].z, 8, ts.tw_short, ft, gt, 32, sync);
            } else {
                auto& me = fs[slot];
                for (int i = gt; i < 256; i += GW) reinterpret_cast<float4*>(me.out)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
                // the spectrum sits in out[0..1024); the pre-twiddle reads all of it before anything is written back
                if constexpr (GW == 64) {
                    NamedSync sync{1 + slot, 64};
                    sync();
                    if (u.window_sequence != SYMGPU_AAC_EIGHT_SHORT)
                        imdct_blocks<9>(me.out, me.out, me.z, 1, ts.tw_long, ft, gt, 64, sync);
                    else
                        imdct_blocks<6>(me.out, me.out, me.z, 8, ts.tw_short, ft, gt, 64, sync);
                } else {
                    WarpSync sync;
                    sync();
                    if (u.window_sequence != SYMGPU_AAC_EIGHT_SHORT)
                        imdct_blocks<9>(me.out, me.out, me.z, 1, ts.tw_long, ft, gt, 32, sync);
                    else
                        imdct_blocks<6>(me.out, me.out, me.z, 8, ts.tw_short, ft, gt, 32, sync);
                }
            }
        } else if (active && grp == 0) {
            // run start: slot 0 holds the delay line itself (Array layout: in out[1024..2048); Z layout: the first 1024 floats)
            if constexpr (ZL) {
                for (int i = gt; i < 1024; i += GW) reinterpret_cast<float*>(fs[slot].z)[i] = st_in[i];
            } else {
                for (int i = gt; i < 1024; i += GW) fs[slot].out[1024 + i] = st_in[i];
            }
        }
        __syncthreads();

        // Pull the next group's spectra towards the SM (HBM -> L2) while this one is windowed.
        if (g + (int)gridDim.x < a.n_groups && gt < 32) {
            int ngrp;
            const int nidx_c = locate(g + gridDim.x, ngrp);
            if (nidx_c >= 0) {
                const CodecChunk nk = a.chunks[nidx_c];
                const int nf = (int)nk.first - 1 + ngrp;
                if (ngrp > 0 || !(nk.flags & kChunkLoadState)) {
                    const size_t nidx = 2 * (size_t)nf + nk.channel;
                    const float* nsrc = ((a.units[nidx].n_tns && !(ZL && a.tns_inline)) ? a.tns_scratch : a.coeffs) + nidx * 1024;
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(nsrc + 32 * gt));
                }
            }
        }

        // window + overlap-add (aac/dsp.rs:103-129): thread = (frame slot, sample)
        if (active && grp >= 1 && grp <= count) {
            const Out out = out_of(slot);
            const Out pout = out_of(slot - 1);
            const symgpu_aac_unit pu = (grp > 1 || !load_state) ? a.units[2 * (size_t)(f - 1) + ch] : symgpu_aac_unit{};
            const bool prev_is_state = grp == 1 && load_state;
            const int seq = u.window_sequence, pseq = pu.window_sequence;
            const float* sw = ts.win_short[u.window_shape ? 1 : 0];
            const float* plw = ts.win_long[u.prev_window_shape ? 1 : 0];
            const float* psw = ts.win_short[u.prev_window_shape ? 1 : 0];
            // windows of the PREVIOUS frame, for its delay line
            const float* q_lw = ts.win_long[pu.window_shape ? 1 : 0];
            const float* q_sw = ts.win_short[pu.window_shape ? 1 : 0];
            const float* q_psw = ts.win_short[pu.prev_window_shape ? 1 : 0];
            float* dst = a.pcm + (2 * (size_t)f + ch) * 1024;
            bool done = false;
            if constexpr (ZL) {
                // long block after long block (the common case): straight from the two z arrays, two adjacent samples at a time
                if (!prev_is_state && (seq == SYMGPU_AAC_ONLY_LONG || seq == SYMGPU_AAC_LONG_START) &&
                    (pseq == SYMGPU_AAC_ONLY_LONG || pseq == SYMGPU_AAC_LONG_STOP)) {
                    auto win2 = [plw, q_lw](bool fall, int idx) { return *reinterpret_cast<const float2*>((fall ? q_lw : plw) + idx); };
                    overlap_add_equal(fs[slot].z, fs[slot - 1].z, 9, win2, dst, gt, 32);
                    done = true;
                }
            }
#pragma unroll 4
            for (int i = gt; i < 1024 && !done; i += GW) {
                const float d = prev_is_state ? pout.state(i) : aac_new_delay(pseq, pout, q_lw, q_sw, q_psw, i);
                float y;
                switch (seq) {
                    case SYMGPU_AAC_ONLY_LONG:
                    case SYMGPU_AAC_LONG_START: y = d + (out.lng(i) * plw[i]); break;
                    case SYMGPU_AAC_EIGHT_SHORT: y = i < P0 ? d : d + aac_pcm_short(out, sw, psw, i - P0); break;
                    default: y = i < P0 ? d : i < P1 ? d + out.lng(i) * psw[i - P0] : d + out.lng(i); break; // LONG_STOP
                }
                dst[i] = y;
            }
            if (grp == count && (ck.flags & kChunkStoreState)) { // the run's last frame leaves its delay line in the state
                const float* lw = ts.win_long[u.window_shape ? 1 : 0];
                for (int i = gt; i < 1024; i += GW) st_out[i] = aac_new_delay(seq, out, lw, sw, psw, i);
            }
        }
        __syncthreads(); // the frame slots are reused by the next group
    }

    // launch epilogue: the last CTA publishes the new state generation (see mp3_kernel.cu)
    if (tid == 0) {
        __threadfence();
        is_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (is_last) {
        for (int i = tid; i < a.n_chunks; i += blockDim.x)
            if ((a.chunks[i].flags & kChunkStoreState) && a.chunks[i].channel == 0) a.gen[a.chunks[i].stream] += 1;
        if (tid == 0) *a.done = 0;
    }
}

} // namespace

template <int GW, int K, bool ZL>
static cudaError_t launch_variant(const AacArgs& b, cudaStream_t stream) {
    constexpr size_t slot = ZL ? sizeof(AacFrameZ) : sizeof(AacFrameSmem);
    constexpr size_t smem = (((K + 1) * slot + 15) & ~size_t(15)) + sizeof(AacTabSmem);
    static int max_grid = 0;
    cudaError_t e;
    if (!max_grid) {
        if ((e = cudaFuncSetAttribute(aac_synth_kernel<GW, K, ZL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
        int dev = 0, n_sm = 0, per_sm = 0;
        if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
        if ((e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
        if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, aac_synth_kernel<GW, K, ZL>, (K + 1) * GW, smem)) != cudaSuccess) return e;
        max_grid = n_sm * (per_sm > 0 ? per_sm : 1);
    }
    aac_synth_kernel<GW, K, ZL><<<b.n_groups < max_grid ? b.n_groups : max_grid, (K + 1) * GW, smem, stream>>>(b);
    return cudaGetLastError();
}

// SYMGPU_AAC_TNS = frames (the default: one pre-pass kernel, a warp per filtered channel-frame) | sorted (round 1's three kernels:
// sort by order / prepare / apply, one filter per lane) | inline (Z kernel only: the filters of a frame run on the lanes of the
// frame's own warp before its IMDCT, no pre-pass and no scratch copy; slower at 20 % TNS -- a CTA pass waits at its barrier for
// the longest recurrence among its 16 frames -- faster at 5 %).
static int aac_tns_mode() { // 0 frames | 1 sorted | 2 inline
    static int mode = -1;
    if (mode < 0) {
        const char* env = getenv("SYMGPU_AAC_TNS");
        mode = !env ? 0 : env[0] == 's' ? 1 : env[0] == 'i' ? 2 : 0;
        if (mode == 2 && aac_kernel_variant() != 2) mode = 0;
    }
    return mode;
}
static bool aac_tns_inline() { return aac_tns_mode() == 2; }
int aac_launch_count(bool any_tns) { return !any_tns ? 1 : aac_tns_mode() == 0 ? 2 : aac_tns_mode() == 1 ? 4 : 1; }

cudaError_t aac_launch(const AacArgs& a, uint32_t n_units, bool any_tns, int n_chunks, int n_groups, cudaStream_t stream) {
    if (any_tns && aac_tns_mode() == 0) {
        aac_tns_frames<<<(n_units + kTnsFrameWarps - 1) / kTnsFrameWarps, kTnsFrameWarps * 32, 0, stream>>>(a.units, a.tns, a.n_tns, a.coeffs, a.tns_scratch_rw, n_units);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    } else if (any_tns && !aac_tns_inline()) {
        // owner[] starts at "no owner" so that filters outside every channel-frame's range are skipped
        cudaError_t e = cudaMemsetAsync(a.tns_owner, 0xff, (size_t)a.n_tns * sizeof(uint32_t), stream);
        if (e != cudaSuccess) return e;
        aac_tns_sort<<<1, 1024, 0, stream>>>(a.tns, a.n_tns, a.tns_sorted);
        aac_tns_prepare<<<(n_units + 7) / 8, 256, 0, stream>>>(a.units, a.coeffs, a.tns_scratch_rw, a.tns_owner, n_units, a.n_tns);
        aac_tns_apply<<<(a.n_tns + kTnsWarps * kTnsPerWarp - 1) / (kTnsWarps * kTnsPerWarp), kTnsWarps * 32, 0, stream>>>(a.tns, a.tns_sorted, a.tns_owner, a.tns_scratch_rw, a.n_tns, n_units);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    AacArgs b = a;
    b.n_chunks = n_chunks;
    b.n_groups = n_groups;
    b.tns_inline = (any_tns && aac_tns_inline()) ? 1 : 0;
    switch (aac_kernel_variant()) {
        case 1: return launch_variant<32, kAacKWarp, false>(b, stream);
        case 2:
            switch (b.z_frames) { // frames per chunk of the Z kernel: 16 warps x 2 CTAs per SM, 10 x 3, 8 x 4 (aac_chunk_frames_for)
                case 9: return launch_variant<32, 9, true>(b, stream);
                case 7: return launch_variant<32, 7, true>(b, stream);
                default: return launch_variant<32, kAacKZ, true>(b, stream);
            }
        default: return launch_variant<64, kAacK, false>(b, stream);
    }
}

// SYMGPU_AAC_KERNEL = pair (two warps per frame, named barriers) | warp (one warp per frame) | z (one warp per frame, Z layout).
int aac_kernel_variant() {
    static int mode = -1;
    if (mode < 0) {
        const char* env = getenv("SYMGPU_AAC_KERNEL");
        mode = !env ? kAacDefaultVariant : env[0] == 'w' ? 1 : env[0] == 'z' ? 2 : env[0] == 'p' ? 0 : kAacDefaultVariant;
    }
    return mode;
}
bool aac_warp_per_frame() { return aac_kernel_variant() != 0; }
// Frames per chunk of the Z kernel, i.e. 16, 10 or 8 warps per CTA at 2, 3 or 4 CTAs per SM.  Long runs fill the large
// chunks; short runs (the mixed corpus: 8-16 frames per stream and call, a chunk plus its state slot fills 9 of the 16 warps)
// leave warps of a large chunk idle.  So the plan takes 9 when the runs are short and 15 otherwise; SYMGPU_AAC_Z_FRAMES =
// 15 | 9 | 7 pins it.
int aac_z_frames(uint32_t mean_run_frames) {
    static int pinned = -1;
    if (pinned < 0) {
        const char* env = getenv("SYMGPU_AAC_Z_FRAMES");
        const int v = env ? atoi(env) : 0;
        pinned = (v == 15 || v == 9 || v == 7) ? v : 0;
    }
    if (pinned) return pinned;
    return mean_run_frames <= 24 ? 9 : kAacKZ;
}
int aac_chunk_frames_for(uint32_t mean_run_frames) {
    return aac_kernel_variant() == 2 ? aac_z_frames(mean_run_frames) : aac_kernel_variant() == 1 ? kAacKWarp : kAacK;
}
int aac_chunk_frames() { return aac_chunk_frames_for(1u << 20); }

} // namespace symgpu
