// Fused MPEG Layer III synthesis kernel for sm_90a:
//   requantize -> joint stereo -> reorder -> antialias -> IMDCT-36/12 + window + overlap-add
//   -> frequency inversion -> DCT-32 -> 512-tap polyphase window  (layer3/mod.rs:421-477)
// in ONE launch, PCM written straight to HBM.  No intermediate ever leaves the SM.
//
// Parallelisation (DESIGN.md §3): every piece of cross-granule state on this path is overwritten,
// never accumulated (hybrid overlap, polyphase FIFO), so a stream is cut into TILES of <= T consecutive
// granules.  A tile that starts a run takes overlap + polyphase history from the stream state in
// HBM; any other tile recomputes a 2-granule halo (the overlap of granule g-1 needs IMDCT of g-1;
// the 15 history slots need the time samples of g-1, which need the overlap of g-2).  The grid is
// PERSISTENT: one CTA of NW warps per SM walks tiles blockIdx, blockIdx+grid, ... with all its
// warps in the same phase (several phases live on one SM thrash the instruction cache, as
// with 2 CTAs/SM).  The spectra of the next tile are fetched by TMA bulk copies
// (cp.async.bulk -> mbarrier) while the current tile is in its DCT / window phases.
//
// Bit-exactness rules: compiled with -fmad=false; every expression keeps the reference's operand
// order; tables come from the host (tables.cpp); tests/test_build_and_abi.py greps the SASS for
// FFMA and fails on any hit.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>

#include "../../include/symgpu.h"
#include "mp3_kernel.h"
#include "tables.h"

namespace symgpu {

// Uniformly indexed coefficient tables live in constant memory (c[3][...] operands cost no issue
// slot); lane-indexed tables stay in global memory behind the read-only path.
struct Mp3Const {
    float imdct_win[4][36];
    float half_cos12[6][6];
    float dct_iv_scale[18];
    float sdct18_scale[9];
    float sdct9_d[7];
    float lee16[16], lee8[8], lee4[4], lee2[2], lee1;
    float is_mpeg1[7][2];
    float is_mpeg2[2][32][2];
    float cs[8], ca[8];
    uint8_t pre_emphasis[24];
    uint8_t mixed_switch[12];
    uint8_t n_edges[9][3];
};
__constant__ Mp3Const c_mp3;

cudaError_t mp3_upload_const(const Mp3Tables& t, cudaStream_t stream) {
    static Mp3Const h; // staging must outlive the async copy
    memcpy(h.imdct_win, t.imdct_win, sizeof h.imdct_win);
    memcpy(h.half_cos12, t.half_cos12, sizeof h.half_cos12);
    memcpy(h.dct_iv_scale, t.dct_iv_scale, sizeof h.dct_iv_scale);
    memcpy(h.sdct18_scale, t.sdct18_scale, sizeof h.sdct18_scale);
    memcpy(h.sdct9_d, t.sdct9_d, sizeof h.sdct9_d);
    memcpy(h.lee16, t.lee16, sizeof h.lee16);
    memcpy(h.lee8, t.lee8, sizeof h.lee8);
    memcpy(h.lee4, t.lee4, sizeof h.lee4);
    memcpy(h.lee2, t.lee2, sizeof h.lee2);
    h.lee1 = t.lee1;
    memcpy(h.is_mpeg1, t.is_mpeg1, sizeof h.is_mpeg1);
    memcpy(h.is_mpeg2, t.is_mpeg2, sizeof h.is_mpeg2);
    memcpy(h.cs, t.cs, sizeof h.cs);
    memcpy(h.ca, t.ca, sizeof h.ca);
    memcpy(h.pre_emphasis, t.pre_emphasis, sizeof h.pre_emphasis);
    memset(h.mixed_switch, 0, sizeof h.mixed_switch);
    memcpy(h.mixed_switch, t.mixed_switch, 9);
    memcpy(h.n_edges, t.n_edges, sizeof h.n_edges);
    cudaError_t e = cudaMemcpyToSymbolAsync(c_mp3, &h, sizeof h, 0, cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(stream);
}

namespace {

constexpr int kPitch = 33; // float2 per slot row: 32 sub-bands + one always-zero column (V[16] = 0)
constexpr float kFrac1Sqrt2 = 0.707106781186547524400844362104849039f;

struct WarpScratch {
    symgpu_mp3_gc gc[2];
    float scale[2][40];
    float2 sratio[40];
    uint8_t smode[40]; // 0 none, 1 mid/side, 2 intensity
    uint8_t nz[40];    // channel-1 interval holds a non-zero line
    // what this warp's job does with its `second` half after the hybrid phase (parked here so that it does not
    // occupy registers during the phase): XT region it is added into, or -1, and the state it is stored to, or null
    int next_region;
    Mp3StreamState* st_out;
};

__device__ __forceinline__ int kind_of(const symgpu_mp3_gc& g) {
    if (g.block_type != SYMGPU_MP3_SHORT) return kKindLong;
    return (g.flags & SYMGPU_MP3_F_MIXED) ? kKindMixed : kKindShort;
}

// ---- 9-point SDCT-II (hybrid_synthesis.rs:721-779); y[j] is the reference's y[2j] ----------  // PHASE: B imdct36
__device__ __forceinline__ void sdct9(const float (&x)[9], float (&y)[9]) {
    const float a01 = x[3] + x[5], a02 = x[3] - x[5], a03 = x[6] + x[2], a04 = x[6] - x[2];
    const float a05 = x[1] + x[7], a06 = x[1] - x[7], a07 = x[8] + x[0], a08 = x[8] - x[0];
    const float a09 = x[4] + a05, a10 = a01 + a03, a11 = a10 + a07, a12 = a03 - a07;
    const float a13 = a01 - a07, a14 = a01 - a03, a15 = a02 - a04, a16 = a15 + a08;
    const float a17 = a04 + a08, a18 = a02 - a08, a19 = a02 + a04, a20 = 2.0f * x[4] - a05;
    const float m1 = c_mp3.sdct9_d[0] * a06, m2 = c_mp3.sdct9_d[1] * a12, m3 = c_mp3.sdct9_d[2] * a13;
    const float m4 = c_mp3.sdct9_d[3] * a14, m5 = c_mp3.sdct9_d[0] * a16, m6 = c_mp3.sdct9_d[4] * a17;
    const float m7 = c_mp3.sdct9_d[5] * a18, m8 = c_mp3.sdct9_d[6] * a19;
    const float a21 = a20 + m2, a22 = a20 - m2, a23 = a20 + m3, a24 = m1 + m6, a25 = m1 - m6, a26 = m1 + m7;
    y[0] = a09 + a11;
    y[1] = m8 - a26;
    y[2] = m4 - a21;
    y[3] = m5;
    y[4] = a22 - m3;
    y[5] = a25 - m7;
    y[6] = a11 - 2.0f * a09;
    y[7] = a24 + m8;
    y[8] = a23 + m4;
}

// ---- 18-point DCT-IV via two 9-point SDCT-IIs (hybrid_synthesis.rs:608-716) -----------------
__device__ __forceinline__ void dct_iv_18(const float (&x)[18], float (&y)[18]) {
    float s[18];
#pragma unroll
    for (int i = 0; i < 18; ++i) s[i] = c_mp3.dct_iv_scale[i] * x[i];
    float even[9], odd[9], ye[9], yo[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) even[i] = s[i] + s[17 - i];
    sdct9(even, ye);
#pragma unroll
    for (int i = 0; i < 9; ++i) odd[i] = c_mp3.sdct18_scale[i] * (s[i] - s[17 - i]);
    sdct9(odd, yo);
#pragma unroll
    for (int j = 1; j < 9; ++j) yo[j] = yo[j] - yo[j - 1]; // y[3]-=y[1]; y[5]-=y[3]; ... sequential
#pragma unroll
    for (int j = 0; j < 9; ++j) {
        y[2 * j] = ye[j];
        y[2 * j + 1] = yo[j];
    }
    y[0] = y[0] * 0.5f; // "/ 2.0" -- exact either way
#pragma unroll
    for (int i = 1; i < 18; ++i) y[i] = (y[i] * 0.5f) - y[i - 1];
}

// imdct36 (hybrid_synthesis.rs:571-603) without the overlap add: first = windowed samples 0..17,
// second = windowed samples 18..35 (the next granule's overlap).
__device__ __forceinline__ void imdct36(const float (&x)[18], const float* __restrict__ win,
                                        float (&first)[18], float (&second)[18]) {
    float dct[18];
    dct_iv_18(x, dct);
#pragma unroll
    for (int i = 0; i < 9; ++i) first[i] = dct[9 + i] * win[i];
#pragma unroll
    for (int i = 9; i < 18; ++i) first[i] = -(dct[26 - i] * win[i]); // overlap - d*w == overlap + (-(d*w))
#pragma unroll
    for (int i = 18; i < 27; ++i) second[i - 18] = -dct[26 - i] * win[i];
#pragma unroll
    for (int i = 27; i < 36; ++i) second[i - 18] = -dct[i - 27] * win[i];
}

// imdct12_win (hybrid_synthesis.rs:363-455) without the overlap add.  // PHASE: B imdct12
__device__ __forceinline__ void imdct12x3(const float (&x)[18], float (&first)[18], float (&second)[18]) {
    float tmp[36];
#pragma unroll
    for (int i = 0; i < 36; ++i) tmp[i] = 0.0f;
    const float* win = c_mp3.imdct_win[2];
#pragma unroll
    for (int w = 0; w < 3; ++w) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float yl = (x[w] * c_mp3.half_cos12[i][0]) + (x[3 + w] * c_mp3.half_cos12[i][1]) +
                             (x[6 + w] * c_mp3.half_cos12[i][2]) + (x[9 + w] * c_mp3.half_cos12[i][3]) +
                             (x[12 + w] * c_mp3.half_cos12[i][4]) + (x[15 + w] * c_mp3.half_cos12[i][5]);
            const float yr = (x[w] * c_mp3.half_cos12[i + 3][0]) + (x[3 + w] * c_mp3.half_cos12[i + 3][1]) +
                             (x[6 + w] * c_mp3.half_cos12[i + 3][2]) + (x[9 + w] * c_mp3.half_cos12[i + 3][3]) +
                             (x[12 + w] * c_mp3.half_cos12[i + 3][4]) + (x[15 + w] * c_mp3.half_cos12[i + 3][5]);
            tmp[6 + 6 * w + 2 - i] += -yl * win[2 - i];
            tmp[6 + 6 * w + i + 3] += yl * win[i + 3];
            tmp[6 + 6 * w + i + 6] += yr * win[i + 6];
            tmp[6 + 6 * w + 11 - i] += yr * win[11 - i];
        }
    }
#pragma unroll
    for (int i = 0; i < 18; ++i) {
        first[i] = tmp[i];
        second[i] = tmp[i + 18];
    }
}

// ---- Lee 32-point DCT (synthesis.rs:348-844) as the recursion the reference hand-flattens ----  // PHASE: C dct32
template <int N> struct LeeCoef;
template <> struct LeeCoef<16> { static __device__ __forceinline__ float at(int i) { return c_mp3.lee16[i]; } };
template <> struct LeeCoef<8> { static __device__ __forceinline__ float at(int i) { return c_mp3.lee8[i]; } };
template <> struct LeeCoef<4> { static __device__ __forceinline__ float at(int i) { return c_mp3.lee4[i]; } };
template <> struct LeeCoef<2> { static __device__ __forceinline__ float at(int i) { return c_mp3.lee2[i]; } };

template <int N>
__device__ __forceinline__ void lee_dct(const float (&x)[N], float (&y)[N]) {
    if constexpr (N == 2) {
        y[0] = x[0] + x[1];
        y[1] = (x[0] - x[1]) * c_mp3.lee1;
    } else {
        constexpr int H = N / 2;
        float lo[H], hi[H], lo_t[H], hi_t[H];
#pragma unroll
        for (int i = 0; i < H; ++i) {
            lo[i] = x[i] + x[N - 1 - i];
            hi[i] = (x[i] - x[N - 1 - i]) * LeeCoef<H>::at(i);
        }
        lee_dct<H>(lo, lo_t);
        lee_dct<H>(hi, hi_t);
#pragma unroll
        for (int i = 0; i < H - 1; ++i) {
            y[2 * i] = lo_t[i];
            y[2 * i + 1] = hi_t[i] + hi_t[i + 1];
        }
        y[N - 2] = lo_t[H - 1];
        y[N - 1] = hi_t[H - 1];
    }
}

// Sign of the frequency inversion (hybrid_synthesis.rs:458-485): odd sample of odd sub-band.  // PHASE: B store
__device__ __forceinline__ float finv(float v, int sb, int t) { return ((sb & t) & 1) ? -v : v; }

} // namespace

// =============================================================================================
namespace {

// ---- mbarrier / TMA bulk-copy wrappers (PTX ISA 8.6, sm_90+) -----------------------------------  // PHASE: tma+mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ float2 lds64(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}


// ---- (ch0, ch1) pair arithmetic of the window phase: one correctly rounded scalar operation per channel, never contracted
__device__ __forceinline__ float2 pk_mul(float2 a, float s) { return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s)); }
__device__ __forceinline__ float2 pk_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// Polyphase window of `total` consecutive time slots whose DCT vectors sit in XT rows row0 ..  // PHASE: D window
// (with the 15 rows before row0 holding the history).  lane = PCM sample index i; each warp walks a
// contiguous range of slots with a 16-deep register window of (V_lo[i], V_hi[i]) for both channels:
//   V_lo[i] =  d[16+i] (i<16) | 0 (i=16, the constant column 32) | -d[48-i] (i>16)
//   V_hi[i] = -d[16-i] (i<=16) | -d[i-16] (i>16)                         (synthesis.rs:247-263)
//   o[i] = sum_j  V_lo(t-2j)[i] * D[64j+i]  then  + V_hi(t-2j-1)[i] * D[64j+32+i]   (:309-323)
// The signs are folded into the per-lane coefficients ((-d)*D == d*(-D) exactly).  `slot_seq0` is the
// batch-wide sequence number of the first slot: slots of a frame are contiguous in a PCM plane
// (plane[gr*576 + t*32 + i]) and frames are SYMGPU_MP3_FRAME_FLOATS apart.
// TWO_JUMPS: a block of 16 slots may cross two frame boundaries (Layer I: 12 slots per frame).
template <bool TWO_JUMPS = false>
__device__ __forceinline__ void window_phase(const float* xt, int row0, int begin, int end, int lane,
                                             const float* __restrict__ synth_d, float* __restrict__ pcm, int slot_seq0,
                                             int slots_per_frame, bool stereo) {
    const int col_lo = lane < 16 ? 16 + lane : (lane == 16 ? 32 : 48 - lane);
    const int col_hi = lane <= 16 ? 16 - lane : lane - 16;
    float dlo[8], dhi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float a0 = __ldg(synth_d + 64 * j + lane);
        dlo[j] = lane > 16 ? -a0 : a0;
        dhi[j] = -__ldg(synth_d + 64 * j + 32 + lane);
    }
    if (begin >= end) return; // [begin, end): slot indices relative to row0
    constexpr uint32_t kRowBytes = kPitch * 8;
    uint32_t a_lo = smem_u32(xt) + (uint32_t)((row0 + begin - 15) * kPitch + col_lo) * 8u;
    uint32_t a_hi = smem_u32(xt) + (uint32_t)((row0 + begin - 15) * kPitch + col_hi) * 8u;
    float2 wl[16], wh[16];
#pragma unroll
    for (int m = 0; m < 15; ++m) { // the 15 slots before `begin` -> window index (m+1)&15
        wl[(m + 1) & 15] = lds64(a_lo + m * kRowBytes);
        wh[(m + 1) & 15] = lds64(a_hi + m * kRowBytes);
    }
    a_lo += 15 * kRowBytes;
    a_hi += 15 * kRowBytes;
    const int off1 = stereo ? 1152 : 0; // mono: the channel-1 store lands on the channel-0 word and is overwritten
    const int frame_jump = SYMGPU_MP3_FRAME_FLOATS - slots_per_frame * 32;
    for (int base = begin; base < end; base += 16) {
        const int seq = slot_seq0 + base;
        const int frame = seq / slots_per_frame, sif = seq - frame * slots_per_frame;
        float* out0 = pcm + (size_t)frame * SYMGPU_MP3_FRAME_FLOATS + sif * 32 + lane;
        float* out1 = out0 + frame_jump;        // valid once the block has crossed into the next frame
        const int kj = slots_per_frame - sif;   // steps until the frame boundary (a frame has >= 18 slots)
        const int cnt = end - base;
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            if (u < cnt) {
                wl[u] = lds64(a_lo + u * kRowBytes);
                wh[u] = lds64(a_hi + u * kRowBytes);
                float2 acc = make_float2(0.0f, 0.0f);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    acc = pk_add(pk_mul(wl[(u - 2 * j) & 15], dlo[j]), acc);
                    acc = pk_add(pk_mul(wh[(u - 2 * j - 1) & 15], dhi[j]), acc);
                }
                float* o = (u < kj ? out0 : out1) + u * 32;
                if (TWO_JUMPS && u >= kj + slots_per_frame) o += frame_jump;
                o[off1] = acc.y;
                o[0] = acc.x;
            }
        }
        a_lo += 16 * kRowBytes;
        a_hi += 16 * kRowBytes;
    }
}

template <int T, int NW>  // PHASE: prologue+tile loop
struct Mp3Smem {
    static constexpr int kRows = 18 * kMp3GroupRegions;   // every piece of the group: one history region + one per granule
    float xt[kRows * kPitch * 2];                         // [row][33][2 channels]
    alignas(16) float spec[NW][2 * 576];                  // TMA destination: spectra of the group's granule jobs
    alignas(16) symgpu_mp3_gc units[NW][2];               // TMA destination: their descriptors
    WarpScratch ws[NW];
    alignas(16) Mp3StreamState carry;                     // state handed from one group of the chain to the next
    alignas(16) Mp3Tile seg_stage[2][kMp3GroupTiles];     // descriptors of the group in flight (by iteration parity)
    uint32_t gen_stage[2][kMp3GroupTiles];                // state generation of their streams at launch
    int nseg_stage[2];
    alignas(8) uint64_t bar;
    bool is_last;
};

} // namespace

// MULTI = false: every group of the plan is a single tile (the shape of large batches); the loops over the
// pieces of a group then fold away at compile time.
template <int T, int NW, bool MULTI>
__global__ void __launch_bounds__(NW * 32, NW <= 8 ? 2 : 1) mp3_synth_kernel(Mp3Args a) {
    static_assert(NW >= T, "one warp per granule job (a tile with a halo holds NW - 2 granules)");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using Smem = Mp3Smem<T, NW>;
    Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
    float* xt = sm.xt;

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const Mp3Tables* __restrict__ tab = a.tab;
    const int n_tiles = a.n_tiles;

    // One thread: the descriptors of the group that starts at tile `ti` (up to and including the tile flagged
    // kTileGroupEnd) and their streams' generations into the stage (ordinary stores, published by the release of
    // the mbarrier arrive), then TMA bulk copies of every piece's descriptors + spectra.  Job slots are handed
    // out in order: a piece with a halo takes n + 2, any other piece n.
    auto issue_prefetch = [&](int ti, int parity) {
        int nseg = 0, jobs = 0;
        for (;;) {
            const Mp3Tile t = a.tiles[ti + nseg];
            sm.seg_stage[parity][nseg] = t;
            sm.gen_stage[parity][nseg] = a.gen[t.stream];
            jobs += t.n_granules + ((t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : 2);
            ++nseg;
            if (!MULTI || (t.flags & kTileGroupEnd) || nseg == kMp3GroupTiles) break;
        }
        sm.nseg_stage[parity] = nseg;
        mbar_expect_tx(&sm.bar, (uint32_t)jobs * (4608u + 128u));
        int slot0 = 0;
        for (int k = 0; k < nseg; ++k) {
            const Mp3Tile t = sm.seg_stage[parity][k];
            const int halo = (t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : 2;
            const int cnt = t.n_granules + halo;
            if (t.gpf == 2) { // granules of consecutive frames are contiguous: [frame][gr][ch][576]
                const size_t src = (size_t)t.first_frame * 2 + t.first_gr - halo;
                tma_bulk_g2s(sm.spec[slot0], a.spectra + src * 1152, (uint32_t)cnt * 4608u, &sm.bar);
                tma_bulk_g2s(sm.units[slot0], a.units + src * 2, (uint32_t)cnt * 128u, &sm.bar);
            } else {          // one granule per frame slot
                for (int j = 0; j < cnt; ++j) {
                    const size_t src = (size_t)((int)t.first_frame + t.first_gr - halo + j) * 2;
                    tma_bulk_g2s(sm.spec[slot0 + j], a.spectra + src * 1152, 4608u, &sm.bar);
                    tma_bulk_g2s(sm.units[slot0 + j], a.units + src * 2, 128u, &sm.bar);
                }
            }
            slot0 += cnt;
        }
    };

    if (threadIdx.x == 0) {
        mbar_init(&sm.bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int t_begin = (int)a.cta_first[blockIdx.x], t_end = (int)a.cta_first[blockIdx.x + 1];
    if (threadIdx.x == 0 && t_begin < t_end) issue_prefetch(t_begin, 0);

    WarpScratch& ws = sm.ws[warp];
    int it = 0;
    for (int ti = t_begin; ti < t_end; ++it) {
        const int par = it & 1;
        mbar_wait(&sm.bar, (uint32_t)par);
        // A GROUP of consecutive tiles of the chain is processed together: each tile ("piece") is a run of
        // consecutive granules of one stream with its own state in / out; together they hold at most NW granule
        // jobs and kMp3GroupRegions XT regions (one history region + one region per granule, per piece).
        const int nseg = MULTI ? sm.nseg_stage[par] : 1;
        // My granule job: warp w takes job w of the group; find its piece.
        Mp3Tile tile = sm.seg_stage[par][0];
        int seg = -1, job0 = 0, reg0 = 0; // my piece, its first job slot and its first XT region
        {
            int jobs = 0, regions = 0;
            for (int k = 0; k < nseg; ++k) {
                const Mp3Tile t = sm.seg_stage[par][k];
                const int cnt = t.n_granules + ((t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : 2);
                if (seg < 0 && warp < jobs + cnt) {
                    seg = k;
                    job0 = jobs;
                    reg0 = regions;
                    tile = t;
                }
                jobs += cnt;
                regions += t.n_granules + 1;
            }
        }
        const int n = tile.n_granules;
        const int n_ch = tile.n_ch;
        // State comes in from HBM (run start) or from the previous group of this CTA's chain (shared memory),
        // and goes out to HBM (run end) or to the next group of the chain; with no input the piece recomputes
        // a 2-granule halo.
        const bool load_state = tile.flags & (kTileLoadState | kTileCarryIn);
        const bool store_state = tile.flags & (kTileStoreState | kTileCarryOut);
        // Stream state in HBM is double-buffered: a launch reads generation g and writes generation g+1, so a
        // run-starting tile never races with the run-ending tile of the same stream.
        const uint32_t gen = sm.gen_stage[par][seg < 0 ? 0 : seg];
        const Mp3StreamState* st_in = (tile.flags & kTileCarryIn) ? &sm.carry : a.states + (size_t)tile.stream * 2 + (gen & 1);
        Mp3StreamState* st_out = (tile.flags & kTileCarryOut) ? &sm.carry : a.states + (size_t)tile.stream * 2 + ((gen + 1) & 1);
        const int j0 = load_state ? 2 : 0; // index of the piece's first job (0, 1 = halo granules)

        // --------------------------------------------------------------------------------------
        // Phase A+B: one warp per granule job (of a piece: g = 0, 1: halo granules g0-2, g0-1; g >= 2: the
        // piece's granules), lane = sub-band, everything in registers.  Job g >= 1 owns XT region reg0 + g - 1.
        // --------------------------------------------------------------------------------------
        const int g = warp - job0 + j0; // job index inside my piece; stage slot = warp
        const bool active = seg >= 0;
        if (lane == 0) {
            ws.next_region = (active && g + 1 < n + 2) ? reg0 + g : -1;
            ws.st_out = (active && g + 1 >= n + 2 && store_state) ? st_out : nullptr;
        }
        float sec[2][18];
        if (active) {
            const symgpu_mp3_gc& g0 = sm.units[warp][0];
            const symgpu_mp3_gc& g1 = sm.units[warp][1];
            const float* S = sm.spec[warp];
            if (lane < 10) reinterpret_cast<uint32_t*>(ws.smode)[lane] = 0;
            if (lane >= 16 && lane < 26) reinterpret_cast<uint32_t*>(ws.nz)[lane - 16] = 0;
            const int sr = g0.sample_rate_idx;
            const int kind0 = kind_of(g0), kind1 = (n_ch == 2) ? kind_of(g1) : kind0;
            const bool ms = (n_ch == 2) && (g0.flags & SYMGPU_MP3_F_MID_SIDE);
            const bool is = (n_ch == 2) && (g0.flags & SYMGPU_MP3_F_INTENSITY);
            int rz0 = g0.rzero, rz1 = (n_ch == 2) ? g1.rzero : 0;

            // A1: per-interval requantisation scale (requantize.rs:240-355)  // PHASE: A1 scale
            for (int ch = 0; ch < n_ch; ++ch) {
                const symgpu_mp3_gc& gg = sm.units[warp][ch];
                const int kind = ch ? kind1 : kind0;
                const int n_iv = c_mp3.n_edges[sr][kind] - 1;
                const int gain = (int)gg.global_gain - 210;
                const int shift = (gg.flags & SYMGPU_MP3_F_SCALEFAC_SCALE) ? 2 : 1;
                const int sw = c_mp3.mixed_switch[sr];
                for (int idx = lane; idx < 40; idx += 32) {
                    float s = 1.0f;
                    if (idx < n_iv) {
                        int e = 0;
                        bool scaled = true;
                        const bool long_part = (kind == kKindLong) || (kind == kKindMixed && idx < sw - 1);
                        if (long_part) {
                            const int pre = (gg.flags & SYMGPU_MP3_F_PREFLAG) ? c_mp3.pre_emphasis[idx] : 0;
                            const int b = ((gg.scalefacs[idx] + pre) << shift) & 0xff;
                            e = gain - b;
                        } else if (kind == kKindMixed && idx == sw - 1) {
                            scaled = false; // lines between the last long band and the first short band
                        } else {
                            const int j = (kind == kKindMixed) ? idx - sw : idx; // scalefacs[switch + j] == scalefacs[idx]
                            const int b = (gg.scalefacs[idx] << shift) & 0xff;
                            e = gain - 8 * (int)gg.subblock_gain[j % 3] - b;
                        }
                        if (scaled) s = __ldg(&tab->pow2q[e - kPow2qMin]);
                    }
                    ws.scale[ch][idx] = s;
                }
            }
            __syncwarp();

            // A2: my 18 lines of each channel, requantised.  The short-block reorder  // PHASE: A2 requant+reorder
            // (hybrid_synthesis.rs:153-215) is a permutation applied AFTER the element-wise requantise
            // and stereo steps, so it is folded into the load: line d of the sub-band comes from source
            // line s, and every per-line decision below is taken on s.
            float x[2][18];
            uint32_t ivq[5] = {0u, 0u, 0u, 0u, 0u}; // interval of the source line behind my i-th value, 4 per word
            // stereo.rs:550-553 sets both rzero to max(rzero) before reorder / antialias / hybrid see them
            const int rz_joint = max(rz0, rz1);
            const int rze[2] = {(ms || is) ? rz_joint : rz0, (ms || is) ? rz_joint : rz1};
            int rzr[2] = {rze[0], rze[1]}; // rzero after the reorder step
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                if (ch >= n_ch) {
#pragma unroll
                    for (int i = 0; i < 18; ++i) x[ch][i] = 0.0f;
                    continue;
                }
                const int kind = ch ? kind1 : kind0;
                const float* Sc = S + ch * 576;
                if (kind == kKindLong) {
                    const uint16_t* iv2 = reinterpret_cast<const uint16_t*>(tab->iv_of_line[sr][kind] + 18 * lane);
#pragma unroll
                    for (int i = 0; i < 18; i += 2) {
                        const float2 v = *reinterpret_cast<const float2*>(Sc + 18 * lane + i);
                        const unsigned ivp = __ldg(iv2 + (i >> 1));
                        // lines at or beyond rzero are +0.0 by contract (requantize.rs:234): 0 * scale = 0
                        x[ch][i] = v.x * ws.scale[ch][ivp & 0xff];
                        x[ch][i + 1] = v.y * ws.scale[ch][ivp >> 8];
                        if (ch) {
                            ivq[i >> 2] |= ivp << (8 * (i & 3)); // i is even: the pair lands in one word
                            if (is) {
                                if (x[ch][i] != 0.0f) ws.nz[ivp & 0xff] = 1;
                                if (x[ch][i + 1] != 0.0f) ws.nz[ivp >> 8] = 1;
                            }
                        }
                    }
                } else {
                    const int m = (kind == kKindMixed) ? 1 : 0;
                    const int sw = m ? c_mp3.mixed_switch[sr] : 0;
                    const uint16_t* e = tab->edges[sr][kind] + sw;
                    const int n_quads = (c_mp3.n_edges[sr][kind] - sw - 1) / 3;
                    const int rz = rze[ch];
                    const bool below = (lane < n_quads) && ((int)e[3 * lane] < rz);
                    const int n_done = __popc(__ballot_sync(0xffffffffu, below)); // reordered quads form a prefix
                    const int start = e[0], i_end = e[3 * n_done];
                    rzr[ch] = max(rz, i_end); // hybrid_synthesis.rs:213
                    const uint32_t* map = tab->short_map[sr][m] + 18 * lane;
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        const int d = 18 * lane + i;
                        const uint32_t e3 = __ldg(map + i);
                        const bool moved = d >= start && d < i_end;
                        const int s = moved ? (int)(e3 & 1023u) : d;
                        const int iv = moved ? (int)((e3 >> 10) & 63u) : (int)((e3 >> 16) & 63u);
                        x[ch][i] = Sc[s] * ws.scale[ch][iv];
                        if (ch) {
                            ivq[i >> 2] |= (uint32_t)iv << (8 * (i & 3));
                            if (is && x[ch][i] != 0.0f) ws.nz[iv] = 1;
                        }
                    }
                }
            }
            __syncwarp();

            // A3/A4: joint stereo (stereo.rs:485-556), decided per SOURCE line  // PHASE: A3 stereo
            if (ms || is) {
                if (is) {
                    // Warp-parallel restatement of the two top-down scans (stereo.rs:198-261, :265-482).
                    const bool mpeg1 = g1.flags & SYMGPU_MP3_F_MPEG1;
                    const int inv_pos = mpeg1 ? 7 : 31;
                    // ratio table in GLOBAL memory: the position differs from lane to lane, and a constant-bank
                    // operand with a lane-dependent index is replayed once per distinct address
                    const float(*rt)[2] = mpeg1 ? tab->is_mpeg1 : tab->is_mpeg2[(g1.flags & SYMGPU_MP3_F_SFC_LSB) ? 1 : 0];
                    const uint16_t* e = tab->edges[sr][kind1];
                    const int n_e = c_mp3.n_edges[sr][kind1];
                    const int n_iv = n_e - 1;
                    const uint8_t mode_hi = ms ? 1 : 0;
                    bool nza = false, nzb = false;
                    if (lane < n_iv) nza = ws.nz[lane] && (kind1 != kKindLong || (int)e[lane] < rz1);
                    if (lane + 32 < n_iv) nzb = ws.nz[lane + 32] && (kind1 != kKindLong || (int)e[lane + 32] < rz1);
                    const unsigned long long nzmask = (unsigned long long)__ballot_sync(0xffffffffu, nza) |
                                                      ((unsigned long long)__ballot_sync(0xffffffffu, nzb) << 32);
                    int is_lo, first_is0, first_is1, first_is2;
                    if (kind1 == kKindLong) {
                        const int hb = nzmask ? 63 - __clzll((long long)nzmask) : -1; // highest non-zero band
                        is_lo = hb + 1;
                        first_is0 = first_is1 = first_is2 = hb + 1;
                    } else {
                        const int sw = (kind1 == kKindMixed) ? c_mp3.mixed_switch[sr] : 0;
                        const int n_quads = (n_e - sw - 1) / 3;
                        int hq0 = -1, hq1 = -1, hq2 = -1; // highest quad whose window w is non-zero
                        for (int q = 0; q < n_quads; ++q) {
                            const unsigned bits = (unsigned)(nzmask >> (sw + 3 * q)) & 7u;
                            if (bits & 1u) hq0 = q;
                            if (bits & 2u) hq1 = q;
                            if (bits & 4u) hq2 = q;
                        }
                        const int qstop = min(hq0, min(hq1, hq2)); // quad where all three windows are done, or -1
                        const int qlo = max(qstop, 0);
                        is_lo = sw + 3 * qlo;
                        first_is0 = sw + 3 * (hq0 + 1);
                        first_is1 = sw + 3 * (hq1 + 1) + 1;
                        first_is2 = sw + 3 * (hq2 + 1) + 2;
                        if (qstop < 0 && kind1 == kKindMixed) { // continue into the long bands of a mixed block
                            const unsigned long long lmask = nzmask & ((1ull << sw) - 1ull);
                            const int hb = lmask ? 63 - __clzll((long long)lmask) : -1;
                            if (hb < sw - 1) is_lo = hb + 1;
                        }
                    }
                    // Mode of every interval: below the intensity region plain / mid-side, inside it intensity
                    // where the position is valid (process_intensity, stereo.rs:168-188), else plain / mid-side.
                    for (int iv = lane; iv < n_iv; iv += 32) {
                        uint8_t mode = mode_hi;
                        if (iv >= is_lo) {
                            bool coded;
                            if (kind1 == kKindLong) {
                                coded = true;
                            } else {
                                const int sw = (kind1 == kKindMixed) ? c_mp3.mixed_switch[sr] : 0;
                                if (iv < sw) coded = true;
                                else {
                                    const int w = (iv - sw) % 3;
                                    coded = iv >= (w == 0 ? first_is0 : w == 1 ? first_is1 : first_is2);
                                }
                            }
                            if (coded) {
                                const int k = (kind1 == kKindLong) ? (iv == 21 ? 20 : iv) : (iv < 36 ? iv : iv - 3);
                                const int pos = g1.scalefacs[k];
                                if (pos < inv_pos) {
                                    mode = 2;
                                    ws.sratio[iv] = __ldg(reinterpret_cast<const float2*>(rt[pos]));
                                }
                            }
                        }
                        ws.smode[iv] = mode;
                    }
                    __syncwarp();
                    // A line takes the mode of the interval of its SOURCE line (remembered from A2).  Lines at or
                    // beyond max(rzero) are +0.0 in both channels and stay +0.0 under either transform.
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        const int iv = (ivq[i >> 2] >> (8 * (i & 3))) & 0xff;
                        const int mode = ws.smode[iv];
                        const float l = x[0][i], r = x[1][i];
                        if (mode == 2) {
                            const float2 ratio = ws.sratio[iv];
                            x[0][i] = ratio.x * l;
                            x[1][i] = ratio.y * l;
                        } else if (mode == 1) { // process_mid_side, stereo.rs:143-152
                            x[0][i] = (l + r) * kFrac1Sqrt2;
                            x[1][i] = (l - r) * kFrac1Sqrt2;
                        }
                    }
                } else {
                    // Mid-side only: every line below max(rzero); the lines above are +0.0 in both channels and
                    // (0 + 0) * c = (0 - 0) * c = +0.0, so the bound needs no test.
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        const float l = x[0][i], r = x[1][i];
                        x[0][i] = (l + r) * kFrac1Sqrt2;
                        x[1][i] = (l - r) * kFrac1Sqrt2;
                    }
                }
            }

            // A6: antialias (hybrid_synthesis.rs:218-277) across neighbouring lanes  // PHASE: A6 antialias
            int rzh[2]; // rzero seen by hybrid_synthesis
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                const int kind = ch ? kind1 : kind0;
                rzh[ch] = rzr[ch];
                if (ch >= n_ch || kind == kKindShort) continue; // (warp-uniform)
                const int sb_limit = (kind == kKindMixed) ? 2 : 32;
                const int rz = 18 * min(min(sb_limit, rzr[ch] / 18 + 2), 32);
                rzh[ch] = rz;
                float nb_lo[8], nb_up[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    nb_lo[i] = __shfl_up_sync(0xffffffffu, x[ch][17 - i], 1);   // lower[li] of the boundary below me
                    nb_up[i] = __shfl_down_sync(0xffffffffu, x[ch][i], 1);      // upper[ui] of the boundary above me
                }
                const bool do_bottom = lane >= 1 && 18 * lane < rz;
                const bool do_top = lane < 31 && 18 * (lane + 1) < rz;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float up = x[ch][i], lo = x[ch][17 - i];
                    if (do_bottom) x[ch][i] = up * c_mp3.cs[i] + nb_lo[i] * c_mp3.ca[i];       // samples[ui]
                    if (do_top) x[ch][17 - i] = lo * c_mp3.cs[i] - nb_up[i] * c_mp3.ca[i];     // samples[li]
                }
            }

            // B: hybrid synthesis (hybrid_synthesis.rs:280-359)  // PHASE: B glue
            float* X = xt + (size_t)(18 * (reg0 + g - 1)) * kPitch * 2; // unused by job 0 (it only hands its overlap on)
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                float first[18];
                if (ch < n_ch) {
                    const symgpu_mp3_gc& gg = sm.units[warp][ch];
                    const int kind = ch ? kind1 : kind0;
                    const int rz = rzh[ch];
                    const int sb_limit = (rz + 17) / 18;
                    const int sb_split = (kind == kKindShort) ? 0 : (kind == kKindMixed) ? 2 : 32;
                    const int long_end = min(sb_split, sb_limit);
                    if (lane < long_end) {
                        const int wsel = gg.block_type == SYMGPU_MP3_START ? 1 : gg.block_type == SYMGPU_MP3_END ? 3 : 0;
                        imdct36(x[ch], c_mp3.imdct_win[wsel], first, sec[ch]);
                    } else if (lane < sb_limit) {
                        imdct12x3(x[ch], first, sec[ch]);
                    } else {
                        // samples = overlap; overlap = 0 (:351-358).  overlap + (-0.0) == overlap bit for bit.
#pragma unroll
                        for (int i = 0; i < 18; ++i) {
                            first[i] = -0.0f;
                            sec[ch][i] = 0.0f;
                        }
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        first[i] = 0.0f;
                        sec[ch][i] = 0.0f;
                    }
                }
                if (g == 2 && load_state) { // a run's first granule takes the overlap of the stream state
#pragma unroll
                    for (int t = 0; t < 18; ++t) first[t] = first[t] + st_in->overlap[ch][lane][t];
                }
                if (g >= 1) {
#pragma unroll
                    for (int t = 0; t < 18; ++t) X[(t * kPitch + lane) * 2 + ch] = finv(first[t], lane, t);
                }
            }
        }
        __syncthreads();  // PHASE: handoff+barriers
        // The stage is free: fetch this CTA's next group while the current one is in its DCT / window phases.
        if (threadIdx.x == NW * 32 - 32 && ti + nseg < t_end) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue_prefetch(ti + nseg, (it + 1) & 1);
        }
        // overlap hand-off: region of job g+1 += second(g); the piece's last granule feeds the stream state
        {
            const int next_region = ws.next_region;
            Mp3StreamState* so = ws.st_out;
            if (next_region >= 0) {
                float* Xn = xt + (size_t)(18 * next_region) * kPitch * 2;
#pragma unroll
                for (int ch = 0; ch < 2; ++ch)
#pragma unroll
                    for (int t = 0; t < 18; ++t) {
                        float* p = Xn + (t * kPitch + lane) * 2 + ch;
                        *p = *p + finv(sec[ch][t], lane, t);
                    }
            } else if (so) {
#pragma unroll
                for (int ch = 0; ch < 2; ++ch)
#pragma unroll
                    for (int t = 0; t < 18; ++t) so->overlap[ch][lane][t] = sec[ch][t];
            }
        }
        // polyphase history (rows 3..17 of a piece's first region) from the state of every piece that has one
        {
            int regions = 0;
            for (int k = 0; k < nseg; ++k) {
                const Mp3Tile t = sm.seg_stage[par][k];
                if (t.flags & (kTileLoadState | kTileCarryIn)) {
                    const uint32_t gk = sm.gen_stage[par][k];
                    const Mp3StreamState* st = (t.flags & kTileCarryIn) ? &sm.carry : a.states + (size_t)t.stream * 2 + (gk & 1);
                    for (int idx = threadIdx.x; idx < 15 * kPitch; idx += NW * 32) {
                        const int srow = idx / kPitch, col = idx - srow * kPitch;
                        float2 v = make_float2(0.0f, 0.0f);
                        if (col < 32) v = st->dhist[srow][col];
                        *reinterpret_cast<float2*>(xt + (size_t)((18 * regions + 3 + srow) * kPitch + col) * 2) = v;
                    }
                }
                regions += t.n_granules + 1;
            }
        }
        __syncthreads();

        // --------------------------------------------------------------------------------------
        // Phase C: DCT-32 of every time slot of the group, in place.  Half-warp = 16 slots of one  // PHASE: C glue
        // channel: the 32-bit accesses of a warp hit 32 distinct banks (row pitch 66 words).  The rows of the
        // pieces are enumerated back to back: a piece with state has 18 n rows from its second region on, a
        // piece with a halo also recomputes the 15 history rows of its first region.
        // --------------------------------------------------------------------------------------
        {
            int total_rows = 0;
            for (int k = 0; k < nseg; ++k) {
                const Mp3Tile t = sm.seg_stage[par][k];
                total_rows += 18 * t.n_granules + ((t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : 15);
            }
            const int chn = lane >> 4;
            for (int base = warp * 16; base < total_rows; base += NW * 16) {
                int r = base + (lane & 15);
                if (r < total_rows) {
                    int regions = 0, row = 0;
                    for (int k = 0; k < nseg; ++k) { // piece that holds enumerated row r
                        const Mp3Tile t = sm.seg_stage[par][k];
                        const int lead = (t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : 15;
                        const int cnt = 18 * t.n_granules + lead;
                        if (r < cnt) {
                            row = 18 * regions + 18 - lead + r;
                            break;
                        }
                        r -= cnt;
                        regions += t.n_granules + 1;
                    }
                    float* rowp = xt + (size_t)row * kPitch * 2 + chn;
                    float v[32], y[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] = rowp[2 * i];
                    lee_dct<32>(v, y);
#pragma unroll
                    for (int i = 0; i < 32; ++i) rowp[2 * i] = y[i];
                    rowp[64] = 0.0f; // column 32: V[16] = 0.0 (synthesis.rs:263)
                }
            }
        }
        __syncthreads();

        // Phase D: polyphase window (synthesis.rs:247-263, :309-327), see window_phase().  The group's slots are  // PHASE: D glue+epilogue
        // enumerated back to back and dealt out in equal shares; a warp's share may span pieces.
        {
            int total_slots = 0;
            for (int k = 0; k < nseg; ++k) total_slots += 18 * sm.seg_stage[par][k].n_granules;
            const int per = (total_slots + NW - 1) / NW;
            const int my_begin = warp * per, my_end = min(total_slots, my_begin + per);
            int regions = 0, first = 0;
            for (int k = 0; k < nseg; ++k) {
                const Mp3Tile t = sm.seg_stage[par][k];
                const int cnt = 18 * t.n_granules;
                const int b = max(my_begin, first) - first, e = min(my_end, first + cnt) - first;
                if (b < e) {
                    const int shift = t.gpf == 2 ? 1 : 0;
                    const int gseq = ((int)t.first_frame << shift) + t.first_gr;
                    window_phase(xt, 18 * (regions + 1), b, e, lane, tab->synth_d, a.pcm, gseq * 18, 18 << shift, t.n_ch == 2);
                }
                first += cnt;
                regions += t.n_granules + 1;
            }
        }
        __syncthreads();
        // A piece that ends its run (or hands over to the next group) publishes the polyphase history: its last 15
        // DCT vectors.
        {
            int regions = 0;
            for (int k = 0; k < nseg; ++k) {
                const Mp3Tile t = sm.seg_stage[par][k];
                if (t.flags & (kTileStoreState | kTileCarryOut)) {
                    const uint32_t gk = sm.gen_stage[par][k];
                    Mp3StreamState* st = (t.flags & kTileCarryOut) ? &sm.carry : a.states + (size_t)t.stream * 2 + ((gk + 1) & 1);
                    const float* last = xt + (size_t)(18 * (regions + t.n_granules + 1) - 15) * kPitch * 2;
                    for (int idx = threadIdx.x; idx < 15 * 32; idx += NW * 32) {
                        const int srow = idx >> 5, col = idx & 31;
                        st->dhist[srow][col] = *reinterpret_cast<const float2*>(last + (size_t)(srow * kPitch + col) * 2);
                    }
                }
                regions += t.n_granules + 1;
            }
        }
        ti += nseg;
        __syncthreads(); // XT and the stage descriptors are reused by the next group
    }

    // Launch epilogue: the last CTA to retire publishes the new state generation of every run.
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        sm.is_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (sm.is_last) {
        for (int i = threadIdx.x; i < n_tiles; i += NW * 32)
            if (a.tiles[i].flags & kTileStoreState) a.gen[a.tiles[i].stream] += 1;
        if (threadIdx.x == 0) *a.done = 0;
    }
}

// =============================================================================================
// MPEG Layer I / II: polyphase synthesis only (synthesis.rs:158-344 called with n_frames = 12 / 36 from
// layer1/mod.rs:184-194 and layer2/mod.rs:374-384).  The sub-band samples the layer decoders produce go
// straight into XT rows; phases C (DCT-32) and D (window) are the Layer III kernel's.  A CTA walks a chain of
// tiles of whole frames of one stream; the 15 history vectors come from the stream state (run start), stay in
// shared memory between the tiles of a chain, or are recomputed from the previous frames' samples (a chain
// that starts inside a run).
// =============================================================================================
namespace {
constexpr int kMpa12Slots = 288; // time slots per tile: 8 Layer II frames or 24 Layer I frames
struct Mpa12Smem {
    float xt[(18 + kMpa12Slots) * kPitch * 2];
    bool is_last;
};
} // namespace

template <int NW>
__global__ void __launch_bounds__(NW * 32, 1) mpa12_synth_kernel(Mpa12Args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Mpa12Smem& sm = *reinterpret_cast<Mpa12Smem*>(smem_raw);
    float* xt = sm.xt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n_slots = a.n_slots;
    const Mp3Tables* __restrict__ tab = a.tab;
    const int t_begin = (int)a.cta_first[blockIdx.x], t_end = (int)a.cta_first[blockIdx.x + 1];
    for (int ti = t_begin; ti < t_end; ++ti) {
        const Mp3Tile tile = a.tiles[ti];
        const int n = tile.n_granules; // frames
        const int total = n * n_slots;
        const bool from_state = tile.flags & kTileLoadState, carried = tile.flags & kTileCarryIn;
        const uint32_t gen = a.gen[tile.stream];
        const Mp3StreamState* st_in = a.states + (size_t)tile.stream * 2 + (gen & 1);
        Mp3StreamState* st_out = a.states + (size_t)tile.stream * 2 + ((gen + 1) & 1);
        const float* in = a.subbands + (size_t)tile.first_frame * 64 * n_slots;
        // history rows 3..17: DCT vectors from the state, or (halo) the raw samples of the 15 slots before the tile
        if (from_state) {
            for (int idx = threadIdx.x; idx < 15 * kPitch; idx += NW * 32) {
                const int srow = idx / kPitch, col = idx - srow * kPitch;
                float2 v = make_float2(0.0f, 0.0f);
                if (col < 32) v = st_in->dhist[srow][col];
                *reinterpret_cast<float2*>(xt + (size_t)((3 + srow) * kPitch + col) * 2) = v;
            }
        } else if (!carried) {
            for (int idx = threadIdx.x; idx < 15 * 64; idx += NW * 32) {
                const int j = idx >> 6, sb = (idx >> 1) & 31, ch = idx & 1;
                const int gslot = (int)tile.first_frame * n_slots - 15 + j; // >= 0: two earlier frames of the run are in the batch
                const int f = gslot / n_slots, s = gslot - f * n_slots;
                float v = 0.0f;
                if (ch < tile.n_ch) v = __ldg(a.subbands + ((size_t)(f * 2 + ch) * 32 + sb) * n_slots + s);
                xt[((3 + j) * kPitch + sb) * 2 + ch] = v;
            }
        }
        // the tile's samples: in[((f * 2 + ch) * 32 + sb) * n_slots + s] -> row 18 + f * n_slots + s, column sb.
        // A thread takes one (frame, sub-band): it reads the n_slots samples of both channels (two contiguous runs
        // of 48 / 144 bytes, float4 loads) and writes (ch0, ch1) pairs -- 64-bit stores, lanes on distinct banks.
        {
            const bool stereo = tile.n_ch == 2;
            for (int pair = threadIdx.x; pair < n * 32; pair += NW * 32) {
                const int f = pair >> 5, sb = pair & 31;
                const float4* s0 = reinterpret_cast<const float4*>(in + ((size_t)(f * 2) * 32 + sb) * n_slots);
                const float4* s1 = reinterpret_cast<const float4*>(in + ((size_t)(f * 2 + 1) * 32 + sb) * n_slots);
                float2* dst = reinterpret_cast<float2*>(xt) + (size_t)(18 + f * n_slots) * kPitch + sb;
                for (int q = 0; q < n_slots / 4; ++q) {
                    const float4 a0 = __ldg(s0 + q);
                    const float4 a1 = stereo ? __ldg(s1 + q) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    dst[(4 * q + 0) * kPitch] = make_float2(a0.x, a1.x);
                    dst[(4 * q + 1) * kPitch] = make_float2(a0.y, a1.y);
                    dst[(4 * q + 2) * kPitch] = make_float2(a0.z, a1.z);
                    dst[(4 * q + 3) * kPitch] = make_float2(a0.w, a1.w);
                }
            }
        }
        __syncthreads();
        { // Phase C
            const int row_begin = (from_state || carried) ? 18 : 3;
            const int row_end = 18 + total;
            const int chn = lane >> 4;
            for (int base = row_begin + warp * 16; base < row_end; base += NW * 16) {
                const int r = base + (lane & 15);
                if (r < row_end) {
                    float* rowp = xt + (size_t)r * kPitch * 2 + chn;
                    float v[32], y[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] = rowp[2 * i];
                    lee_dct<32>(v, y);
#pragma unroll
                    for (int i = 0; i < 32; ++i) rowp[2 * i] = y[i];
                    rowp[64] = 0.0f;
                }
            }
        }
        __syncthreads();
        { // Phase D
            const int per = (total + NW - 1) / NW;
            const int b = warp * per, e = min(total, b + per);
            window_phase<true>(xt, 18, b, e, lane, tab->synth_d, a.pcm, (int)tile.first_frame * n_slots, n_slots, tile.n_ch == 2);
        }
        __syncthreads();
        // the last 15 DCT vectors: rows 3 + total .. 17 + total (older history rows included when total < 15)
        if (tile.flags & (kTileStoreState | kTileCarryOut)) {
            float2 keep[(15 * kPitch + NW * 32 - 1) / (NW * 32)];
            int k = 0;
            for (int idx = threadIdx.x; idx < 15 * kPitch; idx += NW * 32, ++k) {
                const int srow = idx / kPitch, col = idx - srow * kPitch;
                keep[k] = *reinterpret_cast<const float2*>(xt + (size_t)((3 + total + srow) * kPitch + col) * 2);
            }
            __syncthreads();
            k = 0;
            for (int idx = threadIdx.x; idx < 15 * kPitch; idx += NW * 32, ++k) {
                const int srow = idx / kPitch, col = idx - srow * kPitch;
                if (tile.flags & kTileStoreState) {
                    if (col < 32) st_out->dhist[srow][col] = keep[k];
                } else {
                    *reinterpret_cast<float2*>(xt + (size_t)((3 + srow) * kPitch + col) * 2) = keep[k];
                }
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        __threadfence();
        sm.is_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (sm.is_last) {
        for (int i = threadIdx.x; i < a.n_tiles; i += NW * 32)
            if (a.tiles[i].flags & kTileStoreState) a.gen[a.tiles[i].stream] += 1;
        if (threadIdx.x == 0) *a.done = 0;
    }
}

int mpa12_tile_frames(int n_slots) { return n_slots > 0 ? kMpa12Slots / n_slots : 0; }

cudaError_t mpa12_launch(const Mpa12Args& a, cudaStream_t stream) {
    constexpr size_t smem = sizeof(Mpa12Smem);
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(mpa12_synth_kernel<kMp3Warps>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    if (a.n_ctas <= 0) return cudaErrorInvalidConfiguration;
    mpa12_synth_kernel<kMp3Warps><<<a.n_ctas, kMp3Warps * 32, smem, stream>>>(a);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Granules per tile of the launch plan (<= kMp3TileGranules).  SYMGPU_MP3_T overrides it (tuning): with 14 granules a tile's
// 504 DCT vectors fit the 512 threads in one round and its 252 time slots are 16 per warp, one window block each.
int mp3_tile_granules() {
    static int t = 0;
    if (!t) {
        t = kMp3TileGranules;
        if (const char* env = getenv("SYMGPU_MP3_T")) {
            const int v = atoi(env);
            if (v >= 4 && v <= kMp3TileGranules) t = v;
        }
    }
    return t;
}
int mp3_cta_warps() { return kMp3Warps; }
int mp3_halo_tile_granules() { return kMp3Warps - 2 < mp3_tile_granules() ? kMp3Warps - 2 : mp3_tile_granules(); }

int mp3_grid_size(cudaError_t* err) {
    constexpr size_t smem = sizeof(Mp3Smem<kMp3TileGranules, kMp3Warps>);
    static int grid_for_device[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess && !grid_for_device[dev & 63]) {
        int n_sm = 0, per_sm = 0;
        e = cudaFuncSetAttribute(mp3_synth_kernel<kMp3TileGranules, kMp3Warps, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(mp3_synth_kernel<kMp3TileGranules, kMp3Warps, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
        if (e == cudaSuccess)
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mp3_synth_kernel<kMp3TileGranules, kMp3Warps, true>, kMp3Warps * 32, smem);
        if (e == cudaSuccess) grid_for_device[dev & 63] = n_sm * (per_sm > 0 ? per_sm : 1);
    }
    if (err) *err = e;
    return e == cudaSuccess ? grid_for_device[dev & 63] : 0;
}

cudaError_t mp3_launch(const Mp3Args& a, cudaStream_t stream) {
    constexpr size_t smem = sizeof(Mp3Smem<kMp3TileGranules, kMp3Warps>);
    cudaError_t e = cudaSuccess;
    const int max_grid = mp3_grid_size(&e);
    if (e != cudaSuccess) return e;
    if (a.n_ctas <= 0 || a.n_ctas > max_grid) return cudaErrorInvalidConfiguration;
    if (a.multi_tile_groups)
        mp3_synth_kernel<kMp3TileGranules, kMp3Warps, true><<<a.n_ctas, kMp3Warps * 32, smem, stream>>>(a);
    else
        mp3_synth_kernel<kMp3TileGranules, kMp3Warps, false><<<a.n_ctas, kMp3Warps * 32, smem, stream>>>(a);
    return cudaGetLastError();
}

} // namespace symgpu
