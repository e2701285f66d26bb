// Fused MPEG Layer III synthesis kernel for sm_90a, second generation ("v2"):
//   requantize -> joint stereo -> reorder -> antialias -> IMDCT-36/12 + window + overlap-add
//   -> frequency inversion -> DCT-32 -> 512-tap polyphase window  (layer3/mod.rs:421-477)
// in ONE launch, PCM written straight to HBM.
//
// What changed against mp3_kernel.cu (CTA-wide barriers between phases, a large instruction footprint per tile):
//
//  * WARP-AUTONOMOUS.  A warp owns a SHARE: a contiguous piece of the batch's granules in run order.  It walks
//    its granules one at a time through every phase with nothing but __syncwarp() -- no CTA barrier, no
//    hand-off pass, no tile/group bookkeeping.  The hybrid overlap of the previous granule stays in REGISTERS
//    (18 float2 per lane), the last 15 DCT vectors stay in the warp's two-region XT ring in shared memory,
//    the next granule's spectra arrive by a per-warp TMA bulk copy (cp.async.bulk -> mbarrier) issued as
//    soon as the current granule's lines are in registers.  12 warps per SM (3 per scheduler, 168
//    registers; under sm_90a the granule loop spills a few words -- tile loads, the TMA issue, the call of the
//    out-of-line mixed-block helper -- and that helper passes its operands through local memory by design), each in its own phase, share the issue slots; a stall of one warp is filled by
//    the others instead of being multiplied by a barrier.
//  * CHANNEL PAIRS.  Every value on the path exists once per channel, so lane data is held as float2
//    (ch0, ch1): one body of code serves both channels.  Hopper has no packed FP32 arithmetic, so each pair
//    operation is two scalar __fmul_rn / __fadd_rn / __fsub_rn, which the compiler never contracts into an FMA
//    (bit-exactness); tests/test_build_and_abi.py holds the SASS to that: no FFMA anywhere.
//  * One instruction stream for the whole granule loop (one IMDCT-36 body for both channels, one
//    DCT-32 body, one window body), so twelve warps in different phases still fit the instruction caches.
//
// A share that starts inside a run recomputes a 2-granule halo (hybrid of g-2 for its overlap, hybrid + DCT
// of g-1 for the 15 history vectors), exactly as round 1's tiles did; a share that starts a run takes
// overlap + history from the stream state in HBM (double-buffered by a generation counter).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "../../include/symgpu.h"
#include "mp3_kernel.h"
#include "tables.h"

namespace symgpu {

struct Mp3ConstV2 {
    float win_s[4][36];        // imdct windows with the sign of the fold folded in: +w (i < 9), -w (i >= 9)
    float win12[12];           // short window (imdct_win[2][0..11])
    float half_cos12[6][6];
    float dct_iv_scale[18];
    float sdct18_scale[9];
    float sdct9_d[7];
    float lee16[16], lee8[8], lee4[4], lee2[2], lee1;
    float cs[8], ca[8];
    uint8_t pre_emphasis[24];
    uint8_t mixed_switch[12];
    uint8_t n_edges[9][3];
};
__constant__ Mp3ConstV2 c2;

cudaError_t mp3v2_upload_const(const Mp3Tables& t, cudaStream_t stream) {
    static Mp3ConstV2 h; // staging must outlive the async copy
    for (int k = 0; k < 4; ++k)
        for (int i = 0; i < 36; ++i) h.win_s[k][i] = i < 9 ? t.imdct_win[k][i] : -t.imdct_win[k][i];
    memcpy(h.win12, t.imdct_win[2], sizeof h.win12);
    memcpy(h.half_cos12, t.half_cos12, sizeof h.half_cos12);
    memcpy(h.dct_iv_scale, t.dct_iv_scale, sizeof h.dct_iv_scale);
    memcpy(h.sdct18_scale, t.sdct18_scale, sizeof h.sdct18_scale);
    memcpy(h.sdct9_d, t.sdct9_d, sizeof h.sdct9_d);
    memcpy(h.lee16, t.lee16, sizeof h.lee16);
    memcpy(h.lee8, t.lee8, sizeof h.lee8);
    memcpy(h.lee4, t.lee4, sizeof h.lee4);
    memcpy(h.lee2, t.lee2, sizeof h.lee2);
    h.lee1 = t.lee1;
    memcpy(h.cs, t.cs, sizeof h.cs);
    memcpy(h.ca, t.ca, sizeof h.ca);
    memcpy(h.pre_emphasis, t.pre_emphasis, sizeof h.pre_emphasis);
    memset(h.mixed_switch, 0, sizeof h.mixed_switch);
    memcpy(h.mixed_switch, t.mixed_switch, 9);
    memcpy(h.n_edges, t.n_edges, sizeof h.n_edges);
    cudaError_t e = cudaMemcpyToSymbolAsync(c2, &h, sizeof h, 0, cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(stream);
}

namespace {

using f2 = float2;
constexpr int kPitch = 33;            // float2 per XT row: 32 sub-bands + one always-zero column (V[16] = 0)
constexpr uint32_t kRowBytes = kPitch * 8;
constexpr float kFrac1Sqrt2 = 0.707106781186547524400844362104849039f;

// ---- channel-pair arithmetic: one correctly rounded scalar operation per channel, never contracted ----  // PHASE: pair ops
struct Ops {
    __device__ __forceinline__ f2 mul(f2 a, f2 b) const { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
    __device__ __forceinline__ f2 mul(f2 a, float s) const { return mul(a, make_float2(s, s)); }
    __device__ __forceinline__ f2 add(f2 a, f2 b) const { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
    __device__ __forceinline__ f2 sub(f2 a, f2 b) const { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
};

struct WarpSmem {
    alignas(16) float2 xt[36 * kPitch];      // two regions of 18 rows: the granule in flight and the one before it
    alignas(16) float spec[2 * 576];         // TMA destination: spectra of the granule in flight, [ch][576]
    alignas(16) symgpu_mp3_gc units[2][2];   // TMA destination (double-buffered): its descriptors
    float scale[2][40];
    float2 sratio[40];
    uint8_t smode[40]; // 0 none, 1 mid/side, 2 intensity
    uint8_t nz[40];    // channel-1 interval holds a non-zero line
    alignas(8) uint64_t bar;
};

__device__ __forceinline__ int kind_of(const symgpu_mp3_gc& g) {
    if (g.block_type != SYMGPU_MP3_SHORT) return kKindLong;
    return (g.flags & SYMGPU_MP3_F_MIXED) ? kKindMixed : kKindShort;
}

// ---- 9-point SDCT-II (hybrid_synthesis.rs:721-779), both channels; y[j] is the reference's y[2j] ----  // PHASE: B imdct36
__device__ __forceinline__ void sdct9(const Ops& o, const f2 (&x)[9], f2 (&y)[9]) {
    const f2 a01 = o.add(x[3], x[5]), a02 = o.sub(x[3], x[5]), a03 = o.add(x[6], x[2]), a04 = o.sub(x[6], x[2]);
    const f2 a05 = o.add(x[1], x[7]), a06 = o.sub(x[1], x[7]), a07 = o.add(x[8], x[0]), a08 = o.sub(x[8], x[0]);
    const f2 a09 = o.add(x[4], a05), a10 = o.add(a01, a03), a11 = o.add(a10, a07), a12 = o.sub(a03, a07);
    const f2 a13 = o.sub(a01, a07), a14 = o.sub(a01, a03), a15 = o.sub(a02, a04), a16 = o.add(a15, a08);
    const f2 a17 = o.add(a04, a08), a18 = o.sub(a02, a08), a19 = o.add(a02, a04), a20 = o.sub(o.mul(x[4], 2.0f), a05);
    const f2 m1 = o.mul(a06, c2.sdct9_d[0]), m2 = o.mul(a12, c2.sdct9_d[1]), m3 = o.mul(a13, c2.sdct9_d[2]);
    const f2 m4 = o.mul(a14, c2.sdct9_d[3]), m5 = o.mul(a16, c2.sdct9_d[0]), m6 = o.mul(a17, c2.sdct9_d[4]);
    const f2 m7 = o.mul(a18, c2.sdct9_d[5]), m8 = o.mul(a19, c2.sdct9_d[6]);
    const f2 a21 = o.add(a20, m2), a22 = o.sub(a20, m2), a23 = o.add(a20, m3), a24 = o.add(m1, m6), a25 = o.sub(m1, m6),
             a26 = o.add(m1, m7);
    y[0] = o.add(a09, a11);
    y[1] = o.sub(m8, a26);
    y[2] = o.sub(m4, a21);
    y[3] = m5;
    y[4] = o.sub(a22, m3);
    y[5] = o.sub(a25, m7);
    y[6] = o.sub(a11, o.mul(a09, 2.0f));
    y[7] = o.add(a24, m8);
    y[8] = o.add(a23, m4);
}

// ---- 18-point DCT-IV via two 9-point SDCT-IIs (hybrid_synthesis.rs:608-716) -----------------
__device__ __forceinline__ void dct_iv_18(const Ops& o, const f2 (&x)[18], f2 (&y)[18]) {
    f2 s[18];
#pragma unroll
    for (int i = 0; i < 18; ++i) s[i] = o.mul(x[i], c2.dct_iv_scale[i]);
    f2 even[9], odd[9], ye[9], yo[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) even[i] = o.add(s[i], s[17 - i]);
    sdct9(o, even, ye);
#pragma unroll
    for (int i = 0; i < 9; ++i) odd[i] = o.mul(o.sub(s[i], s[17 - i]), c2.sdct18_scale[i]);
    sdct9(o, odd, yo);
#pragma unroll
    for (int j = 1; j < 9; ++j) yo[j] = o.sub(yo[j], yo[j - 1]); // y[3]-=y[1]; y[5]-=y[3]; ... sequential
#pragma unroll
    for (int j = 0; j < 9; ++j) {
        y[2 * j] = ye[j];
        y[2 * j + 1] = yo[j];
    }
    y[0] = o.mul(y[0], 0.5f); // "/ 2.0" -- exact either way
#pragma unroll
    for (int i = 1; i < 18; ++i) y[i] = o.sub(o.mul(y[i], 0.5f), y[i - 1]);
}

// imdct36 (hybrid_synthesis.rs:571-603) without the overlap add: first = windowed samples 0..17, second =
// windowed samples 18..35 (the next granule's overlap), from the 18-point DCT-IV.  Window signs are folded into
// the table (win_s).  LONG2: both channels use the normal window (block type 0): immediate constant operands.
template <bool LONG2>
__device__ __forceinline__ void imdct36_window(const Ops& o, const f2 (&dct)[18], int wsel0, int wsel1, f2 (&first)[18],
                                               f2 (&second)[18]) {
    auto w = [&](int i) -> f2 {
        if (LONG2) return make_float2(c2.win_s[0][i], c2.win_s[0][i]);
        return make_float2(c2.win_s[wsel0][i], c2.win_s[wsel1][i]);
    };
#pragma unroll
    for (int i = 0; i < 9; ++i) first[i] = o.mul(dct[9 + i], w(i));
#pragma unroll
    for (int i = 9; i < 18; ++i) first[i] = o.mul(dct[26 - i], w(i));
#pragma unroll
    for (int i = 18; i < 27; ++i) second[i - 18] = o.mul(dct[26 - i], w(i));
#pragma unroll
    for (int i = 27; i < 36; ++i) second[i - 18] = o.mul(dct[i - 27], w(i));
}
__device__ __forceinline__ void imdct36(const Ops& o, const f2 (&x)[18], int wsel0, int wsel1, f2 (&first)[18], f2 (&second)[18]) {
    f2 dct[18];
    dct_iv_18(o, x, dct);
    if (wsel0 == 0 && wsel1 == 0) imdct36_window<true>(o, dct, 0, 0, first, second);
    else imdct36_window<false>(o, dct, wsel0, wsel1, first, second);
}

// imdct12_win (hybrid_synthesis.rs:363-455) without the overlap add, both channels.  // PHASE: B imdct12
// The reference accumulates into a zeroed 36-sample buffer: tmp[k] = (0.0 + a) [+ b]; the "+ 0.0" is kept
// (it turns a -0.0 product into +0.0).  Window w writes tmp[6 + 6w .. 6 + 6w + 11].
__device__ __forceinline__ void imdct12x3(const Ops& o, const f2 (&x)[18], f2 (&first)[18], f2 (&second)[18]) {
    const f2 zero = make_float2(0.0f, 0.0f);
    f2 tmp[36];
#pragma unroll
    for (int i = 0; i < 36; ++i) tmp[i] = zero;
#pragma unroll
    for (int w = 0; w < 3; ++w) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            f2 yl = o.mul(x[w], c2.half_cos12[i][0]);
            f2 yr = o.mul(x[w], c2.half_cos12[i + 3][0]);
#pragma unroll
            for (int k = 1; k < 6; ++k) {
                yl = o.add(yl, o.mul(x[3 * k + w], c2.half_cos12[i][k]));
                yr = o.add(yr, o.mul(x[3 * k + w], c2.half_cos12[i + 3][k]));
            }
            // tmp[..] += -yl * win[2 - i]  ==  tmp[..] + yl * (-win[2 - i])
            tmp[6 + 6 * w + 2 - i] = o.add(tmp[6 + 6 * w + 2 - i], o.mul(yl, -c2.win12[2 - i]));
            tmp[6 + 6 * w + i + 3] = o.add(tmp[6 + 6 * w + i + 3], o.mul(yl, c2.win12[i + 3]));
            tmp[6 + 6 * w + i + 6] = o.add(tmp[6 + 6 * w + i + 6], o.mul(yr, c2.win12[i + 6]));
            tmp[6 + 6 * w + 11 - i] = o.add(tmp[6 + 6 * w + 11 - i], o.mul(yr, c2.win12[11 - i]));
        }
    }
#pragma unroll
    for (int i = 0; i < 18; ++i) {
        first[i] = tmp[i];
        second[i] = tmp[i + 18];
    }
}

// A sub-band in which one channel is long and the other short: both transforms, component-wise choice.  Only
// frames without mid-side or intensity stereo reach it (stereo, dual-channel, joint stereo with mode_ext 0), where
// each channel switches windows on its own; in such streams it is common wherever one channel is on short blocks.
// Kept out of line with its operands in local memory so that its register needs do not shape the granule loop.
__device__ __noinline__ void hybrid_mixed(const f2* xin, int wsel0, int wsel1, int cat0, int cat1, f2* fout, f2* sout) {
    const Ops o{};
    f2 x[18], fa[18], sa[18], fb[18], sb[18];
#pragma unroll
    for (int i = 0; i < 18; ++i) x[i] = xin[i];
    imdct36(o, x, wsel0, wsel1, fa, sa);
#pragma unroll
    for (int i = 0; i < 18; ++i) {
        fout[i] = fa[i];
        sout[i] = sa[i];
    }
    imdct12x3(o, x, fb, sb);
#pragma unroll
    for (int i = 0; i < 18; ++i) {
        f2 f = fout[i], s2 = sout[i];
        if (cat0 != 36) {
            f.x = fb[i].x;
            s2.x = sb[i].x;
        }
        if (cat1 != 36) {
            f.y = fb[i].y;
            s2.y = sb[i].y;
        }
        fout[i] = f;
        sout[i] = s2;
    }
}

// ---- Lee 32-point DCT (synthesis.rs:348-844) as the recursion the reference hand-flattens, both channels ----  // PHASE: C dct32
template <int N> struct LeeCoef;
template <> struct LeeCoef<16> { static __device__ __forceinline__ float at(int i) { return c2.lee16[i]; } };
template <> struct LeeCoef<8> { static __device__ __forceinline__ float at(int i) { return c2.lee8[i]; } };
template <> struct LeeCoef<4> { static __device__ __forceinline__ float at(int i) { return c2.lee4[i]; } };
template <> struct LeeCoef<2> { static __device__ __forceinline__ float at(int i) { return c2.lee2[i]; } };

template <int N>
__device__ __forceinline__ void lee_dct(const Ops& o, const f2 (&x)[N], f2 (&y)[N]) {
    if constexpr (N == 2) {
        y[0] = o.add(x[0], x[1]);
        y[1] = o.mul(o.sub(x[0], x[1]), c2.lee1);
    } else {
        constexpr int H = N / 2;
        f2 lo[H], hi[H], lo_t[H], hi_t[H];
#pragma unroll
        for (int i = 0; i < H; ++i) {
            lo[i] = o.add(x[i], x[N - 1 - i]);
            hi[i] = o.mul(o.sub(x[i], x[N - 1 - i]), LeeCoef<H>::at(i));
        }
        lee_dct<H>(o, lo, lo_t);
        lee_dct<H>(o, hi, hi_t);
#pragma unroll
        for (int i = 0; i < H - 1; ++i) {
            y[2 * i] = lo_t[i];
            y[2 * i + 1] = o.add(hi_t[i], hi_t[i + 1]);
        }
        y[N - 2] = lo_t[H - 1];
        y[N - 1] = hi_t[H - 1];
    }
}

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
__device__ __forceinline__ f2 lds64(uint32_t addr) {
    f2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, f2 v) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// A warp's position in its share is (ti, k): tile ti, granule k of it (k = -2, -1: the halo granules before
// the tile's first granule).  Tile descriptors are re-read where they are needed (one 16-byte load that hits
// L1) instead of being carried in registers through the whole granule loop.
__device__ __forceinline__ Mp3Tile ld_tile(const Mp3Tile* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    Mp3Tile t;
    t.first_frame = v.x;
    t.stream = v.y;
    t.first_gr = (uint16_t)(v.z & 0xffffu);
    t.n_granules = (uint16_t)(v.z >> 16);
    t.gpf = (uint8_t)(v.w & 0xffu);
    t.n_ch = (uint8_t)((v.w >> 8) & 0xffu);
    t.flags = (uint8_t)((v.w >> 16) & 0xffu);
    t.pad = 0;
    return t;
}
__device__ __forceinline__ int tile_first_k(const Mp3Tile& t) { return (t.flags & (kTileLoadState | kTileCarryIn)) ? 0 : -2; }
// Index of granule k of tile t in units of granule slots ([frame][gr]): spectra at 1152 floats, descriptors at 2 per slot.
__device__ __forceinline__ size_t granule_slot(const Mp3Tile& t, int k) {
    if (t.gpf == 2) return (size_t)t.first_frame * 2 + t.first_gr + k;
    return (size_t)((int)t.first_frame + t.first_gr + k) * 2;
}

template <int NW>
struct Mp3V2Smem {
    WarpSmem w[NW];
    alignas(8) uint64_t lag_bar[3];
    int max_iters;
    bool is_last;
};

// Variant bits (experiments, SYMGPU_MP3_V2_VARIANT=<warps>:<mode>):
//   1  LOCKSTEP: the CTA's warps meet at three named-barrier points per granule.  No data crosses them -- they only
//      keep the warps in the same stretch of code, so that one instruction fetch serves all of them.
//   2  WIN_SCALAR_ADD: the polyphase window accumulates with two scalar FADD per product pair instead of one FFMA2
//      (FFMA2 issues once per 3 cycles, two FADD take 2 cycles of the same pipe but 2 issue slots).
//   4 / 8  WIN_GROUP2 / WIN_GROUP3: the window accumulates 2 / 3 time slots side by side (independent dependency chains).
//   16 / 32  (with LOCKSTEP) only the first / the first two of the three meeting points: the warps re-align once per granule
//      and may drift by a phase in between.
enum : int { kV2Lockstep = 1, kV2WinScalarAdd = 2, kV2WinGroup2 = 4, kV2WinGroup3 = 8, kV2SyncTopOnly = 16, kV2SyncTopHybrid = 32, kV2Compact = 64, kV2Lagged = 128 };
//   128  LAGGED (with LOCKSTEP): a meeting point lets a warp through once every warp has passed the PREVIOUS point (mbarrier
//      arrive here, wait for the one before): the warps stay within one phase of each other, so the instruction stream stays
//      shared, but a warp delayed in one phase (a short-block or intensity-stereo granule) is waited for one phase later,
//      when the delays of different warps have had a chance to even out.
//   64  COMPACT: smaller instruction footprint (the channel loop of the load phase and the two halves of the window are
//      rolled), a few register moves more: for warps that are NOT kept in lockstep and must share the instruction caches.

} // namespace

template <int NW, int MODE>
__global__ void __launch_bounds__(NW * 32, (NW <= 6 ? 12 / NW : 1)) mp3v2_synth_kernel(Mp3V2Args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using Smem = Mp3V2Smem<NW>;
    Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
    constexpr bool LOCK = (MODE & kV2Lockstep) != 0;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    uint32_t lag_round = 0; // meeting points passed so far (LAGGED)
    auto phase_sync = [&](int point = 0) {
        if (!LOCK) return;
        if constexpr ((MODE & kV2Lagged) != 0) {
            // point p of round r: arrive on bar[p]; wait until bar[(p + 2) % 3] has completed the point before this one
            if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&sm.lag_bar[point])) : "memory");
            if (lag_round > 0) {
                const int prev = (point + 2) % 3;
                const uint32_t uses = (lag_round - 1) / 3; // completed phases of bar[prev] before the one awaited
                mbar_wait(&sm.lag_bar[prev], uses & 1u);
            }
            ++lag_round;
            return;
        }
        if ((MODE & kV2SyncTopOnly) && point != 0) return;
        if ((MODE & kV2SyncTopHybrid) && point == 2) return;
        asm volatile("bar.sync 1, %0;" ::"n"(NW * 32) : "memory");
    };
    WarpSmem& ws = sm.w[warp];
    const Mp3Tables* __restrict__ tab = a.tab;
    const Ops o{};

    if (lane == 0) {
        mbar_init(&ws.bar, 1);
        if (LOCK && (MODE & kV2Lagged) && warp == 0)
            for (int i = 0; i < 3; ++i) mbar_init(&sm.lag_bar[i], NW);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();

    // share s -> (warp s / grid, CTA s % grid): a small batch spreads over the SMs before it stacks warps on one
    const int share = warp * (int)gridDim.x + (int)blockIdx.x;
    int t_begin = 0, t_end = 0;
    if (share < a.n_shares) {
        t_begin = (int)a.first[share];
        t_end = (int)a.first[share + 1];
    }

    // One lane: TMA bulk copies of granule (t, k): 4608 B of spectra + 128 B of descriptors.  // PHASE: tma+mbarrier
    auto issue = [&](const Mp3Tile& t, int k, int ubuf) {
        const size_t slot = granule_slot(t, k);
        mbar_expect_tx(&ws.bar, 4608u + 128u);
        tma_bulk_g2s(ws.spec, a.spectra + slot * 1152, 4608u, &ws.bar);
        tma_bulk_g2s(ws.units[ubuf], a.units + slot * 2, 128u, &ws.bar);
    };

    int my_iters = 0;
    if (LOCK) {
        for (int i = t_begin; i < t_end; ++i) {
            const Mp3Tile t = ld_tile(a.tiles + i);
            my_iters += (int)t.n_granules - tile_first_k(t);
        }
        if (threadIdx.x == 0) sm.max_iters = 0;
        __syncthreads();
        if (lane == 0) atomicMax(&sm.max_iters, my_iters);
        __syncthreads();
    }

    if (t_begin < t_end) {
        int ti = t_begin, k;
        {
            const Mp3Tile t0 = ld_tile(a.tiles + ti);
            k = tile_first_k(t0);
            if (lane == 0) issue(t0, k, 0);
        }

        f2 sec[18]; // windowed second half of the previous granule's IMDCT = this granule's overlap (not yet inverted)
#pragma unroll
        for (int i = 0; i < 18; ++i) sec[i] = make_float2(0.0f, 0.0f);
        uint32_t phase = 0; // bit 0: parity of the stage (mbarrier phase, descriptor buffer); bit 1: XT region in flight

        for (;;) {  // PHASE: prologue+tile loop
            const Mp3Tile tile = ld_tile(a.tiles + ti);
            const int n_ch = tile.n_ch;
            const int ubuf = (int)(phase & 1u);
            const int region = (int)((phase >> 1) & 1u);
            const bool last_of_tile = k + 1 >= (int)tile.n_granules;
            const bool has_next = !last_of_tile || ti + 1 < (int)__ldg(a.first + share + 1);
            const uint32_t xt_base = smem_u32(ws.xt);
            const uint32_t cur_rows = xt_base + (uint32_t)(18 * region) * kRowBytes;
            const uint32_t prev_rows = xt_base + (uint32_t)(18 * (region ^ 1)) * kRowBytes;

            // A run's first granule takes overlap + polyphase history from the stream state (generation gen).
            if (k == 0 && (tile.flags & kTileLoadState)) {
                const uint32_t gen = __ldg(a.gen + tile.stream); // bumped only by the launch epilogue
                const Mp3StreamState* st = a.states + (size_t)tile.stream * 2 + (gen & 1);
                // overlap[ch][sub-band][18]: fetched with coalesced 16-byte loads into the (still unused) region of the granule in
                // flight, then read per lane -- a lane's own 18 values lie 72 bytes apart from its neighbour's
                {
                    float* scr = reinterpret_cast<float*>(ws.xt) + (size_t)(18 * region) * kPitch * 2;
                    const float4* src = reinterpret_cast<const float4*>(&st->overlap[0][0][0]);
#pragma unroll
                    for (int i = 0; i < 9; ++i) reinterpret_cast<float4*>(scr)[lane + 32 * i] = __ldg(src + lane + 32 * i);
                    __syncwarp();
#pragma unroll
                    for (int t = 0; t < 18; ++t) sec[t] = make_float2(scr[18 * lane + t], scr[576 + 18 * lane + t]);
                    __syncwarp();
                }
                for (int idx = lane; idx < 15 * kPitch; idx += 32) {
                    const int srow = idx / kPitch, col = idx - srow * kPitch;
                    f2 v = make_float2(0.0f, 0.0f);
                    if (col < 32) v = st->dhist[srow][col];
                    sts64(prev_rows + (uint32_t)((3 + srow) * kPitch + col) * 8u, v);
                }
            }

            phase_sync();
            mbar_wait(&ws.bar, phase & 1u);
            const symgpu_mp3_gc& g0 = ws.units[ubuf][0];
            const symgpu_mp3_gc& g1 = ws.units[ubuf][1];
            const float* S = ws.spec;
            if (lane < 10) reinterpret_cast<uint32_t*>(ws.smode)[lane] = 0;
            if (lane >= 16 && lane < 26) reinterpret_cast<uint32_t*>(ws.nz)[lane - 16] = 0;
            const int sr = g0.sample_rate_idx;
            const int kind0 = kind_of(g0), kind1 = (n_ch == 2) ? kind_of(g1) : kind0;
            const bool ms = (n_ch == 2) && (g0.flags & SYMGPU_MP3_F_MID_SIDE);
            const bool is = (n_ch == 2) && (g0.flags & SYMGPU_MP3_F_INTENSITY);
            const int rz0 = g0.rzero, rz1 = (n_ch == 2) ? g1.rzero : 0;

            // A1: per-interval requantisation scale (requantize.rs:240-355)  // PHASE: A1 scale
            for (int ch = 0; ch < n_ch; ++ch) {
                const symgpu_mp3_gc& gg = ws.units[ubuf][ch];
                const int kind = ch ? kind1 : kind0;
                const int n_iv = c2.n_edges[sr][kind] - 1;
                const int gain = (int)gg.global_gain - 210;
                const int shift = (gg.flags & SYMGPU_MP3_F_SCALEFAC_SCALE) ? 2 : 1;
                const int sw = c2.mixed_switch[sr];
                for (int idx = lane; idx < 40; idx += 32) {
                    float s = 1.0f;
                    if (idx < n_iv) {
                        int e = 0;
                        bool scaled = true;
                        const bool long_part = (kind == kKindLong) || (kind == kKindMixed && idx < sw - 1);
                        if (long_part) {
                            const int pre = (gg.flags & SYMGPU_MP3_F_PREFLAG) ? c2.pre_emphasis[idx] : 0;
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

            // A2: my 18 lines of each channel, requantised, as (ch0, ch1) pairs.  The short-block reorder  // PHASE: A2 requant+reorder
            // (hybrid_synthesis.rs:153-215) is a permutation applied AFTER the element-wise requantise and stereo
            // steps, so it is folded into the load: line d of the sub-band comes from source line s, and every
            // per-line decision below is taken on s.
            f2 x[18];
#pragma unroll
            for (int i = 0; i < 18; ++i) x[i] = make_float2(0.0f, 0.0f);
            uint32_t ivq[5] = {0u, 0u, 0u, 0u, 0u}; // interval of the source line behind my i-th channel-1 value, 4 per word
            // stereo.rs:550-553 sets both rzero to max(rzero) before reorder / antialias / hybrid see them
            const int rz_joint = max(rz0, rz1);
            const int rze[2] = {(ms || is) ? rz_joint : rz0, (ms || is) ? rz_joint : rz1};
            int rzr[2] = {rze[0], rze[1]}; // rzero after the reorder step
            if constexpr ((MODE & kV2Compact) != 0) {
                // one copy of the load code: channel 1 first into .x, moved to .y when channel 0 follows
#pragma unroll 1
                for (int pass = 0; pass < 2; ++pass) {
                    const int ch = 1 - pass;
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        x[i].y = x[i].x;
                        x[i].x = 0.0f;
                    }
                    if (ch >= n_ch) continue;
                    const int kind = ch ? kind1 : kind0;
                    const float* Sc = S + ch * 576;
                    const float* scl = ws.scale[ch];
                    const bool track = is && ch == 1;
                    if (kind == kKindLong) {
                        const uint16_t* iv2 = reinterpret_cast<const uint16_t*>(tab->iv_of_line[sr][kind] + 18 * lane);
#pragma unroll
                        for (int i = 0; i < 18; i += 2) {
                            const float2 v = *reinterpret_cast<const float2*>(Sc + 18 * lane + i);
                            const unsigned ivp = __ldg(iv2 + (i >> 1));
                            const float xa = v.x * scl[ivp & 0xff];
                            const float xb = v.y * scl[ivp >> 8];
                            x[i].x = xa;
                            x[i + 1].x = xb;
                            if (track) {
                                ivq[i >> 2] |= ivp << (8 * (i & 3));
                                if (xa != 0.0f) ws.nz[ivp & 0xff] = 1;
                                if (xb != 0.0f) ws.nz[ivp >> 8] = 1;
                            }
                        }
                    } else {
                        const int m = (kind == kKindMixed) ? 1 : 0;
                        const int sw = m ? c2.mixed_switch[sr] : 0;
                        const uint16_t* e = tab->edges[sr][kind] + sw;
                        const int n_quads = (c2.n_edges[sr][kind] - sw - 1) / 3;
                        const int rz = ch ? rze[1] : rze[0];
                        const bool below = (lane < n_quads) && ((int)e[3 * lane] < rz);
                        const int n_done = __popc(__ballot_sync(0xffffffffu, below)); // reordered quads form a prefix
                        const int start = e[0], i_end = e[3 * n_done];
                        if (ch) rzr[1] = max(rz, i_end); // hybrid_synthesis.rs:213
                        else rzr[0] = max(rz, i_end);
                        const uint32_t* map = tab->short_map[sr][m] + 18 * lane;
#pragma unroll
                        for (int i = 0; i < 18; ++i) {
                            if (i == 6 || i == 12) asm volatile("" ::: "memory");
                            const int d = 18 * lane + i;
                            const uint32_t e3 = __ldg(map + i);
                            const bool moved = d >= start && d < i_end;
                            const int sl = moved ? (int)(e3 & 1023u) : d;
                            const int iv = moved ? (int)((e3 >> 10) & 63u) : (int)((e3 >> 16) & 63u);
                            const float xv = Sc[sl] * scl[iv];
                            x[i].x = xv;
                            if (track) {
                                ivq[i >> 2] |= (uint32_t)iv << (8 * (i & 3));
                                if (xv != 0.0f) ws.nz[iv] = 1;
                            }
                        }
                    }
                }
            } else {
    #pragma unroll
                for (int ch = 0; ch < 2; ++ch) {
                    if (ch >= n_ch) continue;
                    const int kind = ch ? kind1 : kind0;
                    const float* Sc = S + ch * 576;
                    if (kind == kKindLong) {
                        const uint16_t* iv2 = reinterpret_cast<const uint16_t*>(tab->iv_of_line[sr][kind] + 18 * lane);
    #pragma unroll
                        for (int i = 0; i < 18; i += 2) {
                            const float2 v = *reinterpret_cast<const float2*>(Sc + 18 * lane + i);
                            const unsigned ivp = __ldg(iv2 + (i >> 1));
                            // lines at or beyond rzero are +0.0 by contract (requantize.rs:234): 0 * scale = 0
                            const float xa = v.x * ws.scale[ch][ivp & 0xff];
                            const float xb = v.y * ws.scale[ch][ivp >> 8];
                            if (ch == 0) {
                                x[i].x = xa;
                                x[i + 1].x = xb;
                            } else {
                                x[i].y = xa;
                                x[i + 1].y = xb;
                                ivq[i >> 2] |= ivp << (8 * (i & 3)); // i is even: the pair lands in one word
                                if (is) {
                                    if (xa != 0.0f) ws.nz[ivp & 0xff] = 1;
                                    if (xb != 0.0f) ws.nz[ivp >> 8] = 1;
                                }
                            }
                        }
                    } else {
                        const int m = (kind == kKindMixed) ? 1 : 0;
                        const int sw = m ? c2.mixed_switch[sr] : 0;
                        const uint16_t* e = tab->edges[sr][kind] + sw;
                        const int n_quads = (c2.n_edges[sr][kind] - sw - 1) / 3;
                        const int rz = rze[ch];
                        const bool below = (lane < n_quads) && ((int)e[3 * lane] < rz);
                        const int n_done = __popc(__ballot_sync(0xffffffffu, below)); // reordered quads form a prefix
                        const int start = e[0], i_end = e[3 * n_done];
                        rzr[ch] = max(rz, i_end); // hybrid_synthesis.rs:213
                        const uint32_t* map = tab->short_map[sr][m] + 18 * lane;
    #pragma unroll
                        for (int i = 0; i < 18; ++i) {
                            if (i == 6 || i == 12) asm volatile("" ::: "memory"); // keep the 18 lookups from being hoisted together
                            const int d = 18 * lane + i;
                            const uint32_t e3 = __ldg(map + i);
                            const bool moved = d >= start && d < i_end;
                            const int s = moved ? (int)(e3 & 1023u) : d;
                            const int iv = moved ? (int)((e3 >> 10) & 63u) : (int)((e3 >> 16) & 63u);
                            const float xv = Sc[s] * ws.scale[ch][iv];
                            if (ch == 0) {
                                x[i].x = xv;
                            } else {
                                x[i].y = xv;
                                ivq[i >> 2] |= (uint32_t)iv << (8 * (i & 3));
                                if (is && xv != 0.0f) ws.nz[iv] = 1;
                            }
                        }
                    }
                }
            }
            __syncwarp();
            // The stage is free: fetch the next granule while this one runs through its phases.
            if (has_next && lane == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                if (!last_of_tile) {
                    issue(tile, k + 1, ubuf ^ 1);
                } else {
                    const Mp3Tile tn = ld_tile(a.tiles + ti + 1);
                    issue(tn, tile_first_k(tn), ubuf ^ 1);
                }
            }

            // A3/A4: joint stereo (stereo.rs:485-556), decided per SOURCE line  // PHASE: A3 stereo
            if (ms || is) {
                if (is) {
                    // Warp-parallel restatement of the two top-down scans (stereo.rs:198-261, :265-482).
                    const bool mpeg1 = g1.flags & SYMGPU_MP3_F_MPEG1;
                    const int inv_pos = mpeg1 ? 7 : 31;
                    const float(*rt)[2] = mpeg1 ? tab->is_mpeg1 : tab->is_mpeg2[(g1.flags & SYMGPU_MP3_F_SFC_LSB) ? 1 : 0];
                    const uint16_t* e = tab->edges[sr][kind1];
                    const int n_e = c2.n_edges[sr][kind1];
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
                        const int sw = (kind1 == kKindMixed) ? c2.mixed_switch[sr] : 0;
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
                                const int sw = (kind1 == kKindMixed) ? c2.mixed_switch[sr] : 0;
                                if (iv < sw) coded = true;
                                else {
                                    const int w = (iv - sw) % 3;
                                    coded = iv >= (w == 0 ? first_is0 : w == 1 ? first_is1 : first_is2);
                                }
                            }
                            if (coded) {
                                const int kk = (kind1 == kKindLong) ? (iv == 21 ? 20 : iv) : (iv < 36 ? iv : iv - 3);
                                const int pos = g1.scalefacs[kk];
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
                        const float l = x[i].x, r = x[i].y;
                        if (mode == 2) {
                            const float2 ratio = ws.sratio[iv];
                            x[i].x = ratio.x * l;
                            x[i].y = ratio.y * l;
                        } else if (mode == 1) { // process_mid_side, stereo.rs:143-152
                            x[i].x = (l + r) * kFrac1Sqrt2;
                            x[i].y = (l - r) * kFrac1Sqrt2;
                        }
                    }
                } else {
                    // Mid-side only: every line below max(rzero); the lines above are +0.0 in both channels and
                    // (0 + 0) * c = (0 - 0) * c = +0.0, so the bound needs no test.
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        const float l = x[i].x, r = x[i].y;
                        x[i] = o.mul(make_float2(l + r, l - r), kFrac1Sqrt2);
                    }
                }
            }

            // A6: antialias (hybrid_synthesis.rs:218-277) across neighbouring lanes  // PHASE: A6 antialias
            int rzh[2] = {rzr[0], rzr[1]}; // rzero seen by hybrid_synthesis
            bool bot[2] = {false, false}, top[2] = {false, false};
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                const int kind = ch ? kind1 : kind0;
                if (ch >= n_ch || kind == kKindShort) continue; // (warp-uniform)
                const int sb_limit = (kind == kKindMixed) ? 2 : 32;
                const int rz = 18 * min(min(sb_limit, rzr[ch] / 18 + 2), 32);
                rzh[ch] = rz;
                bot[ch] = lane >= 1 && 18 * lane < rz;
                top[ch] = lane < 31 && 18 * (lane + 1) < rz;
            }
            {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const f2 up = x[i], lo = x[17 - i];
                    f2 nb_lo, nb_up; // lower[li] of the boundary below me, upper[ui] of the boundary above me
                    nb_lo.x = __shfl_up_sync(0xffffffffu, lo.x, 1);
                    nb_lo.y = __shfl_up_sync(0xffffffffu, lo.y, 1);
                    nb_up.x = __shfl_down_sync(0xffffffffu, up.x, 1);
                    nb_up.y = __shfl_down_sync(0xffffffffu, up.y, 1);
                    const f2 r_up = o.add(o.mul(up, c2.cs[i]), o.mul(nb_lo, c2.ca[i])); // samples[ui]
                    const f2 r_lo = o.sub(o.mul(lo, c2.cs[i]), o.mul(nb_up, c2.ca[i])); // samples[li]
                    x[i].x = bot[0] ? r_up.x : up.x;
                    x[i].y = bot[1] ? r_up.y : up.y;
                    x[17 - i].x = top[0] ? r_lo.x : lo.x;
                    x[17 - i].y = top[1] ? r_lo.y : lo.y;
                }
            }

            // B: hybrid synthesis (hybrid_synthesis.rs:280-359).  Per channel a sub-band is long (IMDCT-36),  // PHASE: B glue
            // short (3 x IMDCT-12) or beyond the coded lines (samples = overlap, overlap = 0).
            int cat[2] = {0, 0}; // 36, 12 or 0
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                if (ch >= n_ch) continue;
                const int kind = ch ? kind1 : kind0;
                const int sb_limit = (rzh[ch] + 17) / 18;
                const int sb_split = (kind == kKindShort) ? 0 : (kind == kKindMixed) ? 2 : 32;
                const int long_end = min(sb_split, sb_limit);
                cat[ch] = lane < long_end ? 36 : lane < sb_limit ? 12 : 0;
            }
            f2 first[18], nsec[18];
            const int wsel0 = g0.block_type == SYMGPU_MP3_START ? 1 : g0.block_type == SYMGPU_MP3_END ? 3 : 0;
            const int wsel1 = (n_ch == 2) ? (g1.block_type == SYMGPU_MP3_START ? 1 : g1.block_type == SYMGPU_MP3_END ? 3 : 0) : 0;
            if (cat[0] != 12 && cat[1] != 12) {
                if (cat[0] == 36 || cat[1] == 36) {
                    imdct36(o, x, wsel0, wsel1, first, nsec);
                } else {
#pragma unroll
                    for (int i = 0; i < 18; ++i) {
                        first[i] = make_float2(-0.0f, -0.0f);
                        nsec[i] = make_float2(0.0f, 0.0f);
                    }
                }
            } else if (cat[0] != 36 && cat[1] != 36) {
                imdct12x3(o, x, first, nsec);
            } else {
                f2 lx[18], lf[18], ls[18];
#pragma unroll
                for (int i = 0; i < 18; ++i) lx[i] = x[i];
                hybrid_mixed(lx, wsel0, wsel1, cat[0], cat[1], lf, ls);
#pragma unroll
                for (int i = 0; i < 18; ++i) {
                    first[i] = lf[i];
                    nsec[i] = ls[i];
                }
            }
            // A channel beyond its coded lines: samples = overlap (overlap + (-0.0) == overlap bit for bit), overlap = 0
            if ((cat[0] == 0) != (cat[1] == 0)) {
#pragma unroll
                for (int i = 0; i < 18; ++i) {
                    if (cat[0] == 0) {
                        first[i].x = -0.0f;
                        nsec[i].x = 0.0f;
                    } else {
                        first[i].y = -0.0f;
                        nsec[i].y = 0.0f;
                    }
                }
            }
            // samples = overlap + first, frequency inversion (hybrid_synthesis.rs:458-485: odd sample of odd
            // sub-band), transposed into XT[t][sub-band].  The first halo granule only hands its overlap on.
            if (k >= -1) {  // PHASE: B store
                const float sgn = (lane & 1) ? -1.0f : 1.0f;
                const uint32_t dst = cur_rows + (uint32_t)lane * 8u;
#pragma unroll
                for (int t = 0; t < 18; ++t) {
                    f2 v = o.add(first[t], sec[t]);
                    if (t & 1) v = o.mul(v, sgn);
                    sts64(dst + (uint32_t)t * kRowBytes, v);
                }
            }
#pragma unroll
            for (int t = 0; t < 18; ++t) sec[t] = nsec[t];
            __syncwarp();
            phase_sync(1);

            if (k >= -1) {
                // C: DCT-32 of the granule's 18 time slots, in place; lane = slot, both channels packed.  // PHASE: C glue
                if (lane < 18) {
                    const uint32_t rowp = cur_rows + (uint32_t)lane * kRowBytes;
                    f2 v[32], y[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) v[i] = lds64(rowp + 8u * i);
                    lee_dct<32>(o, v, y);
#pragma unroll
                    for (int i = 0; i < 32; ++i) sts64(rowp + 8u * i, y[i]);
                    sts64(rowp + 8u * 32, make_float2(0.0f, 0.0f)); // column 32: V[16] = 0.0 (synthesis.rs:263)
                }
                __syncwarp();
            }

            phase_sync(2);
            if (k >= 0) {
                // D: polyphase window (synthesis.rs:247-263, :309-327).  lane = PCM sample index i; a 16-deep  // PHASE: D window
                // register window of (V_lo[i], V_hi[i]) for both channels walks the 18 slots:
                //   V_lo[i] =  d[16+i] (i<16) | 0 (i=16, the constant column 32) | -d[48-i] (i>16)
                //   V_hi[i] = -d[16-i] (i<=16) | -d[i-16] (i>16)
                //   o[i] = sum_j  V_lo(t-2j)[i] * D[64j+i]  then  + V_hi(t-2j-1)[i] * D[64j+32+i]
                // The signs are folded into the per-lane coefficients ((-d)*D == d*(-D) exactly).
                const int col_lo = lane < 16 ? 16 + lane : (lane == 16 ? 32 : 48 - lane);
                const int col_hi = lane <= 16 ? 16 - lane : lane - 16;
                float dlo[8], dhi[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float a0 = __ldg(tab->synth_d + 64 * j + lane);
                    dlo[j] = lane > 16 ? -a0 : a0;
                    dhi[j] = -__ldg(tab->synth_d + 64 * j + 32 + lane);
                }
                // V values of slots -15 .. 17 at index slot + 15: all indices are compile-time, a value lives in a register
                // from its load to its last tap.  WG slots are accumulated side by side (independent chains): a single
                // chain of 16 dependent sums leaves the FMA pipe idle for most of its latency.
                constexpr int WG = (MODE & kV2WinGroup3) ? 3 : (MODE & kV2WinGroup2) ? 2 : 1;
                const Mp3Tile tw = ld_tile(a.tiles + ti);
                const int lin = (tw.gpf == 2) ? (int)tw.first_frame * 2 + tw.first_gr + k : ((int)tw.first_frame + tw.first_gr + k) * 2;
                float* out = a.pcm + (size_t)(lin >> 1) * SYMGPU_MP3_FRAME_FLOATS + (lin & 1) * 576 + lane;
                const bool stereo = tw.n_ch == 2;
                if constexpr ((MODE & kV2Compact) != 0) {
                    // two passes of 9 slots over one copy of the code; the 15 newest V values move down in between
                    f2 wl[24], wh[24];
                    {
                        const uint32_t h_lo = prev_rows + (uint32_t)(3 * kPitch + col_lo) * 8u;
                        const uint32_t h_hi = prev_rows + (uint32_t)(3 * kPitch + col_hi) * 8u;
#pragma unroll
                        for (int m = 0; m < 15; ++m) {
                            wl[m] = lds64(h_lo + m * kRowBytes);
                            wh[m] = lds64(h_hi + m * kRowBytes);
                        }
                    }
                    uint32_t a_lo = cur_rows + (uint32_t)col_lo * 8u;
                    uint32_t a_hi = cur_rows + (uint32_t)col_hi * 8u;
#pragma unroll 1
                    for (int half = 0; half < 2; ++half) {
#pragma unroll
                        for (int g0 = 0; g0 < 9; g0 += 3) {
                            f2 acc[3];
#pragma unroll
                            for (int q = 0; q < 3; ++q) {
                                wl[15 + g0 + q] = lds64(a_lo + (g0 + q) * kRowBytes);
                                wh[15 + g0 + q] = lds64(a_hi + (g0 + q) * kRowBytes);
                                acc[q] = make_float2(0.0f, 0.0f);
                            }
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
#pragma unroll
                                for (int q = 0; q < 3; ++q) acc[q] = o.add(o.mul(wl[15 + g0 + q - 2 * j], dlo[j]), acc[q]);
#pragma unroll
                                for (int q = 0; q < 3; ++q) acc[q] = o.add(o.mul(wh[15 + g0 + q - 2 * j - 1], dhi[j]), acc[q]);
                            }
#pragma unroll
                            for (int q = 0; q < 3; ++q) {
                                out[(g0 + q) * 32] = acc[q].x;
                                if (stereo) out[1152 + (g0 + q) * 32] = acc[q].y;
                            }
                        }
#pragma unroll
                        for (int e = 0; e < 15; ++e) {
                            wl[e] = wl[e + 9];
                            wh[e] = wh[e + 9];
                        }
                        a_lo += 9 * kRowBytes;
                        a_hi += 9 * kRowBytes;
                        out += 9 * 32;
                    }
                } else {
                    f2 wl[33], wh[33];
                    {
                        const uint32_t h_lo = prev_rows + (uint32_t)(3 * kPitch + col_lo) * 8u;
                        const uint32_t h_hi = prev_rows + (uint32_t)(3 * kPitch + col_hi) * 8u;
    #pragma unroll
                        for (int m = 0; m < 15; ++m) { // the 15 slots before slot 0
                            wl[m] = lds64(h_lo + m * kRowBytes);
                            wh[m] = lds64(h_hi + m * kRowBytes);
                        }
                    }
                    const uint32_t a_lo = cur_rows + (uint32_t)col_lo * 8u;
                    const uint32_t a_hi = cur_rows + (uint32_t)col_hi * 8u;
    #pragma unroll
                    for (int g0 = 0; g0 < 18; g0 += WG) {
                        f2 acc[WG];
    #pragma unroll
                        for (int q = 0; q < WG; ++q) {
                            wl[15 + g0 + q] = lds64(a_lo + (g0 + q) * kRowBytes);
                            wh[15 + g0 + q] = lds64(a_hi + (g0 + q) * kRowBytes);
                            acc[q] = make_float2(0.0f, 0.0f);
                        }
    #pragma unroll
                        for (int j = 0; j < 8; ++j) {
    #pragma unroll
                            for (int q = 0; q < WG; ++q) {
                                const f2 p0 = o.mul(wl[15 + g0 + q - 2 * j], dlo[j]);
                                if (MODE & kV2WinScalarAdd) {
                                    acc[q].x += p0.x;
                                    acc[q].y += p0.y;
                                } else {
                                    acc[q] = o.add(p0, acc[q]);
                                }
                            }
    #pragma unroll
                            for (int q = 0; q < WG; ++q) {
                                const f2 p1 = o.mul(wh[15 + g0 + q - 2 * j - 1], dhi[j]);
                                if (MODE & kV2WinScalarAdd) {
                                    acc[q].x += p1.x;
                                    acc[q].y += p1.y;
                                } else {
                                    acc[q] = o.add(p1, acc[q]);
                                }
                            }
                        }
    #pragma unroll
                        for (int q = 0; q < WG; ++q) {
                            out[(g0 + q) * 32] = acc[q].x;
                            if (stereo) out[1152 + (g0 + q) * 32] = acc[q].y;
                        }
                    }
            
                }
            }

            // A tile that ends its run publishes overlap + the last 15 DCT vectors to generation gen + 1.
            {  // PHASE: D glue+epilogue
                const Mp3Tile te = ld_tile(a.tiles + ti);
                const bool last = k + 1 >= (int)te.n_granules;
                if (last && (te.flags & kTileStoreState)) {
                    const uint32_t gen = __ldg(a.gen + te.stream);
                    Mp3StreamState* st = a.states + (size_t)te.stream * 2 + ((gen + 1) & 1);
                    for (int idx = lane; idx < 15 * 32; idx += 32) {
                        const int srow = idx >> 5, col = idx & 31;
                        st->dhist[srow][col] = lds64(cur_rows + (uint32_t)((3 + srow) * kPitch + col) * 8u);
                    }
                    // overlap: through the region of the granule before (its last reader, the window phase, is done), so that
                    // the stores to HBM are coalesced 16-byte ones
                    {
                        __syncwarp();
                        float* scr = reinterpret_cast<float*>(ws.xt) + (size_t)(18 * (region ^ 1)) * kPitch * 2;
#pragma unroll
                        for (int t = 0; t < 18; ++t) {
                            scr[18 * lane + t] = sec[t].x;
                            scr[576 + 18 * lane + t] = te.n_ch == 2 ? sec[t].y : 0.0f;
                        }
                        __syncwarp();
                        float4* dst = reinterpret_cast<float4*>(&st->overlap[0][0][0]);
#pragma unroll
                        for (int i = 0; i < 9; ++i) dst[lane + 32 * i] = reinterpret_cast<const float4*>(scr)[lane + 32 * i];
                    }
                }
                if (last && ti + 1 >= (int)__ldg(a.first + share + 1)) break;
                __syncwarp(); // the window's reads of the previous region are done before the next granule overwrites it
                phase ^= (k >= -1) ? 3u : 1u;
                if (!last) {
                    ++k;
                } else {
                    ++ti;
                    const Mp3Tile tn = ld_tile(a.tiles + ti);
                    k = tile_first_k(tn);
                    if (!(tn.flags & kTileCarryIn)) {
                        // a new run: nothing carries over (its state comes from HBM at k == 0)
#pragma unroll
                        for (int i = 0; i < 18; ++i) sec[i] = make_float2(0.0f, 0.0f);
                    }
                }
            }
        }
    }

    if (LOCK) {
        for (int i = my_iters; i < sm.max_iters; ++i) {
            phase_sync(0);
            phase_sync(1);
            phase_sync(2);
        }
    }

    // Launch epilogue: the last CTA to retire publishes the new state generation of every run.
    __syncthreads();
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

namespace {
struct V2Variant {
    int nw, mode;
    void (*kernel)(Mp3V2Args);
    size_t smem;
};
#define V2_VARIANT(NW, MODE) {NW, MODE, mp3v2_synth_kernel<NW, MODE>, sizeof(Mp3V2Smem<NW>)}
// The first entry is the default: 12 warps in lockstep at the top of a granule and after the hybrid phase.
const V2Variant kV2Variants[] = {V2_VARIANT(kMp3V2Warps, 33), V2_VARIANT(kMp3V2Warps, 0),  V2_VARIANT(kMp3V2Warps, 1),
                                 V2_VARIANT(kMp3V2Warps, 5),  V2_VARIANT(kMp3V2Warps, 17), V2_VARIANT(kMp3V2Warps, 81),
                                 V2_VARIANT(kMp3V2Warps, 64), V2_VARIANT(14, 33),          V2_VARIANT(14, 97),
                                 V2_VARIANT(10, 33),          V2_VARIANT(kMp3V2Warps, 129), V2_VARIANT(kMp3V2Warps, 193)};
int g_v2_variant = 0;
} // namespace

// Selects the kernel instantiation (process-wide; experiments): warps per CTA and variant bits.  False if not built.
bool mp3v2_set_variant(int nw, int mode) {
    for (size_t i = 0; i < sizeof kV2Variants / sizeof kV2Variants[0]; ++i)
        if (kV2Variants[i].nw == nw && kV2Variants[i].mode == mode) {
            g_v2_variant = (int)i;
            return true;
        }
    return false;
}

int mp3v2_cta_warps() { return kV2Variants[g_v2_variant].nw; }
// Resident CTAs per SM: small CTAs are stacked so that an SM always runs 12 warps (168 registers each).
int mp3v2_ctas_per_sm() { return kV2Variants[g_v2_variant].nw <= 6 ? 12 / kV2Variants[g_v2_variant].nw : 1; }

namespace {
// Raises the dynamic shared-memory limit of variant `vi` on the current device once.
cudaError_t configure_variant(int vi, int dev) {
    static bool done[64][sizeof kV2Variants / sizeof kV2Variants[0]] = {};
    if (done[dev & 63][vi]) return cudaSuccess;
    const V2Variant& v = kV2Variants[vi];
    cudaError_t e = cudaFuncSetAttribute(v.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)v.smem);
    if (e == cudaSuccess) done[dev & 63][vi] = true;
    return e;
}
int variant_index(int nw, int mode) {
    for (size_t i = 0; i < sizeof kV2Variants / sizeof kV2Variants[0]; ++i)
        if (kV2Variants[i].nw == nw && kV2Variants[i].mode == mode) return (int)i;
    return -1;
}
} // namespace

int mp3v2_sm_count(cudaError_t* err) {
    static int sm_for_device[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess && !sm_for_device[dev & 63]) {
        int n_sm = 0;
        e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
        if (e == cudaSuccess) sm_for_device[dev & 63] = n_sm;
    }
    if (err) *err = e;
    return e == cudaSuccess ? sm_for_device[dev & 63] : 0;
}

// short_runs: the plan is made of many short runs (the serving shape: a frame or two per stream).  Unless an experiment
// pinned a variant, such plans take the compact instantiation that re-aligns its warps once per granule only: with a state
// load and store around almost every granule the phases of different warps differ too much for three meeting points.
cudaError_t mp3v2_launch(const Mp3V2Args& a, int n_ctas, cudaStream_t stream, bool short_runs) {
    cudaError_t e = cudaSuccess;
    const int n_sm = mp3v2_sm_count(&e);
    if (e != cudaSuccess) return e;
    int vi = g_v2_variant;
    if (vi == 0 && short_runs) {
        const int alt = variant_index(kV2Variants[0].nw, kV2Lockstep | kV2SyncTopOnly | kV2Compact);
        if (alt >= 0) vi = alt;
    }
    int dev = 0;
    e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = configure_variant(vi, dev);
    if (e != cudaSuccess) return e;
    const V2Variant& v = kV2Variants[vi];
    if (n_ctas <= 0 || n_ctas > n_sm * mp3v2_ctas_per_sm() || a.n_shares > n_ctas * v.nw) return cudaErrorInvalidConfiguration;
    v.kernel<<<n_ctas, v.nw * 32, v.smem, stream>>>(a);
    return cudaGetLastError();
}

} // namespace symgpu
