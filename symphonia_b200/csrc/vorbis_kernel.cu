// Vorbis synthesis for sm_90a (codec-vorbis/src/lib.rs:250-315):
//   floor-1 curve (floor.rs:568-653, :776-825)  ->  inverse coupling (lib.rs:252-278)
//   -> floor * residue (lib.rs:282-292) -> IMDCT -> power-sine window + overlap-add (dsp.rs:68-145)
//
// The overlap line is overwritten by every packet, never accumulated (dsp.rs:125): what a packet
// overlaps with is the second half of the PREVIOUS packet's IMDCT output.  So a CTA takes a chunk of
// consecutive packets of one stream plus the packet before it, gives every packet its own group of
// 64 threads with its own named barrier (both channels in the group, because the coupling step
// mixes them), runs all the IMDCTs independently, and after one CTA barrier windows / overlap-adds
// every packet against its predecessor's tail.  A run's first chunk takes the tail from the
// (double-buffered) stream state instead.  The number of packet slots adapts to the block size
// (8 slots of 22 KB at blocksize_1 = 2048).
//
// Floor step 1 is an integer recurrence over <= 65 posts, swept level by level of its dependency forest with
// one lane per post; step 2 is evaluated per spectral line in closed form: after d steps of render_line's error accumulator,
//   y(d) = y0 + d*base + sign(dy) * floor(d*ady / adx)
// which is the same integer the reference's loop reaches, so the table lookup is identical.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>

#include "../../include/symgpu.h"
#include "codec_kernels.h"
#include "imdct.cuh"
#include "tables.h"

namespace symgpu {
namespace {

constexpr int kVorbisThreads = 64;

// One segment of the rendered curve: the line from (x0, y0) to the next point.  16 bytes, read as one word group.
struct alignas(16) FloorSeg {
    int x0;
    int16_t y0;
    int16_t base;   // dy / adx, truncated toward zero (floor.rs:790)
    int16_t ady;    // |dy| - |base| * adx
    int16_t adx_s;  // adx, negated when dy < 0
    float inv;      // ~ 1 / adx: seeds the exact integer division below
};

struct alignas(16) FloorPoints { // curve of one channel: seg[0 .. n-2] plus a sentinel; built by one warp
    FloorSeg seg[68];
    int16_t final_y[66]; // step-1 amplitudes
    int n;
};

// floor(a / b) for 0 <= a < 2^24, 1 <= b <= 2^12, exactly: `inv` ~ 1/b seeds an estimate that is off by at
// most one (a and the product are exact or within 2^-20 relative), the two tests make it exact.
__device__ __forceinline__ int div_seeded(int a, int b, float inv) {
    int q = __float2int_rz(__int2float_rn(a) * inv);
    if (q * b > a) --q;
    if ((q + 1) * b <= a) ++q;
    return q;
}

__device__ __forceinline__ int render_point(int x0, int y0, int x1, int y1, int x) { // floor.rs:776-782
    const int dy = y1 - y0;
    const int adx = x1 - x0;
    const int off = div_seeded(abs(dy) * (x - x0), adx, __fdividef(1.0f, (float)adx));
    return dy < 0 ? y0 - off : y0 + off;
}

// Floor synthesis step 1 (floor.rs:568-625), the sort-order walk of step 2 (floor.rs:627-653) and the
// per-segment constants of render_line (floor.rs:785-800), by one warp.
//   Step 1 is a recurrence over the posts, but post i only needs its two neighbours among the EARLIER posts:
//   the posts form a dependency forest whose levels the host computed when the setup was registered
//   (FloorAux.level), so the warp sweeps level by level, one lane per post.
//   step2_flag[i] ends up true iff post i's own value is non-zero or a LATER post with a non-zero value has
//   it as a neighbour (later writes only ever set the flag), which is an OR over lanes.
__device__ __forceinline__ void floor1_build(const symgpu_vorbis_floor1& s, const FloorAux& aux, const uint16_t* __restrict__ fy,
                                             int n_half, FloorPoints& out, int lane) {
    const int count = s.n_posts;
    const int mult = s.multiplier;
    const int range = mult == 1 ? 256 : mult == 2 ? 128 : mult == 3 ? 86 : 64;
    int16_t* final_y = out.final_y;
    // my posts: i = lane, lane + 32, lane + 64  (ordering the posts by level on the host, so that a level touches fewer of the
    // three slots, gains too little to be worth the table)
    int px[3], plo[3], phi[3], pxlo[3], pxhi[3], pval[3], plvl[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = lane + 32 * k;
        px[k] = plo[k] = phi[k] = pxlo[k] = pxhi[k] = pval[k] = 0;
        plvl[k] = 0xff;
        if (i < count) {
            px[k] = s.x_list[i];
            pval[k] = fy[i];
            if (i >= 2) {
                plo[k] = s.low[i];
                phi[k] = s.high[i];
                pxlo[k] = s.x_list[plo[k]];
                pxhi[k] = s.x_list[phi[k]];
                plvl[k] = aux.level[i];
            } else {
                final_y[i] = (int16_t)pval[k];
            }
        }
    }
    __syncwarp();
    // step2 flags: posts 0..63 in a 64-bit mask, post 64 (a setup may hold 65 posts, floor.rs:455-560) on its own
    unsigned long long bits = 0ull;
    bool bit64 = false;
    const int max_level = aux.max_level;
    for (int level = 1; level <= max_level; ++level) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (plvl[k] == level) {
                const int predicted = render_point(pxlo[k], final_y[plo[k]], pxhi[k], final_y[phi[k]], px[k]);
                const int val = pval[k];
                const int highroom = range - predicted, lowroom = predicted;
                int fin = predicted;
                if (val != 0) {
                    const int room = 2 * (highroom < lowroom ? highroom : lowroom);
                    bits |= (1ull << plo[k]) | (1ull << phi[k]); // neighbours are earlier posts: indices <= 63
                    if (lane + 32 * k < 64) bits |= 1ull << (lane + 32 * k);
                    else bit64 = true;
                    if (val >= room) fin = highroom > lowroom ? val - lowroom + predicted : predicted - val + highroom - 1;
                    else fin = (val & 1) ? predicted - ((val + 1) / 2) : predicted + (val / 2);
                }
                final_y[lane + 32 * k] = (int16_t)fin;
            }
        }
        __syncwarp();
    }
    const unsigned f_lo = __reduce_or_sync(0xffffffffu, (unsigned)bits) | 3u; // floor_step2_flag[0] = [1] = true
    const unsigned f_hi = __reduce_or_sync(0xffffffffu, (unsigned)(bits >> 32));
    const unsigned long long flag = ((unsigned long long)f_hi << 32) | f_lo;
    const bool flag64 = __any_sync(0xffffffffu, bit64);

    // points in X order: the flagged posts, amplitudes scaled and clamped (floor.rs:631-648)
    int n = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int r = lane + 32 * k;
        int i = 0;
        bool on = false;
        if (r < count) {
            i = s.sort_order[r];
            on = i < 64 ? (bool)((flag >> i) & 1ull) : flag64;
        }
        const unsigned vote = __ballot_sync(0xffffffffu, on);
        if (on) {
            FloorSeg& g = out.seg[n + __popc(vote & ((1u << lane) - 1u))];
            g.x0 = s.x_list[i];
            g.y0 = (int16_t)min(max((int)final_y[i] * mult, 0), 255);
        }
        n += __popc(vote);
    }
    __syncwarp();
    if (lane == 0) {
        const int hx = out.seg[n - 1].x0, hy = out.seg[n - 1].y0;
        if (hx < n_half) { // render_line(hx, hy, n, hy): a flat tail (floor.rs:650-652)
            out.seg[n].x0 = n_half;
            out.seg[n].y0 = (int16_t)hy;
            out.seg[n + 1].x0 = 0x7fffffff;
        } else {
            out.seg[n].x0 = 0x7fffffff; // sentinel for the segment walk
        }
        out.n = hx < n_half ? n + 1 : n;
    }
    __syncwarp();
    n = out.n;
    // per-segment constants
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int sgi = lane + 32 * k;
        if (sgi + 1 < n) {
            const int x0 = out.seg[sgi].x0, y0 = out.seg[sgi].y0, x1 = out.seg[sgi + 1].x0, y1 = out.seg[sgi + 1].y0;
            const int dy = y1 - y0, adx = x1 - x0;
            const int base = dy / adx;
            out.seg[sgi].base = (int16_t)base;
            out.seg[sgi].ady = (int16_t)(abs(dy) - abs(base) * adx);
            out.seg[sgi].adx_s = (int16_t)(dy < 0 ? -adx : adx);
            out.seg[sgi].inv = __fdividef(1.0f, (float)adx);
        }
    }
    __syncwarp();
}

// Index of line x in a channel's curve buffer (one byte per line: the floor1_inverse_dB_table index): lane l of the rendering warp
// owns the L = n_half / 32 consecutive lines [l * L, (l + 1) * L); four pad bytes per lane-run put the lanes on distinct banks.
__device__ __forceinline__ int ybuf_index(int x, int log2_l) { return log2_l >= 2 ? x + ((x >> log2_l) << 2) : x; }

// Renders the curve (floor.rs:785-825) as table indices: every lane walks ITS run of consecutive lines with render_line's own
// error accumulator -- y += base; err += ady; on err >= adx: err -= adx, y += sign(dy) -- entered in the middle of a segment
// through the closed form  y(d) = y0 + d * base + sign(dy) * floor(d * ady / adx),  err(d) = d * ady mod adx  (one exact
// division per lane instead of one per line).
struct SegList { // what floor1_render reads: the segments and their count (points = segments + 1, a sentinel behind them)
    const FloorSeg* seg;
    int n;
};
__device__ __forceinline__ void floor1_render(const SegList p, int n_half, int lane, uint8_t* ybuf) {
    const int log2_l = 31 - __clz(n_half >> 5);
    const int len = 1 << log2_l;
    int x = lane << log2_l;
    // the segment that holds x: the last one whose x0 <= x (seg[0].x0 = 0; a sentinel ends the list)
    int lo = 0, hi = p.n - 1; // p.n points: segments 0 .. n - 2, the sentinel behind them
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (p.seg[mid].x0 <= x) lo = mid;
        else hi = mid - 1;
    }
    int seg = lo;
    int4 w = *reinterpret_cast<const int4*>(&p.seg[seg]);
    int x1 = p.seg[seg + 1].x0;
    int base = w.y >> 16, ady = (int)(short)(w.z & 0xffff), adx_s = w.z >> 16;
    int adx = abs(adx_s), sgn = adx_s < 0 ? -1 : 1;
    const int d = x - w.x;
    const int carries = ady ? div_seeded(d * ady, adx, __int_as_float(w.w)) : 0;
    int err = d * ady - carries * adx;
    int y = (int)(short)(w.y & 0xffff) + d * base + sgn * carries;
    uint8_t* dst = ybuf + ybuf_index(x, log2_l);
    for (int j = 0; j < len; ++j) {
        dst[j] = (uint8_t)y;
        ++x;
        if (x == x1) { // the next segment starts exactly on its own first point
            ++seg;
            w = *reinterpret_cast<const int4*>(&p.seg[seg]);
            x1 = p.seg[seg + 1].x0;
            base = w.y >> 16, ady = (int)(short)(w.z & 0xffff), adx_s = w.z >> 16;
            adx = abs(adx_s), sgn = adx_s < 0 ? -1 : 1;
            y = (int)(short)(w.y & 0xffff);
            err = 0;
        } else {
            y += base;
            err += ady;
            if (err >= adx) {
                err -= adx;
                y += sgn;
            }
        }
    }
}

template <int LOG2>
__device__ __forceinline__ void imdct_one(const float* spec, float* out, float2* z, const CodecTables* tab, int gt, NamedSync sync) {
    const FftTables* ft = reinterpret_cast<const FftTables*>(tab->fft_lit16);
    const float2* tw = reinterpret_cast<const float2*>(tab->vorbis_tw) + ((1 << LOG2) - 16);
    imdct_blocks<LOG2>(spec, out, z, 1, tw, ft, gt, kVorbisThreads, sync);
}

__device__ void imdct_dispatch(int log2_n2, const float* spec, float* out, float2* z, const CodecTables* tab, int gt,
                               NamedSync sync) {
    switch (log2_n2) { // FFT size = blocksize / 4
        case 4: imdct_one<4>(spec, out, z, tab, gt, sync); break;
        case 5: imdct_one<5>(spec, out, z, tab, gt, sync); break;
        case 6: imdct_one<6>(spec, out, z, tab, gt, sync); break;
        case 7: imdct_one<7>(spec, out, z, tab, gt, sync); break;
        case 8: imdct_one<8>(spec, out, z, tab, gt, sync); break;
        case 9: imdct_one<9>(spec, out, z, tab, gt, sync); break;
        case 10: imdct_one<10>(spec, out, z, tab, gt, sync); break;
        default: imdct_one<11>(spec, out, z, tab, gt, sync); break;
    }
}

// Shared-memory bytes of one packet slot for blocksize_1 / 2 = slot_smem floats per channel:
// out[2][2*slot_smem] (the spectrum of a channel lives in the first half of its `out` until the
// pre-twiddle has consumed it) | z | floor points of both channels.
__host__ __device__ inline size_t vorbis_slot_bytes(int slot_smem) {
    size_t b = sizeof(float) * 4 * (size_t)slot_smem + sizeof(float2) * zpad_len(slot_smem / 2);
    b = (b + 15) & ~(size_t)15; // the floor points are read 16 bytes at a time
    return b + 2 * sizeof(FloorPoints);
}

__global__ void __launch_bounds__(512) vorbis_synth_kernel(VorbisArgs a, int slot_smem) {
    extern __shared__ __align__(16) unsigned char raw[];
    __shared__ bool is_last;
    __shared__ float inv_db_s[256]; // floor1_inverse_dB_table (floor.rs:21-86): 2 K lookups per long packet
    const int tid = threadIdx.x, grp = tid >> 6, gt = tid & 63, warp_in_grp = gt >> 5, lane = tid & 31;
    const size_t slot_bytes = vorbis_slot_bytes(slot_smem);
    auto slot_out = [&](int k, int ch) { return reinterpret_cast<float*>(raw + k * slot_bytes) + (size_t)ch * 2 * slot_smem; };
    float2* z = reinterpret_cast<float2*>(reinterpret_cast<float*>(raw + grp * slot_bytes) + 4 * slot_smem);
    FloorPoints* pts = reinterpret_cast<FloorPoints*>(raw + (grp + 1) * slot_bytes - 2 * sizeof(FloorPoints));

    for (int i = threadIdx.x; i < 256; i += blockDim.x) inv_db_s[i] = a.tab->vorbis_inverse_db[i]; // (a CTA may have fewer than 256 threads)
    __syncthreads();
    const CodecChunk ck = a.chunks[blockIdx.x];
    const symgpu_vorbis_stream cfg = a.streams[ck.stream];
    const CodecTables* __restrict__ tab = a.tab;
    const int bs0 = 1 << cfg.bs0_exp, bs1 = 1 << cfg.bs1_exp;
    const int n_ch = cfg.channels;
    const uint32_t gen = a.gen[ck.stream];
    const float* st_in = a.states + ((size_t)ck.stream * 2 + (gen & 1)) * kVorbisStateFloats;
    float* st_out = a.states + ((size_t)ck.stream * 2 + ((gen + 1) & 1)) * kVorbisStateFloats;
    const bool load_state = ck.flags & kChunkLoadState;
    const int count = ck.count;
    const int half1 = bs1 >> 1;

    // slot 0 = the packet before the chunk (or the stream state), slot k = chunk packet k-1
    const int p = (int)ck.first - 1 + grp;
    const bool have_packet = grp <= count && (grp > 0 || !load_state);
    symgpu_vorbis_unit u = {};
    int bs = bs0;
    if (have_packet) {
        u = a.units[p];
        bs = u.block_flag ? bs1 : bs0;
        const int n2 = bs >> 1;
        NamedSync sync{1 + grp, kVorbisThreads};
        // pull this packet's residue (both channels) towards the SM while the floors are built
        for (uint32_t i = 32u * gt; i < (uint32_t)n_ch * a.slot; i += 32u * kVorbisThreads)
            if ((i % a.slot) < (uint32_t)n2)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(a.residue + ((size_t)p * a.pkt_ch + a.ch_base) * a.slot + i));
        // (1) floor curves: warp = channel.  The curve is kept as one table index per line, in the upper half of the channel's
        //     area (free until the IMDCT writes its output); the look-up happens where the value is used, in (2).
        const int log2_l = 31 - __clz(n2 >> 5);
        bool used[2] = {false, false};
        for (int ch = 0; ch < n_ch; ++ch) used[ch] = u.floor[ch] != 0xffff && u.floor[ch] < a.n_floors;
        if (warp_in_grp < n_ch && used[warp_in_grp]) {
            const int ch = warp_in_grp;
            floor1_build(a.floors[u.floor[ch]], a.floor_aux[u.floor[ch]], a.floor_y + ((size_t)p * a.pkt_ch + a.ch_base + ch) * 65, n2, pts[ch], lane);
            floor1_render(SegList{pts[ch].seg, pts[ch].n}, n2, lane, reinterpret_cast<uint8_t*>(slot_out(grp, ch) + n2));
        }
        sync();
        // (2) inverse coupling + dot product (an unused floor is all zeros: ch.floor[..n2].fill(0.0))
        const float* r0 = a.residue + ((size_t)p * a.pkt_ch + a.ch_base) * a.slot;
        const float* r1 = r0 + a.slot;
        float* spec0 = slot_out(grp, 0);
        float* spec1 = slot_out(grp, 1);
        const uint8_t* yb0 = reinterpret_cast<const uint8_t*>(spec0 + n2);
        const uint8_t* yb1 = reinterpret_cast<const uint8_t*>(spec1 + n2);
        // four lines per thread and trip: the eight residue loads of a trip are issued together (they are L2 hits thanks to the
        // prefetch above, but 16 dependent round trips per packet were 8 % of the kernel's stall samples)
        for (int i0 = gt; i0 < n2; i0 += 4 * kVorbisThreads) {
            float mm[4], aa[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int i = i0 + q * kVorbisThreads;
                mm[q] = i < n2 ? __ldg(r0 + i) : 0.0f;
                aa[q] = (i < n2 && n_ch == 2) ? __ldg(r1 + i) : 0.0f;
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int i = i0 + q * kVorbisThreads;
                if (i >= n2) break;
                float m = mm[q], ang = aa[q];
                if (cfg.coupled && n_ch == 2) { // lib.rs:267-277: comparisons are "> 0.0"
                    float nm, na;
                    if (m > 0.0f) {
                        if (ang > 0.0f) { nm = m; na = m - ang; } else { nm = m + ang; na = m; }
                    } else {
                        if (ang > 0.0f) { nm = m; na = m + ang; } else { nm = m - ang; na = m; }
                    }
                    m = nm;
                    ang = na;
                }
                const int yi = ybuf_index(i, log2_l);
                const float f0 = used[0] ? inv_db_s[yb0[yi]] : 0.0f;
                spec0[i] = u.do_not_decode[0] ? f0 : f0 * m;
                if (n_ch == 2) {
                    const float f1 = used[1] ? inv_db_s[yb1[yi]] : 0.0f;
                    spec1[i] = u.do_not_decode[1] ? f1 : f1 * ang;
                }
            }
        }
        sync();
        // (3) IMDCT per channel, in place over the channel's area (the spectrum is dead after the pre-twiddle)
        for (int ch = 0; ch < n_ch; ++ch) imdct_dispatch(31 - __clz(bs >> 2), slot_out(grp, ch), slot_out(grp, ch), z, tab, gt, sync);
    } else if (grp == 0) {
        // run start: slot 0 holds the overlap line itself, as the tail of a maximum-size block
        for (int i = gt; i < 2 * half1; i += kVorbisThreads) slot_out(0, i / half1)[half1 + (i % half1)] = st_in[i];
    }
    __syncthreads();

    // (4) window + overlap-add against the previous packet's tail (dsp.rs:83-122)
    if (grp >= 1 && grp <= count) {
        const bool block_flag = u.block_flag != 0, prev_flag = u.prev_block_flag != 0;
        const bool prev_is_state = grp == 1 && load_state;
        const int pbs = prev_is_state ? bs1 : (a.units[p - 1].block_flag ? bs1 : bs0); // geometry of slot grp-1's tail
        const int out_len = ((prev_flag ? bs1 : bs0) + bs) >> 2;
        const float* win = tab->vorbis_win + (((block_flag && prev_flag) ? bs1 : bs0) / 2 - 32);
        for (int ch = 0; ch < n_ch; ++ch) {
            const float* out = slot_out(grp, ch);
            const float* ov = slot_out(grp - 1, ch) + pbs / 2; // overlap[..] = imdct[bs/2..bs] of the previous packet
            float* dst = a.pcm + ((size_t)p * a.pkt_ch + a.ch_base + ch) * a.slot;
            if (prev_flag == block_flag) {
                const int len = bs / 2;
                for (int k = gt; k < len; k += kVorbisThreads)
                    dst[k] = ov[k] * __ldg(win + len - 1 - k) + out[k] * __ldg(win + k);
            } else if (prev_flag && !block_flag) {
                const int start = (bs1 - bs0) / 4, len = bs0 / 2;
                for (int k = gt; k < out_len; k += kVorbisThreads) {
                    if (k < start) dst[k] = ov[k];
                    else {
                        const int j = k - start;
                        dst[k] = ov[k] * __ldg(win + len - 1 - j) + out[j] * __ldg(win + j);
                    }
                }
            } else {
                const int start = (bs1 - bs0) / 4, len = bs0 / 2, end = start + len;
                for (int k = gt; k < out_len; k += kVorbisThreads) {
                    if (k < len) dst[k] = ov[k] * __ldg(win + len - 1 - k) + out[start + k] * __ldg(win + k);
                    else dst[k] = out[end + (k - len)];
                }
            }
            if (grp == count && (ck.flags & kChunkStoreState)) // the run's last packet leaves its tail in the state
                for (int k = gt; k < bs / 2; k += kVorbisThreads) st_out[ch * half1 + k] = out[bs / 2 + k];
        }
    }

    __syncthreads();
    if (tid == 0) {
        __threadfence();
        is_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (is_last) {
        for (unsigned i = tid; i < gridDim.x; i += blockDim.x)
            if (a.chunks[i].flags & kChunkStoreState) a.gen[a.chunks[i].stream] += 1;
        if (tid == 0) *a.done = 0;
    }
}


// ---- mbarrier / TMA bulk copy (as in mp3_kernel.cu): the Z kernel pulls its stream's FFT and IMDCT twiddle tables into shared
// memory with three bulk copies issued by one thread at CTA start; every warp waits for them right before its IMDCT, which is
// after its floor curve is built -- no CTA barrier, no exposed latency.
__device__ __forceinline__ uint32_t vz_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void vz_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(vz_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void vz_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(vz_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void vz_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(vz_smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void vz_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(vz_smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(vz_smem_u32(bar))
                 : "memory");
}
// Table area behind the unit slots, in float2: FFT prefix (lit16, lit32, merge tables up to size n2max) | twiddles of the long
// block (n2max) | twiddles of the short block (at most n2max / 2 when the two sizes differ), n2max = slot_smem / 2.
__host__ __device__ inline size_t vorbis_z_tab_bytes(int slot_smem) {
    const int n2max = slot_smem / 2;
    const int fft = n2max >= 64 ? n2max - 8 : 24;
    return sizeof(float2) * (size_t)(fft + n2max + n2max / 2);
}

// =========================================================================================================================
// Z layout (the default): one WARP per (packet, channel).  The IMDCT output is kept as its post-twiddled complex values
// (imdct.cuh: imdct_to_z / imdct_out), floor x residue is formed inside the pre-twiddle straight from global memory, and the
// floor points share the bytes of z (they are dead once the curve is rendered).  A unit then takes 5.8 KB of shared memory at
// blocksize_1 = 2048 instead of 10.5 KB, the kernel runs at 64 registers, and two CTAs of 8 packet slots share an SM: 32 warps
// per SM instead of 16, and no named barrier anywhere -- channels only meet in the inverse coupling, which both warps of a
// packet evaluate from the two residues.
// =========================================================================================================================
__host__ __device__ inline size_t vorbis_unit_z_bytes(int slot_smem) {  // z | floor points | the state tail of slot 0
    size_t b = sizeof(float2) * zpad_len(slot_smem / 2);
    if (b < sizeof(FloorPoints)) b = sizeof(FloorPoints);
    return (b + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t vorbis_unit_bytes(int slot_smem) { // + one table index per line (ybuf_index pads)
    return vorbis_unit_z_bytes(slot_smem) + (((size_t)slot_smem + 128 + 15) & ~(size_t)15);
}

template <int LOG2, typename Pair>
__device__ __forceinline__ void imdct_z_one(Pair pair, float2* z, const FftTables* ft, const float2* tw, int lane) {
    imdct_to_z_from<LOG2>(pair, z, 1, tw, ft, lane, 32, WarpSync{});
}

__global__ void __launch_bounds__(512, 2) vorbis_synth_kernel_z(VorbisArgs a, int slot_smem) {
    extern __shared__ __align__(16) unsigned char raw[];
    __shared__ bool is_last;
    __shared__ float inv_db_s[256]; // floor1_inverse_dB_table (floor.rs:21-86)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int grp = warp >> 1, ch = warp & 1; // packet slot, channel
    const size_t unit_bytes = vorbis_unit_bytes(slot_smem), z_bytes = vorbis_unit_z_bytes(slot_smem);
    auto unit_z = [&](int k, int c) { return reinterpret_cast<float2*>(raw + (size_t)(2 * k + c) * unit_bytes); };
    auto unit_y = [&](int k, int c) { return raw + (size_t)(2 * k + c) * unit_bytes + z_bytes; };

    __shared__ __align__(8) uint64_t tab_bar;
    const CodecChunk ck = a.chunks[blockIdx.x];
    const symgpu_vorbis_stream cfg = a.streams[ck.stream];
    const CodecTables* __restrict__ tab = a.tab;
    const int bs0 = 1 << cfg.bs0_exp, bs1 = 1 << cfg.bs1_exp;
    // the stream's tables: FFT prefix for sizes up to bs1 / 4, IMDCT twiddles of both block sizes
    const int n2max = slot_smem / 2, n2_1 = bs1 >> 2, n2_0 = bs0 >> 2;
    float2* tab_s = reinterpret_cast<float2*>(raw + (size_t)(blockDim.x >> 5) * unit_bytes);
    float2* tw1_s = tab_s + (n2max >= 64 ? n2max - 8 : 24);
    float2* tw0_s = n2_0 == n2_1 ? tw1_s : tw1_s + n2max;
    if (tid == 0) {
        vz_mbar_init(&tab_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t fft_bytes = (uint32_t)sizeof(float2) * (n2_1 >= 64 ? n2_1 - 8 : 24);
        const uint32_t tw1_bytes = (uint32_t)sizeof(float2) * n2_1, tw0_bytes = n2_0 == n2_1 ? 0u : (uint32_t)sizeof(float2) * n2_0;
        vz_mbar_expect_tx(&tab_bar, fft_bytes + tw1_bytes + tw0_bytes);
        vz_bulk_g2s(tab_s, tab->fft_lit16, fft_bytes, &tab_bar);
        vz_bulk_g2s(tw1_s, reinterpret_cast<const float2*>(tab->vorbis_tw) + (n2_1 - 16), tw1_bytes, &tab_bar);
        if (tw0_bytes) vz_bulk_g2s(tw0_s, reinterpret_cast<const float2*>(tab->vorbis_tw) + (n2_0 - 16), tw0_bytes, &tab_bar);
    }
    for (int i = threadIdx.x; i < 256; i += blockDim.x) inv_db_s[i] = a.tab->vorbis_inverse_db[i]; // (a CTA may have fewer than 256 threads)
    __syncthreads(); // also publishes the initialised mbarrier
    const int n_ch = cfg.channels;
    const uint32_t gen = a.gen[ck.stream];
    const float* st_in = a.states + ((size_t)ck.stream * 2 + (gen & 1)) * kVorbisStateFloats;
    float* st_out = a.states + ((size_t)ck.stream * 2 + ((gen + 1) & 1)) * kVorbisStateFloats;
    const bool load_state = ck.flags & kChunkLoadState;
    const int count = ck.count;
    const int half1 = bs1 >> 1;

    // slot 0 = the packet before the chunk (or the stream state), slot k = chunk packet k-1
    const int p = (int)ck.first - 1 + grp;
    const bool have_packet = grp <= count && (grp > 0 || !load_state);
    symgpu_vorbis_unit u = {};
    int bs = bs0;
    if (have_packet && ch < n_ch) {
        u = a.units[p];
        bs = u.block_flag ? bs1 : bs0;
        const int n2 = bs >> 1;
        const float* r0 = a.residue + ((size_t)p * a.pkt_ch + a.ch_base) * a.slot;
        const float* r1 = r0 + a.slot;
        // pull this channel's residue towards the SM while the floor is built (the other channel's warp pulls the other one)
        for (int i = 32 * lane; i < n2; i += 32 * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"((ch ? r1 : r0) + i));
        // (1) floor curve as one table index per line
        const int log2_l = 31 - __clz(n2 >> 5);
        const bool used = u.floor[ch] != 0xffff && u.floor[ch] < a.n_floors;
        const uint8_t* yb = unit_y(grp, ch);
        if (used) {
            // the floor points share the bytes that will hold z
            FloorPoints& pts = *reinterpret_cast<FloorPoints*>(unit_z(grp, ch));
            floor1_build(a.floors[u.floor[ch]], a.floor_aux[u.floor[ch]], a.floor_y + ((size_t)p * a.pkt_ch + a.ch_base + ch) * 65, n2, pts, lane);
            floor1_render(SegList{pts.seg, pts.n}, n2, lane, unit_y(grp, ch));
        }
        __syncwarp();
        // (2) + (3) inverse coupling (lib.rs:267-277: the comparisons are "> 0.0"), floor x residue (an unused floor is all
        //     zeros) and the IMDCT's pre-twiddle in one pass over the lines; then the FFT and the post-twiddle in place
        const bool couple = cfg.coupled && n_ch == 2;
        const bool dnd = u.do_not_decode[ch] != 0;
        auto line = [&](float m, float ang, int i) -> float {
            if (couple) {
                float nm, na;
                if (m > 0.0f) {
                    if (ang > 0.0f) { nm = m; na = m - ang; } else { nm = m + ang; na = m; }
                } else {
                    if (ang > 0.0f) { nm = m; na = m + ang; } else { nm = m - ang; na = m; }
                }
                m = nm;
                ang = na;
            }
            const float f = used ? inv_db_s[yb[ybuf_index(i, log2_l)]] : 0.0f;
            return dnd ? f : f * (ch ? ang : m);
        };
        auto pair = [&](int, int l) -> float2 {
            const float2 m = __ldg(reinterpret_cast<const float2*>(r0 + l));
            const float2 g = n_ch == 2 ? __ldg(reinterpret_cast<const float2*>(r1 + l)) : make_float2(0.0f, 0.0f);
            return make_float2(line(m.x, g.x, l), line(m.y, g.y, l + 1));
        };
        float2* z = unit_z(grp, ch);
        vz_mbar_wait(&tab_bar, 0); // the tables have landed (long ago, as a rule)
        const FftTables* ft = reinterpret_cast<const FftTables*>(tab_s);
        const float2* tw = u.block_flag ? tw1_s : tw0_s;
        switch (31 - __clz(bs >> 2)) { // FFT size = blocksize / 4
            case 4: imdct_z_one<4>(pair, z, ft, tw, lane); break;
            case 5: imdct_z_one<5>(pair, z, ft, tw, lane); break;
            case 6: imdct_z_one<6>(pair, z, ft, tw, lane); break;
            case 7: imdct_z_one<7>(pair, z, ft, tw, lane); break;
            case 8: imdct_z_one<8>(pair, z, ft, tw, lane); break;
            case 9: imdct_z_one<9>(pair, z, ft, tw, lane); break;
            case 10: imdct_z_one<10>(pair, z, ft, tw, lane); break;
            default: imdct_z_one<11>(pair, z, ft, tw, lane); break;
        }
    } else if (grp == 0 && ch < n_ch) {
        // run start: slot 0 holds the overlap line itself (plain floats where a packet would keep z)
        float* zf = reinterpret_cast<float*>(unit_z(0, ch));
        for (int i = lane; i < half1; i += 32) zf[i] = st_in[ch * half1 + i];
    }
    __syncthreads();

    // (4) window + overlap-add against the previous packet's tail (dsp.rs:83-122)
    if (grp >= 1 && grp <= count && ch < n_ch) {
        const bool block_flag = u.block_flag != 0, prev_flag = u.prev_block_flag != 0;
        const bool prev_is_state = grp == 1 && load_state;
        const int pbs = prev_is_state ? bs1 : (a.units[p - 1].block_flag ? bs1 : bs0); // geometry of slot grp-1's tail
        const int out_len = ((prev_flag ? bs1 : bs0) + bs) >> 2;
        const float* win = tab->vorbis_win + (((block_flag && prev_flag) ? bs1 : bs0) / 2 - 32);
        const float2* zc = unit_z(grp, ch);
        const float2* zp = unit_z(grp - 1, ch);
        const int lg = 31 - __clz(bs >> 2), plg = 31 - __clz(pbs >> 2);
        auto out = [&](int j) { return imdct_out_rt(zc, lg, j); };
        // overlap[k] = imdct[pbs/2 + k] of the previous packet, or the state line
        auto ov = [&](int k) { return prev_is_state ? reinterpret_cast<const float*>(zp)[k] : imdct_out_rt(zp, plg, (pbs >> 1) + k); };
        float* dst = a.pcm + ((size_t)p * a.pkt_ch + a.ch_base + ch) * a.slot;
        if (prev_flag == block_flag && !prev_is_state) {
            // two blocks of one size (the common case): straight from the two z arrays, two adjacent samples at a time
            auto win2 = [win](bool, int idx) { return __ldg(reinterpret_cast<const float2*>(win + idx)); };
            overlap_add_equal(zc, zp, lg, win2, dst, lane, 32);
        } else if (prev_flag == block_flag) {
            const int len = bs / 2;
#pragma unroll 4
            for (int k = lane; k < len; k += 32) dst[k] = ov(k) * __ldg(win + len - 1 - k) + out(k) * __ldg(win + k);
        } else if (prev_flag && !block_flag) {
            const int start = (bs1 - bs0) / 4, len = bs0 / 2;
            for (int k = lane; k < out_len; k += 32) {
                if (k < start) dst[k] = ov(k);
                else {
                    const int j = k - start;
                    dst[k] = ov(k) * __ldg(win + len - 1 - j) + out(j) * __ldg(win + j);
                }
            }
        } else {
            const int start = (bs1 - bs0) / 4, len = bs0 / 2, end = start + len;
            for (int k = lane; k < out_len; k += 32) {
                if (k < len) dst[k] = ov(k) * __ldg(win + len - 1 - k) + out(start + k) * __ldg(win + k);
                else dst[k] = out(end + (k - len));
            }
        }
        if (grp == count && (ck.flags & kChunkStoreState)) // the run's last packet leaves its tail in the state
            for (int k = lane; k < bs / 2; k += 32) st_out[ch * half1 + k] = out(bs / 2 + k);
    }

    __syncthreads();
    if (tid == 0) {
        __threadfence();
        is_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (is_last) {
        for (unsigned i = tid; i < gridDim.x; i += blockDim.x)
            if (a.chunks[i].flags & kChunkStoreState) a.gen[a.chunks[i].stream] += 1;
        if (tid == 0) *a.done = 0;
    }
}

} // namespace


// ---- multichannel helpers --------------------------------------------------------------------------------------------
namespace {
// Inverse coupling of every step of the packet's mapping, in the reference's order (lib.rs:252-278: `for coupling in
// mapping.couplings.iter()`), one thread per spectral line: the steps of a line only touch that line.
__global__ void __launch_bounds__(256) vorbis_mc_decouple_kernel(const symgpu_vorbis_unit_mc* __restrict__ units, const uint32_t* __restrict__ stream_of_packet,
                                                                 const symgpu_vorbis_stream_mc* __restrict__ streams, float* residue,
                                                                 uint32_t n_packets, uint32_t channels, uint32_t slot) {
    const uint32_t p = blockIdx.y;
    if (p >= n_packets) return;
    const uint32_t sidx = stream_of_packet[p];
    if (sidx == 0xffffffffu) return; // a packet no run names
    const symgpu_vorbis_stream_mc& cfg = streams[sidx];
    const int n2 = (units[p].block_flag ? (1 << cfg.bs1_exp) : (1 << cfg.bs0_exp)) >> 1;
    float* base = residue + (size_t)p * channels * slot;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
        for (int c = 0; c < cfg.n_couplings; ++c) {
            float* pm = base + (size_t)cfg.magnitude_ch[c] * slot + i;
            float* pa = base + (size_t)cfg.angle_ch[c] * slot + i;
            const float m = *pm, ang = *pa;
            float nm, na;
            if (m > 0.0f) {
                if (ang > 0.0f) { nm = m; na = m - ang; } else { nm = m + ang; na = m; }
            } else {
                if (ang > 0.0f) { nm = m; na = m + ang; } else { nm = m - ang; na = m; }
            }
            *pm = nm;
            *pa = na;
        }
    }
}

__global__ void __launch_bounds__(256) vorbis_mc_split_units_kernel(const symgpu_vorbis_unit_mc* __restrict__ units, uint32_t n_packets, uint32_t pair,
                                                                    symgpu_vorbis_unit* __restrict__ out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_packets) return;
    const symgpu_vorbis_unit_mc u = units[p];
    symgpu_vorbis_unit o{};
    o.block_flag = u.block_flag;
    o.prev_block_flag = u.prev_block_flag;
    for (int c = 0; c < 2; ++c) {
        const uint32_t ch = 2 * pair + c;
        o.do_not_decode[c] = ch < SYMGPU_VORBIS_MAX_CHANNELS ? u.do_not_decode[ch] : 1;
        o.floor[c] = ch < SYMGPU_VORBIS_MAX_CHANNELS ? u.floor[ch] : 0xffff;
    }
    out[p] = o;
}
} // namespace

cudaError_t vorbis_mc_decouple_launch(const symgpu_vorbis_unit_mc* units, const uint32_t* stream_of_packet, const symgpu_vorbis_stream_mc* streams,
                                      float* residue, uint32_t n_packets, uint32_t channels, uint32_t slot, cudaStream_t stream) {
    if (n_packets == 0) return cudaSuccess;
    const dim3 grid((slot + 255) / 256 < 16 ? (slot + 255) / 256 : 16, n_packets);
    vorbis_mc_decouple_kernel<<<grid, 256, 0, stream>>>(units, stream_of_packet, streams, residue, n_packets, channels, slot);
    return cudaGetLastError();
}

cudaError_t vorbis_mc_split_units_launch(const symgpu_vorbis_unit_mc* units, uint32_t n_packets, uint32_t pair, symgpu_vorbis_unit* out,
                                         cudaStream_t stream) {
    if (n_packets == 0) return cudaSuccess;
    vorbis_mc_split_units_kernel<<<(n_packets + 255) / 256, 256, 0, stream>>>(units, n_packets, pair, out);
    return cudaGetLastError();
}

// SYMGPU_VORBIS_KERNEL = z (one warp per packet-channel, Z layout: the default) | pair (64 threads per packet, array layout)
bool vorbis_kernel_z() {
    static int mode = -1;
    if (mode < 0) {
        const char* env = getenv("SYMGPU_VORBIS_KERNEL");
        mode = (env && env[0] == 'p') ? 0 : 1;
    }
    return mode == 1;
}

int vorbis_slots_for(int max_bs1_exp) {
    if (vorbis_kernel_z()) {
        // eight slots when two CTAs of them share an SM or when they fit at all; fewer for the largest blocks
        const size_t per = 2 * vorbis_unit_bytes(1 << (max_bs1_exp - 1));
        const int n = (int)((216u * 1024u - vorbis_z_tab_bytes(1 << (max_bs1_exp - 1))) / per);
        return n < 2 ? 2 : (n > 8 ? 8 : n);
    }
    const size_t per = vorbis_slot_bytes(1 << (max_bs1_exp - 1));
    const int n = (int)((200u * 1024u) / per);
    return n < 2 ? 2 : (n > 8 ? 8 : n);
}

// n_slots: packet slots per CTA the chunks were cut for (chunk packets + 1), at most vorbis_slots_for(max_bs1_exp); batches of
// short runs use fewer, so that more (smaller) CTAs share an SM instead of leaving warps of a big one idle.
cudaError_t vorbis_launch(const VorbisArgs& a, int n_chunks, int max_bs1_exp, int n_slots, cudaStream_t stream) {
    const int slot_smem = 1 << (max_bs1_exp - 1);
    if (n_slots < 2 || n_slots > vorbis_slots_for(max_bs1_exp)) n_slots = vorbis_slots_for(max_bs1_exp);
    if (vorbis_kernel_z()) {
        const size_t smem = 2 * vorbis_unit_bytes(slot_smem) * n_slots + vorbis_z_tab_bytes(slot_smem);
        static size_t configured = 0;
        if (smem > configured) {
            cudaError_t e = cudaFuncSetAttribute(vorbis_synth_kernel_z, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            configured = smem;
        }
        vorbis_synth_kernel_z<<<n_chunks, n_slots * 64, smem, stream>>>(a, slot_smem);
        return cudaGetLastError();
    }
    const size_t smem = vorbis_slot_bytes(slot_smem) * n_slots;
    static size_t configured = 0;
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(vorbis_synth_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        configured = smem;
    }
    vorbis_synth_kernel<<<n_chunks, n_slots * kVorbisThreads, smem, stream>>>(a, slot_smem);
    return cudaGetLastError();
}

} // namespace symgpu
