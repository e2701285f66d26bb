// Layer III entropy decoding of ONE granule-channel -- scale factors (part 2) and the Huffman-coded spectrum (part 3) --
// written once for host and device.  The CPU front-end (mp3_frontend.cpp) calls these functions frame after frame; the
// device path (mp3_entropy_kernel.cu) calls the SAME functions with one thread per granule-channel, which is possible
// because a granule-channel's first bit is known from the side information alone: the sum of the part2_3_length fields
// before it (layer3/mod.rs:272-370 advances `part2_3_begin` by exactly that).  So every CPU test of the front-end is a
// test of the code the kernel runs.
//
// The per-packet rules of Layer III live here too, for the same reason: the packet prologue (shared with Layer I / II,
// mpa12_entropy.h), the side read into a FrameSide record and one step of the bit reservoir.  symgpu_mp3_fe_decode,
// symgpu_mp3_entropy_plan and the device decoder (mp3_decode_kernel.cu) are loops over them.
//
// Reference: read_scale_factors_mpeg1 / _mpeg2 (symphonia-bundle-mp3/src/layer3/bitstream.rs:240-427),
// read_huffman_samples (layer3/requantize.rs:47-237), BitReaderLtr::read_codebook (symphonia-core/src/io/bit.rs:771-808).
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

#ifdef __CUDACC__
#define SYMGPU_HD __host__ __device__ __forceinline__
#else
#define SYMGPU_HD inline
#endif
#ifdef __CUDA_ARCH__
#define SYMGPU_UNROLL _Pragma("unroll")
#else
#define SYMGPU_UNROLL
#endif

namespace symgpu {
namespace mp3e {

// All Huffman lookup tables in one flat array (host: built once; device: a copy in global memory).
// Table t (0..31 big values by table_select, 32 / 33 the two quad tables) starts at base[t]; first_bits[t] == 0 marks the
// tables that hold no codes (0, 4, 14).  Entry: bits 0-7 value, 8-12 code length | bit 31: bits 0-23 offset (from the
// table's base) of a second-level table indexed by the next (bits 24-28) bits.
struct HuffSet {
    const uint32_t* lut;
    uint32_t base[34];
    uint8_t first_bits[34];
    uint8_t linbits[32];
};

// What the side information says about one granule-channel (GranuleChannel, layer3/mod.rs:145-205).
struct GcSide {
    uint16_t part2_3_length, big_values, scalefac_compress;
    uint16_t region1_start, region2_start;
    uint8_t global_gain, block_type, mixed, preflag, scalefac_scale, count1table;
    uint8_t subblock_gain[3], table_select[3];
};

// Most-significant-bit-first reader over [p, p + n_bits / 8): reads past the end fail, the window pads with zeros.
struct Bits {
    const uint8_t* p;
    size_t n_bits;
    size_t at;
    SYMGPU_HD Bits(const uint8_t* data, size_t n_bytes, size_t start_bit = 0) : p(data), n_bits(n_bytes * 8), at(start_bit) {}
    SYMGPU_HD uint32_t window() const {  // the next 32 bits, left-aligned
        const size_t byte = at >> 3, n = n_bits >> 3;
#if !defined(__CUDA_ARCH__) && !defined(SYMGPU_MP3E_DEVICE_WINDOW)
        if (byte + 8 <= n) {  // host fast path: one unaligned load (SYMGPU_MP3E_DEVICE_WINDOW: build the host code with the device's path, for tests)
            uint64_t w;
            __builtin_memcpy(&w, p + byte, 8);
            return uint32_t((__builtin_bswap64(w) << (at & 7)) >> 32);
        }
#endif
        uint64_t v = 0;
SYMGPU_UNROLL
        for (int k = 0; k < 5; ++k) v = v << 8 | (byte + k < n ? p[byte + k] : 0);
        return uint32_t((v << (at & 7)) >> 8);
    }
    SYMGPU_HD size_t left() const { return n_bits - at; }
    SYMGPU_HD bool read(unsigned width, uint32_t& v) {  // width <= 25
        if (width > left()) return false;
        v = width ? window() >> (32 - width) : 0;
        at += width;
        return true;
    }
    SYMGPU_HD bool skip(size_t width) {
        if (width > left()) return false;
        at += width;
        return true;
    }
};

SYMGPU_HD void huff_decode(const HuffSet& hs, int table, uint32_t win, unsigned& value, unsigned& len) {
    const uint32_t* lut = hs.lut + hs.base[table];
    const unsigned first = hs.first_bits[table];
    uint32_t e = lut[win >> (32 - first)];
    if (e & 0x80000000u) {
        const unsigned sub = (e >> 24) & 31;
        e = lut[(e & 0xffffff) + ((win << first) >> (32 - sub))];
    }
    value = e & 0xff, len = (e >> 8) & 31;
}

// Part 2 of an MPEG-1 granule-channel.  `copy_from`: granule 0's scale factors of the same channel when this is granule
// 1 (groups flagged in scfsi are copied instead of read), else null.  Returns the bits read, -1 when they run out.
SYMGPU_HD int read_scale_factors_mpeg1(Bits& bs, const GcSide& c, const uint8_t* copy_from, unsigned scfsi_mask, uint8_t* scalefacs) {
    const unsigned sfc = c.scalefac_compress & 15;
    // slen1 = 0 0 0 0 3 1 1 1 2 2 2 3 3 3 4 4 and slen2 = 0 1 2 3 0 1 2 3 1 2 3 1 2 3 2 3 by scalefac_compress, one nibble each
    const unsigned s1 = (0x4433322211130000ull >> (4 * sfc)) & 15, s2 = (0x3232132132103210ull >> (4 * sfc)) & 15;
    uint32_t v;
    if (c.block_type == 2) {
        const int n1 = c.mixed ? 17 : 18;
        if (s1)
            for (int i = 0; i < n1; ++i) {
                if (!bs.read(s1, v)) return -1;
                scalefacs[i] = uint8_t(v);
            }
        if (s2)
            for (int i = n1; i < n1 + 18; ++i) {
                if (!bs.read(s2, v)) return -1;
                scalefacs[i] = uint8_t(v);
            }
        return n1 * int(s1) + 18 * int(s2);
    }
    int bits = 0;
    for (int g = 0; g < 4; ++g) {
        const int a = g == 0 ? 0 : g == 1 ? 6 : g == 2 ? 11 : 16, b = g == 0 ? 6 : g == 1 ? 11 : g == 2 ? 16 : 21;
        const unsigned s = g < 2 ? s1 : s2;
        if (copy_from && (scfsi_mask >> g & 1)) {
            for (int i = a; i < b; ++i) scalefacs[i] = copy_from[i];
        } else if (s) {
            for (int i = a; i < b; ++i) {
                if (!bs.read(s, v)) return -1;
                scalefacs[i] = uint8_t(v);
            }
            bits += int(s) * (b - a);
        }
    }
    return bits;
}

// Part 2 of an MPEG-2 / 2.5 granule-channel; sets *preflag for a channel that is not the intensity channel.
SYMGPU_HD int read_scale_factors_mpeg2(Bits& bs, bool intensity_channel, const GcSide& c, uint8_t* preflag, uint8_t* scalefacs) {
    // band counts per partition [table row][long | short | mixed], ISO 13818-3 2.4.3.2
    const uint8_t nsfb[6][3][4] = {
        {{7, 7, 7, 0}, {12, 12, 12, 0}, {6, 15, 12, 0}}, {{6, 6, 6, 3}, {12, 9, 9, 6}, {6, 12, 9, 6}}, {{8, 8, 5, 0}, {15, 12, 9, 0}, {6, 18, 9, 0}},
        {{6, 5, 5, 5}, {9, 9, 9, 9}, {6, 9, 9, 9}},      {{6, 5, 7, 3}, {9, 9, 12, 6}, {6, 9, 12, 6}}, {{11, 10, 0, 0}, {18, 18, 0, 0}, {15, 18, 0, 0}}};
    const int block = c.block_type == 2 ? (c.mixed ? 2 : 1) : 0;
    unsigned slen[4] = {0, 0, 0, 0};
    int row;
    if (intensity_channel) {
        const unsigned sfc = c.scalefac_compress >> 1;
        if (sfc < 180) row = 0, slen[0] = sfc / 36, slen[1] = (sfc % 36) / 6, slen[2] = (sfc % 36) % 6;
        else if (sfc < 244) row = 1, slen[0] = ((sfc - 180) % 64) >> 4, slen[1] = ((sfc - 180) % 16) >> 2, slen[2] = (sfc - 180) % 4;
        else row = 2, slen[0] = (sfc - 244) / 3, slen[1] = (sfc - 244) % 3;
    } else {
        const unsigned sfc = c.scalefac_compress;
        *preflag = sfc >= 500;
        if (sfc < 400) row = 3, slen[0] = (sfc >> 4) / 5, slen[1] = (sfc >> 4) % 5, slen[2] = (sfc % 16) >> 2, slen[3] = sfc % 4;
        else if (sfc < 500) row = 4, slen[0] = ((sfc - 400) >> 2) / 5, slen[1] = ((sfc - 400) >> 2) % 5, slen[2] = (sfc - 400) % 4;
        else row = 5, slen[0] = (sfc - 500) / 3, slen[1] = (sfc - 500) % 3;
    }
    int bits = 0, start = 0;
    uint32_t v;
    for (int k = 0; k < 4; ++k) {
        const int n = nsfb[row][block][k];
        if (slen[k]) {
            for (int i = start; i < start + n; ++i) {
                if (!bs.read(slen[k], v)) return -1;
                scalefacs[i] = uint8_t(v);
            }
            bits += int(slen[k]) * n;
        }
        start += n;
    }
    return bits;
}

// Part 3: the spectrum as sign * x (the reference writes sign * POW43[x], requantize.rs:128, :144); all 576 lines of `q`
// are written.  Returns rzero, -1 on an over-read.
SYMGPU_HD int read_huffman(Bits& bs, const HuffSet& hs, const GcSide& c, uint32_t part3_bits, int16_t* q) {
    if (part3_bits == 0) {
        for (int k = 0; k < 576; ++k) q[k] = 0;
        return 0;
    }
    const size_t end = bs.at + part3_bits;  // the reference's "bits_read < part3_bits" is "bs.at < end"
    const int big_len = 2 * int(c.big_values);
    int i = 0;
    for (int r = 0; r < 3; ++r) {
        const int limit = r == 0 ? c.region1_start : r == 1 ? c.region2_start : 576;
        const int region_end = limit < big_len ? limit : big_len;
        const int table = c.table_select[r];
        const unsigned linbits = hs.linbits[table];
        if (hs.first_bits[table] == 0) {  // tables 0, 4, 14: a silent region that costs no bits
            for (; i < region_end; ++i) q[i] = 0;
            continue;
        }
        while (i < region_end && bs.at < end) {
            unsigned value, len;
            const uint32_t win = bs.window();
            huff_decode(hs, table, win, value, len);
            if (len > bs.left()) return -1;
            if (!linbits) {
                // tables without linbits (0..15): the code (<= 19 bits) and its at most two sign bits sit in one window
                const unsigned x = value >> 4, y = value & 15;
                const unsigned need = len + (x != 0) + (y != 0);
                if (need > bs.left()) return -1;
                uint32_t tail = win << len;  // the bits behind the code, left-aligned
                int16_t ox = 0, oy = 0;
                if (x) ox = int16_t((tail >> 31) ? -int(x) : int(x)), tail <<= 1;
                if (y) oy = int16_t((tail >> 31) ? -int(y) : int(y));
                q[i] = ox, q[i + 1] = oy;
                bs.at += need;
                i += 2;
                continue;
            }
            bs.at += len;
SYMGPU_UNROLL
            for (int k = 0; k < 2; ++k) {
                unsigned x = k == 0 ? value >> 4 : value & 15;
                int16_t out = 0;
                if (x) {
                    uint32_t extra, sign;
                    if (x == 15) {
                        if (!bs.read(linbits, extra)) return -1;
                        x += extra;
                    }
                    if (!bs.read(1, sign)) return -1;
                    out = int16_t(sign ? -int(x) : int(x));
                }
                q[i + k] = out;
            }
            i += 2;
        }
    }
    const int quad = 32 + c.count1table;
    while (i <= 572 && bs.at < end) {
        unsigned value, len;
        huff_decode(hs, quad, bs.window(), value, len);
        if (len > bs.left()) return -1;
        bs.at += len;
        const unsigned ones = (value >> 3 & 1) + (value >> 2 & 1) + (value >> 1 & 1) + (value & 1);
        uint32_t signs;
        if (!bs.read(ones, signs)) return -1;
        // sign bits come in the order v, w, x, y; the reference peels them off from the last one (requantize.rs:170-203)
SYMGPU_UNROLL
        for (int k = 3; k >= 0; --k) {
            int16_t out = 0;
            if (value & (1u << (3 - k))) {
                out = (signs & 1) ? -1 : 1;
                signs >>= 1;
            }
            q[i + k] = out;
        }
        i += 4;
    }
    if (bs.at < end) {
        if (!bs.skip(end - bs.at)) return -1;  // stuffing
    } else if (bs.at > end && i > big_len) {
        i -= 4;  // the last quad came out of bits that belong to the next granule: undo it (requantize.rs:222-226)
    }
    for (int k = i; k < 576; ++k) q[k] = 0;
    return i;
}

// ---- one granule-channel as a unit of parallel work ---------------------------------------------------------------
// The host walks the frames once (headers, side information, bit-reservoir arithmetic: none of it needs the Huffman
// data) and emits one job per unit slot; the main data of all frames is compacted into one byte stream `md`, in which
// a frame's reservoir -- the bytes main_data_begin reaches back to plus its own -- is one contiguous window.
enum : uint8_t { kJobDecode = 0, kJobSilent = 1, kJobMute = 2 };
struct GcJob {  // 64 bytes
    uint64_t seg_begin;      // byte offset in md of the frame's reservoir window
    uint32_t seg_len;        // its length: reads beyond it fail exactly where the reference's reservoir ends
    uint32_t bit_begin;      // first bit of this granule-channel's part 2, from seg_begin
    uint32_t gr0_bit_begin;  // MPEG-1 granule 1 with scfsi: where granule 0's part 2 (same channel) starts; ~0u = it was never read
    uint32_t out_index;      // unit slot: frame * 4 + granule * 2 + channel
    GcSide side;             // 22 bytes
    uint16_t gr0_scalefac_compress;
    uint8_t gr0_block_type, gr0_mixed;
    uint8_t kind;            // kJobDecode | kJobSilent (bits lost to an underflow: zeros, side information kept) | kJobMute (absent unit)
    uint8_t mpeg1, intensity_channel, scfsi;
    uint8_t unit_flags;      // frame-level SYMGPU_MP3_F_* bits
    uint8_t sample_rate_idx;
    uint8_t reserved[8];
};
static_assert(sizeof(GcJob) == 64, "GcJob is 64 bytes");

// Fills one unit and its 576 quantised lines.  Returns 0, or 1 when the reference would refuse the frame here
// ("part2_3_length is not valid", "huffman decode overrun", an offset past the reservoir: layer3/mod.rs:318-358).
SYMGPU_HD int decode_gc_job(const GcJob& j, const uint8_t* md, const HuffSet& hs, symgpu_mp3_gc* unit, int16_t* q) {
    symgpu_mp3_gc u;
    u.rzero = 0, u.global_gain = 0, u.block_type = 0, u.flags = j.unit_flags, u.sample_rate_idx = j.sample_rate_idx;
    for (int k = 0; k < 3; ++k) u.subblock_gain[k] = 0;
    for (int k = 0; k < 39; ++k) u.scalefacs[k] = 0;
    for (int k = 0; k < 16; ++k) u.reserved[k] = 0;
    int status = 0;
    if (j.kind == kJobMute) {
        u.flags |= SYMGPU_MP3_F_MUTE;
        for (int k = 0; k < 576; ++k) q[k] = 0;
    } else {
        const GcSide& c = j.side;
        uint8_t preflag = c.preflag;
        int rzero = 0;
        if (j.kind == kJobSilent) {
            for (int k = 0; k < 576; ++k) q[k] = 0;
        } else {
            const uint8_t* seg = md + j.seg_begin;
            Bits bs(seg, j.seg_len, j.bit_begin);
            int part2 = -1;
            if ((j.bit_begin >> 3) <= j.seg_len && bs.at <= bs.n_bits) {
                if (j.mpeg1) {
                    uint8_t first[39];
                    const uint8_t* copy_from = nullptr;
                    if (j.scfsi && c.block_type != 2 && (j.out_index & 2)) {  // granule 1 repeating groups of granule 0
                        for (int k = 0; k < 39; ++k) first[k] = 0;
                        copy_from = first;
                        if (j.gr0_bit_begin != ~0u) {
                            GcSide g0 = c;
                            g0.scalefac_compress = j.gr0_scalefac_compress, g0.block_type = j.gr0_block_type, g0.mixed = j.gr0_mixed;
                            Bits b0(seg, j.seg_len, j.gr0_bit_begin);
                            read_scale_factors_mpeg1(b0, g0, nullptr, 0, first);  // its own failure is granule 0's job to report
                        }
                    }
                    part2 = read_scale_factors_mpeg1(bs, c, copy_from, j.scfsi, u.scalefacs);
                } else {
                    part2 = read_scale_factors_mpeg2(bs, j.intensity_channel != 0, c, &preflag, u.scalefacs);
                }
            }
            if (part2 < 0 || uint32_t(part2) > c.part2_3_length) {
                status = 1;
                for (int k = 0; k < 576; ++k) q[k] = 0;
            } else {
                rzero = read_huffman(bs, hs, c, uint32_t(c.part2_3_length) - uint32_t(part2), q);
                if (rzero < 0) status = 1, rzero = 0;
            }
        }
        u.rzero = uint16_t(rzero), u.global_gain = c.global_gain, u.block_type = c.block_type;
        u.flags |= uint8_t((c.mixed ? SYMGPU_MP3_F_MIXED : 0) | (c.scalefac_scale ? SYMGPU_MP3_F_SCALEFAC_SCALE : 0) | (preflag ? SYMGPU_MP3_F_PREFLAG : 0) |
                           ((c.scalefac_compress & 1) ? SYMGPU_MP3_F_SFC_LSB : 0));
        for (int k = 0; k < 3; ++k) u.subblock_gain[k] = c.subblock_gain[k];
    }
    *unit = u;
    return status;
}

// ---- packet prologue (decoder.rs:87-128), in the reference's order; all MPEG audio layers ------------------------------
// 1. read_header: the sync search inside the packet, the header parse, frame_size == the bytes after the header word.
// 2. (the caller) the signal specification: the first packet that passes 1 fixes (sample rate, channels); a later packet
//    that differs is refused.  So a packet of the wrong layer but the right size still fixes it.
// 3. body_of: the layer check, the CRC skip.
enum : int { kDecoded = 0, kRefused = 1, kUnsupported = 2 };
SYMGPU_HD int read_header(const uint8_t* frame, size_t n, symgpu::packet::MpaHeader& h, size_t& q) {
    using namespace symgpu::packet;
    uint32_t word = 0;
    for (q = 0;; ++q) {  // decoder.rs:87: synchronise inside the packet
        if (q + 4 > n) return kRefused;
        word = detail::be32(frame + q);
        if (mpa_is_synced(word) && mpa_check_header(word)) break;
    }
    const Status hs = mpa_parse_header(word, h);
    if (hs != Status::Ok) return hs == Status::Unsupported ? kUnsupported : kRefused;
    return h.frame_size == n - q - 4 ? kDecoded : kRefused;
}
SYMGPU_HD bool body_of(const symgpu::packet::MpaHeader& h, int layer, size_t n, size_t q, uint32_t& at, uint32_t& bytes) {
    if (h.layer != layer) return false;
    const size_t body_len = n - q - 4, crc_len = h.crc ? 2 : 0;
    if (body_len < crc_len) return false;
    at = uint32_t(q + 4 + crc_len), bytes = uint32_t(body_len - crc_len);
    return true;
}

// ---- Layer III side information of one packet --------------------------------------------------------------------------
// The long-block band edges the side read needs (region boundaries), by sample-rate index: computed once on the host
// (tables.cpp) and handed to the kernels as a parameter, never rebuilt in device code.
struct LongEdges {
    uint16_t e[9][23];
};

enum : uint8_t { kSideRefused = 0, kSideBad = 1, kSideOk = 2 };

// What the prologue and the side read leave for the reservoir walk.  108 bytes.
struct FrameSide {
    uint32_t body_at;          // byte offset, in the packet, of the side information (after the header word and the CRC)
    uint32_t body_bytes;       // bytes from there to the end of the packet
    uint16_t main_data_begin;
    uint8_t state;             // kSideRefused (the prologue refused the packet), kSideBad (the side read failed), kSideOk
    uint8_t n_ch, n_gr, mpeg1, intensity, side_len;
    uint8_t unit_flags;        // frame-level SYMGPU_MP3_F_* bits
    uint8_t sample_rate_idx;
    uint8_t mismatch;          // joint stereo with channels on different window sequences (stereo.rs:503-505)
    uint8_t scfsi[2];          // bit g: group g of granule 1 repeats granule 0's scale factors
    uint8_t reserved;
    GcSide gc[2][2];
};

// bitstream.rs:57-236
SYMGPU_HD bool read_side_info(Bits& bs, const symgpu::packet::MpaHeader& h, const uint16_t* long_edges, FrameSide& f) {
    using symgpu::packet::MpaVersion;
    const bool mpeg1 = h.version == MpaVersion::Mpeg1;
    const int n_ch = h.n_channels(), n_gr = h.n_granules();
    uint32_t v;
    if (mpeg1) {
        if (!bs.read(9, v)) return false;
        f.main_data_begin = uint16_t(v);
        if (!bs.skip(n_ch == 1 ? 5 : 3)) return false;
        for (int ch = 0; ch < n_ch; ++ch) {
            if (!bs.read(4, v)) return false;
            f.scfsi[ch] = uint8_t((v >> 3 & 1) | (v >> 1 & 2) | (v << 1 & 4) | (v << 3 & 8));  // first bit read = group 0
        }
    } else {
        if (!bs.read(8, v)) return false;
        f.main_data_begin = uint16_t(v);
        if (!bs.skip(n_ch == 1 ? 1 : 2)) return false;
    }
    for (int gr = 0; gr < n_gr; ++gr)
        for (int ch = 0; ch < n_ch; ++ch) {
            GcSide& c = f.gc[gr][ch];
            if (!bs.read(12, v)) return false;
            c.part2_3_length = uint16_t(v);
            if (!bs.read(9, v)) return false;
            c.big_values = uint16_t(v);
            if (c.big_values > 288) return false;
            if (!bs.read(8, v)) return false;
            c.global_gain = uint8_t(v);
            if (!bs.read(mpeg1 ? 4 : 9, v)) return false;
            c.scalefac_compress = uint16_t(v);
            if (!bs.read(1, v)) return false;
            if (v) {  // window switching
                uint32_t type, mixed;
                if (!bs.read(2, type) || !bs.read(1, mixed)) return false;
                if (type == 0) return false;
                c.block_type = uint8_t(type == 1 ? SYMGPU_MP3_START : type == 2 ? SYMGPU_MP3_SHORT : SYMGPU_MP3_END);
                c.mixed = type == 2 && mixed;
                for (int i = 0; i < 2; ++i) {
                    if (!bs.read(5, v)) return false;
                    c.table_select[i] = uint8_t(v);
                }
                for (int i = 0; i < 3; ++i) {
                    if (!bs.read(3, v)) return false;
                    c.subblock_gain[i] = uint8_t(v);
                }
                // region0 ends after 36 lines (MPEG-1, and short blocks of MPEG-2), 54 (MPEG-2 long transitions), or,
                // for MPEG-2.5, after 6 (pure short) / 8 long bands of the rate's table (bitstream.rs:108-150)
                if (h.version == MpaVersion::Mpeg2p5) c.region1_start = long_edges[type == 2 && !mixed ? 6 : 8];
                else c.region1_start = (mpeg1 || type == 2) ? 36 : 54;
                c.region2_start = 576;
            } else {
                c.block_type = SYMGPU_MP3_LONG;
                for (int i = 0; i < 3; ++i) {
                    if (!bs.read(5, v)) return false;
                    c.table_select[i] = uint8_t(v);
                }
                uint32_t r0, r1;
                if (!bs.read(4, r0) || !bs.read(3, r1)) return false;
                const unsigned a = r0 + 1, b = r1 + a + 1;
                c.region1_start = long_edges[a];
                c.region2_start = b <= 22 ? long_edges[b] : 576;
            }
            if (mpeg1) {
                if (!bs.read(1, v)) return false;
                c.preflag = uint8_t(v);
            }
            if (!bs.read(1, v)) return false;
            c.scalefac_scale = uint8_t(v);
            if (!bs.read(1, v)) return false;
            c.count1table = uint8_t(v);
        }
    return true;
}

// The side read of a packet that passed the prologue and the layer check: `side` = the packet + at, `bytes` long.  Fills
// the whole record; state kSideBad where the read fails (the reference then empties the reservoir).
SYMGPU_HD void read_frame_side(const uint8_t* side, uint32_t at, uint32_t bytes, const symgpu::packet::MpaHeader& h, const LongEdges& E,
                               FrameSide& f) {
    using symgpu::packet::MpaMode;
    f = FrameSide{};
    f.body_at = at, f.body_bytes = bytes;
    f.n_ch = uint8_t(h.n_channels()), f.n_gr = uint8_t(h.n_granules()), f.mpeg1 = h.version == symgpu::packet::MpaVersion::Mpeg1;
    f.intensity = h.mode == MpaMode::JointStereo && h.intensity;
    f.side_len = uint8_t(h.side_info_len());
    f.sample_rate_idx = h.sample_rate_idx;
    const bool mid_side = h.mode == MpaMode::JointStereo && h.mid_side;
    f.unit_flags = uint8_t((f.mpeg1 ? SYMGPU_MP3_F_MPEG1 : 0) | (mid_side ? SYMGPU_MP3_F_MID_SIDE : 0) | (f.intensity ? SYMGPU_MP3_F_INTENSITY : 0));
    Bits bs(side, bytes);
    // (side_len > bytes cannot happen for a frame of the right size; the reference would panic slicing)
    if (!read_side_info(bs, h, E.e[h.sample_rate_idx], f) || f.side_len > bytes) {
        f.state = kSideBad;
        return;
    }
    f.state = kSideOk;
    // a joint-stereo pair must share its window sequence: the reference refuses the frame in its stereo stage, after the
    // main data was read (stereo.rs:503-505)
    if (f.n_ch == 2 && (mid_side || f.intensity))
        for (int gr = 0; gr < f.n_gr; ++gr) {
            const GcSide &a = f.gc[gr][0], &b = f.gc[gr][1];
            if (a.block_type != b.block_type || (a.block_type == SYMGPU_MP3_SHORT && a.mixed != b.mixed)) f.mismatch = 1;
        }
}

// ---- one step of the bit reservoir (BitResevoir::fill / consume, layer3/mod.rs:42-108, :272-370) ------------------------
// The reservoir as byte counts: `len` bytes held, `consumed` of them read; md_at = where the next frame's main data goes in
// the compacted stream md.  A frame's reservoir window is the `reuse` bytes main_data_begin reaches back to (at most what
// is unread) plus its own slot: one contiguous range of md.
struct Reservoir {
    uint32_t len, consumed;
    uint64_t md_at;
};
enum : int { kStepDecoded = 0, kStepRefused = 1, kStepFailed = 2, kStepLeftOut = 3 };
struct StepOut {
    uint64_t copy_at;      // where the frame's slot goes in md (kStepDecoded, kStepLeftOut)
    uint32_t slot;         // its main-data bytes in this packet
    uint32_t reuse;        // bytes of the window that come from earlier frames
    uint32_t underflow;    // main_data_begin pointed this many bytes before what the reservoir holds
    uint32_t used;         // bytes of the window the frame's granules take
};

// One packet's effect on the reservoir.  bad: 0, 1 = its main data is known to over-read (the reference drops the frame
// and empties the reservoir), 2 = left out although its main data is consumed (the device path passes 2 for s.mismatch).
//   kStepRefused  the prologue refused the packet (nothing changes); the side read failed (the reservoir is emptied);
//                 main_data_begin + slot > 2048 (refused before the reservoir is touched, mod.rs:49-51)
//   kStepFailed   bad == 1: the reservoir is emptied (mod.rs:409-414)
//   kStepLeftOut  the reservoir moves on as for a decoded frame; the frame yields no audio
//   kStepDecoded  a frame
// For kStepDecoded and kStepLeftOut, jobs[0..3] (when not null) are the frame's four granule-channels, unit slots
// out_frame * 4 + granule * 2 + channel, seg_begin in md.
SYMGPU_HD int reservoir_step(Reservoir& r, const FrameSide& s, uint8_t bad, uint32_t out_frame, GcJob* jobs, StepOut& o) {
    if (s.state == kSideRefused) return kStepRefused;
    if (s.state == kSideBad) {
        r.len = r.consumed = 0;
        return kStepRefused;
    }
    const uint32_t slot = s.body_bytes - s.side_len, begin = s.main_data_begin;
    if (begin + slot > 2048) return kStepRefused;
    if (bad == 1) {
        r.len = r.consumed = 0;
        return kStepFailed;
    }
    const uint32_t unread = r.len - r.consumed;
    const uint32_t reuse = begin <= unread ? begin : unread;
    o.copy_at = r.md_at, o.slot = slot, o.reuse = reuse, o.underflow = begin - reuse;
    const uint64_t seg_begin = r.md_at - reuse;
    const uint32_t seg_len = reuse + slot;
    r.md_at += slot;
    r.len = seg_len, r.consumed = 0;
    const uint32_t underflow_bits = 8 * o.underflow;
    uint32_t skipped = 0, gr0_begin[2] = {~0u, ~0u};
    uint32_t part_begin = 0;
    for (int gr = 0; gr < 2; ++gr) {
        const bool silent = gr < s.n_gr && skipped < underflow_bits;
        for (int ch = 0; ch < 2; ++ch) {
            GcJob j{};
            j.seg_begin = seg_begin, j.seg_len = seg_len, j.out_index = out_frame * 4 + uint32_t(gr * 2 + ch);
            j.unit_flags = s.unit_flags, j.sample_rate_idx = s.sample_rate_idx, j.mpeg1 = s.mpeg1, j.gr0_bit_begin = ~0u;
            if (gr >= s.n_gr || ch >= s.n_ch) {
                j.kind = kJobMute;
            } else {
                const GcSide& c = s.gc[gr][ch];
                j.side = c;
                j.intensity_channel = ch > 0 && s.intensity, j.scfsi = s.scfsi[ch];
                if (silent) {
                    j.kind = kJobSilent;
                    skipped += c.part2_3_length;
                } else {
                    j.kind = kJobDecode;
                    j.bit_begin = part_begin;
                    if (gr == 0) gr0_begin[ch] = j.bit_begin;
                    else {
                        j.gr0_bit_begin = gr0_begin[ch];
                        j.gr0_scalefac_compress = s.gc[0][ch].scalefac_compress, j.gr0_block_type = s.gc[0][ch].block_type, j.gr0_mixed = s.gc[0][ch].mixed;
                    }
                    part_begin += c.part2_3_length;
                }
            }
            if (jobs) jobs[gr * 2 + ch] = j;
        }
        if (silent && skipped > underflow_bits) part_begin = skipped - underflow_bits;
    }
    o.used = (part_begin + 7) >> 3;
    r.consumed = r.len < o.used ? r.len : o.used;
    return bad == 2 ? kStepLeftOut : kStepDecoded;
}

}  // namespace mp3e

// The flat tables (host memory, built once; thread-safe).  `words` = length of lut.
const mp3e::HuffSet& mp3_huffset_host(size_t* words);
// The long-block band edges of every sample rate (host memory, built once from tables.cpp; thread-safe).
const mp3e::LongEdges& mp3_long_edges_host();
#ifdef __CUDACC__
// The same Huffman tables with `lut` in global memory of `device`, uploaded once per device (mp3_entropy_kernel.cu).
cudaError_t device_huffset(int device, mp3e::HuffSet& out);
#endif

}  // namespace symgpu
