// FLAC frame decoding of ONE packet -- sync search, frame header with its CRC-8, sub-frame headers, warm-up samples,
// quantised predictor coefficients and Rice-coded residuals -- written once for host and device.  The CPU front-end
// (flac_frontend.cpp, symgpu_flac_fe_decode_packets) calls decode_packet packet after packet; the device path
// (flac_decode_kernel.cu) calls the SAME function with one thread per packet, which is possible because a FLAC frame
// carries no state into the next one.  So every CPU test of the front-end is a test of the code the kernel runs.
//
// Reference: sync_frame, read_frame_header (symphonia-bundle-flac/src/frame.rs:66-233, utf8 :281-333),
// FlacDecoder::decode_inner up to the restoration (decoder.rs:139-228), read_subframe and decode_* (decoder.rs:340-520),
// decode_residual / decode_rice_partition (decoder.rs:522-640).
//
// The bit reader is mp3_entropy.h's Bits: its window pads with zeros past the end of the packet and every read that
// would leave the packet fails, so nothing outside [p, p + len) is ever loaded -- what makes it safe to run on
// untrusted bytes on the device.  Prediction, wasted-bit shifts, decorrelation and scaling are NOT done here: they are
// the data-parallel half (flac_kernel.cu).
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu.h"
#include "mp3_entropy.h"  // Bits, SYMGPU_HD

namespace symgpu {
namespace flace {

using mp3e::Bits;

SYMGPU_HD uint8_t crc8(const uint8_t* p, size_t n) {  // polynomial 0x07, initial value 0 (symphonia-core/src/checksum/crc8.rs:32-65)
    uint8_t c = 0;
    for (size_t i = 0; i < n; ++i) {
        c ^= p[i];
        for (int k = 0; k < 8; ++k) c = uint8_t(c & 0x80 ? (c << 1) ^ 0x07 : c << 1);
    }
    return c;
}

SYMGPU_HD int32_t sign_extend(uint32_t v, unsigned bits) { return bits ? int32_t(v << (32 - bits)) >> (32 - bits) : 0; }

SYMGPU_HD unsigned clz32(uint32_t w) {  // w != 0
#ifdef __CUDA_ARCH__
    return unsigned(__clz(w));
#else
    return unsigned(__builtin_clz(w));
#endif
}

struct Reader {  // bit reader with the two reads FLAC adds: up to 32 bits, and unary
    Bits b;
    SYMGPU_HD Reader(const uint8_t* p, size_t n) : b(p, n) {}
    SYMGPU_HD bool read(unsigned width, uint32_t& v) {  // width <= 32
        if (width <= 24) return b.read(width, v);
        uint32_t hi, lo;
        if (!b.read(width - 16, hi) || !b.read(16, lo)) return false;
        v = hi << 16 | lo;
        return true;
    }
    SYMGPU_HD bool read_signed(unsigned width, int32_t& v) {
        uint32_t u;
        if (!read(width, u)) return false;
        v = sign_extend(u, width);
        return true;
    }
    SYMGPU_HD bool unary(uint32_t& zeros) {  // zeros before the next 1 bit (bit.rs:642-671); the data ending first is an error
        zeros = 0;
        for (;;) {
            if (b.left() == 0) return false;
            const uint32_t w = b.window();
            const size_t take = b.left() < 32 ? b.left() : 32;
            if (w == 0) {
                zeros += uint32_t(take), b.at += take;
                continue;
            }
            const unsigned lead = clz32(w);
            if (lead >= take) {
                zeros += uint32_t(take), b.at += take;
                continue;
            }
            zeros += lead, b.at += lead + 1;
            return true;
        }
    }
};

struct Header {
    uint64_t sequence;
    bool by_sample;
    uint32_t block, rate, bps;  // rate / bps 0: not in the header
    uint32_t channels;
    uint8_t assignment;
    size_t size;                // bytes, sync code to CRC-8 inclusive
};

SYMGPU_HD uint32_t rate_of_code(uint32_t code) {  // codes 0..11 (frame.rs:150-175); 0: take it from the stream information
    switch (code) {
        case 1: return 88200;
        case 2: return 176400;
        case 3: return 192000;
        case 4: return 8000;
        case 5: return 16000;
        case 6: return 22050;
        case 7: return 24000;
        case 8: return 32000;
        case 9: return 44100;
        case 10: return 48000;
        case 11: return 96000;
        default: return 0;
    }
}

// frame.rs:66-233.  0 ok, 1 decode error.
SYMGPU_HD int read_header(const uint8_t* p, size_t n, size_t at, Header& h) {
    const size_t start = at;
    if (at + 4 > n) return 1;
    const uint16_t sync = uint16_t(p[at] << 8 | p[at + 1]);
    const uint16_t desc = uint16_t(p[at + 2] << 8 | p[at + 3]);
    at += 4;
    h.by_sample = sync & 1;
    const uint32_t bs_enc = desc >> 12, sr_enc = (desc >> 8) & 15, ch_enc = (desc >> 4) & 15, bps_enc = (desc >> 1) & 7;
    if (desc & 1) return 1;
    // the sequence number, "extended UTF-8" (frame.rs:281-333)
    {
        if (at + 1 > n) return 1;
        uint64_t v = p[at++];
        int more;
        if (v < 0x80) more = 0;
        else if (v >= 0xc0 && v <= 0xdf) more = 1, v &= 0x1f;
        else if (v >= 0xe0 && v <= 0xef) more = 2, v &= 0x0f;
        else if (v >= 0xf0 && v <= 0xf7) more = 3, v &= 0x07;
        else if (v >= 0xf8 && v <= 0xfb) more = 4, v &= 0x03;
        else if (v >= 0xfc && v <= 0xfd) more = 5, v &= 0x01;
        else if (v == 0xfe) more = 6, v = 0;
        else return 1;  // 10xxxxxx or 0xff cannot start a sequence
        for (int k = 0; k < more; ++k) {
            if (at + 1 > n) return 1;
            v = v << 6 | (p[at++] & 0x3f);
        }
        if (v > (h.by_sample ? 0x000fffffffffull : 0x7fffffffull)) return 1;
        h.sequence = v;
    }
    if (bs_enc == 0) return 1;
    else if (bs_enc == 1) h.block = 192;
    else if (bs_enc <= 5) h.block = 576u << (bs_enc - 2);
    else if (bs_enc == 6) {
        if (at + 1 > n) return 1;
        h.block = uint32_t(p[at++]) + 1;
    } else if (bs_enc == 7) {
        if (at + 2 > n) return 1;
        const uint32_t v = uint32_t(p[at] << 8 | p[at + 1]);
        at += 2;
        if (v == 0xffff) return 1;
        h.block = v + 1;
    } else h.block = 256u << (bs_enc - 8);
    if (sr_enc < 12) h.rate = rate_of_code(sr_enc);
    else if (sr_enc == 12) {
        if (at + 1 > n) return 1;
        h.rate = uint32_t(p[at++]) * 1000;
    } else if (sr_enc == 15) return 1;
    else {
        if (at + 2 > n) return 1;
        h.rate = uint32_t(p[at] << 8 | p[at + 1]) * (sr_enc == 14 ? 10 : 1);
        at += 2;
    }
    if (sr_enc != 0 && (h.rate < 1 || h.rate > 655350)) return 1;
    if (bps_enc == 3) return 1;  // widths by code: 0 (stream information), 8, 12, reserved, 16, 20, 24, 32
    h.bps = bps_enc == 0 ? 0 : bps_enc == 1 ? 8 : bps_enc == 2 ? 12 : bps_enc == 4 ? 16 : bps_enc == 5 ? 20 : bps_enc == 6 ? 24 : 32;
    if (ch_enc <= 7) h.channels = ch_enc + 1, h.assignment = SYMGPU_FLAC_INDEPENDENT;
    else if (ch_enc == 8) h.channels = 2, h.assignment = SYMGPU_FLAC_LEFT_SIDE;
    else if (ch_enc == 9) h.channels = 2, h.assignment = SYMGPU_FLAC_RIGHT_SIDE;
    else if (ch_enc == 10) h.channels = 2, h.assignment = SYMGPU_FLAC_MID_SIDE;
    else return 1;
    if (at + 1 > n) return 1;
    if (p[at] != crc8(p + start, at - start)) return 1;
    ++at;
    h.size = at - start;
    return 0;
}

// decoder.rs:522-640: residuals of samples [prelude, n) into out.  0 ok, 1 decode error.
SYMGPU_HD int read_residual(Reader& r, uint32_t prelude, int32_t* out, uint32_t n) {
    uint32_t method, order;
    if (!r.read(2, method) || method > 1 || !r.read(4, order)) return 1;
    const unsigned param_bits = method ? 5 : 4;
    const uint32_t per = n >> order;
    if (prelude > per || (uint64_t(per) << order) != n) return 1;
    for (uint32_t part = 0; part < (1u << order); ++part) {
        const uint32_t a = part ? part * per : prelude, b = (part + 1) * per;
        uint32_t param;
        if (!r.read(param_bits, param)) return 1;
        if (param < (1u << param_bits) - 1) {
            for (uint32_t i = a; i < b; ++i) {
                uint32_t q, low = 0;
                if (!r.unary(q) || !r.read(param, low)) return 1;
                const uint32_t word = (param < 32 ? q << param : 0) | low;  // (q << param) wraps in the reference for q this large; not reachable in a sized packet
                out[i] = int32_t(word >> 1) ^ -int32_t(word & 1);
            }
        } else {
            uint32_t width;
            if (!r.read(5, width)) return 1;
            for (uint32_t i = a; i < b; ++i)
                if (!r.read_signed(width, out[i])) return 1;
        }
    }
    return 0;
}

// decoder.rs:340-520.  0 ok, 1 decode error, 2 unsupported.
SYMGPU_HD int read_subframe(Reader& r, uint32_t frame_bps, uint32_t n, symgpu_flac_subframe& sf, int32_t* out) {
    uint32_t v;
    if (!r.read(1, v) || v) return 1;
    uint32_t type;
    if (!r.read(6, type)) return 1;
    uint32_t order = 0;
    if (type == 0) sf.type = SYMGPU_FLAC_CONSTANT;
    else if (type == 1) sf.type = SYMGPU_FLAC_VERBATIM;
    else if (type >= 8 && type <= 15) {
        order = type & 7;
        if (order > 4) return 1;
        sf.type = SYMGPU_FLAC_FIXED;
    } else if (type >= 32) {
        order = (type & 31) + 1;
        sf.type = SYMGPU_FLAC_LPC;
    } else return 1;
    uint32_t wasted = 0;
    if (!r.read(1, v)) return 1;
    if (v) {
        if (!r.unary(wasted)) return 1;
        ++wasted;
    }
    if (wasted > frame_bps) return 1;
    const uint32_t bps = frame_bps - wasted;
    if (bps > 32) return 2;  // a 33-bit side channel: the reference's 32-bit reads cannot carry it either
    sf.wasted = uint8_t(wasted), sf.order = uint8_t(order), sf.shift = 0;
    for (uint32_t i = 0; i < n; ++i) out[i] = 0;
    switch (sf.type) {
        case SYMGPU_FLAC_CONSTANT:
            return r.read_signed(bps, out[0]) ? 0 : 1;
        case SYMGPU_FLAC_VERBATIM:
            for (uint32_t i = 0; i < n; ++i)
                if (!r.read_signed(bps, out[i])) return 1;
            return 0;
        case SYMGPU_FLAC_FIXED:
            if (order > n) return 1;
            for (uint32_t i = 0; i < order; ++i)
                if (!r.read_signed(bps, out[i])) return 1;
            return read_residual(r, order, out, n);
        default: {
            if (order > n) return 1;
            for (uint32_t i = 0; i < order; ++i)
                if (!r.read_signed(bps, out[i])) return 1;
            uint32_t precision;
            int32_t shift;
            if (!r.read(4, precision)) return 1;
            if (++precision > 15) return 1;
            if (!r.read_signed(5, shift)) return 1;
            if (shift < 0) return 2;
            sf.shift = uint8_t(shift);
            for (uint32_t j = 0; j < order; ++j)  // coefficient j multiplies the sample j + 1 back (the reference stores them reversed)
                if (!r.read_signed(precision, sf.coeffs[j])) return 1;
            return read_residual(r, order, out, n);
        }
    }
}

// What decode_packet reports for one packet.
enum : int { kDecoded = 0, kRefused = 1, kNoRoom = 2 };

// One packet p[0, len) of a stream whose information block says stream_bps / stream_channels / max_block (0 = unknown).
// The frame's sub-frames go to subs[0 .. channels) -- subs[c].offset = sample_base + c * block -- and their samples to
// samples[c * block .. (c + 1) * block); both are written only within subs_room records, samples_room samples, and for a
// block of at most block_room samples.  On kDecoded *frame (first_subframe = first_subframe) and *info are written.
// kRefused: the reference refuses the packet (the sub-frames read before the error are left as they are).  kNoRoom: the
// header is acceptable but the frame does not fit; nothing has been written.
SYMGPU_HD int decode_packet(const uint8_t* p, size_t len, uint32_t stream_bps, uint32_t stream_channels, uint32_t max_block, uint32_t first_subframe,
                            symgpu_flac_subframe* subs, size_t subs_room, int32_t* samples, uint64_t sample_base, size_t samples_room, uint32_t block_room,
                            symgpu_flac_frame* frame, symgpu_flac_frame_info* info) {
    // frame.rs:66-79: a 14-bit sync code on a byte boundary, searched as 1111 1111 1111 10xx
    size_t at = 0;
    for (;; ++at) {
        if (at + 2 > len) break;
        if (p[at] == 0xff && (p[at + 1] & 0xfc) == 0xf8) break;
    }
    if (at + 2 > len) return kRefused;
    Header h{};
    if (read_header(p, len, at, h)) return kRefused;
    const uint32_t bps = h.bps ? h.bps : stream_bps;
    if (bps == 0 || bps > 32) return kRefused;
    if (max_block && h.block > max_block) return kRefused;
    if (stream_channels && h.channels > stream_channels) return kRefused;
    if (h.channels > subs_room || size_t(h.channels) * h.block > samples_room || h.block > block_room) return kNoRoom;
    Reader r(p + at + h.size, len - at - h.size);
    for (uint32_t c = 0; c < h.channels; ++c) {
        // the difference channel of a decorrelated pair carries one more bit (decoder.rs:193-225)
        const bool side = (h.assignment == SYMGPU_FLAC_LEFT_SIDE && c == 1) || (h.assignment == SYMGPU_FLAC_MID_SIDE && c == 1) ||
                          (h.assignment == SYMGPU_FLAC_RIGHT_SIDE && c == 0);
        symgpu_flac_subframe& sf = subs[c];
        sf = symgpu_flac_subframe{};
        sf.offset = sample_base + uint64_t(c) * h.block, sf.n = h.block;
        if (read_subframe(r, bps + (side ? 1 : 0), h.block, sf, samples + size_t(c) * h.block) != 0) return kRefused;
    }
    *frame = symgpu_flac_frame{};
    frame->first_subframe = first_subframe, frame->channels = uint8_t(h.channels), frame->assignment = h.assignment, frame->bits_per_sample = uint8_t(bps);
    *info = symgpu_flac_frame_info{};
    info->sequence = h.sequence, info->block_size = h.block, info->sample_rate = h.rate, info->by_sample = h.by_sample;
    return kDecoded;
}

}  // namespace flace
}  // namespace symgpu
