// ALAC decoding of ONE packet, written once for host and device: the element loop with its channel headers, tail bits and
// adaptive Golomb residuals (decode_packet), the adaptive predictor of one channel (predict_channel) and the per-sample
// finish -- mid/side, tail-bit splice, the scale to 32 bits (finish_sample).  The CPU front-end (alac_frontend.cpp,
// symgpu_alac_fe_decode_packets) runs the three steps packet after packet; the device path (alac_decode_kernel.cu) runs
// decode_packet with one thread per packet, predict_channel with one thread per decoded channel and finish_sample across a
// CTA per packet.  An ALAC packet carries no state into the next one (AlacDecoder::reset does nothing), so a packet is an
// independent job, and every CPU test of the front-end is a test of the code the kernels run.
//
// Reference (symphonia-codec-alac/src/lib.rs): map_channels :56-68, ElementChannel::try_read / read_residuals / predict
// :82-264, AlacDecoder::decode_inner :315-418, decode_sce_or_cpe :471-603, lg3a / read_rice_code / rice_code_to_signed /
// clip_msbs / decorrelate_mid_side :605-671.
//
// Every refusal of the reference refuses the whole packet, so where it is found does not matter: decode_packet finds them
// all, including the two the reference only meets later (a mode of 1 to 14 in predict, a mid/side shift above 31 before the
// decorrelation), and the predictor and the finish cannot fail.  The reference's release build wraps on signed overflow;
// here that arithmetic is done on uint32_t, and every left shift is of an unsigned value.
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu.h"
#include "mp3_entropy.h"  // Bits, SYMGPU_HD, SYMGPU_UNROLL

namespace symgpu {
namespace alac {

using mp3e::Bits;

// What decode_packet reports for one packet (the values of SYMGPU_FLAC_JOB_*).
enum : int { kDecoded = 0, kRefused = 1, kNoRoom = 2 };

enum : uint8_t { kNone = 0, kCompressed = 1, kUncompressed = 2 };
enum : uint8_t { kSce = 0, kFirst = 1, kSecond = 2 };

// One output channel of one packet, as its element left it.
struct Channel {             // 80 bytes
    uint32_t n;              // samples its element decoded; 0: no element wrote it (silence)
    uint8_t kind;            // kNone / kCompressed / kUncompressed
    uint8_t mode, order;     // predictor mode (0 or 15) and order
    uint8_t shift;           // predictor shift
    uint8_t bps;             // bits per coded sample: the predictor clips to it
    uint8_t tail;            // tail bits spliced under each sample: 0, 8 or 16
    uint8_t role;            // kSce, or which channel of a CPE it is
    uint8_t partner;         // the other channel of its CPE
    uint8_t ms_shift;
    int8_t ms_weight;
    uint8_t reserved[2];
    int16_t coeffs[32];      // as read; predict_channel adapts a copy
};
static_assert(sizeof(Channel) == 80, "Channel layout");

SYMGPU_HD uint32_t clz32(uint32_t w) {  // 32 at 0, where Rust's leading_zeros is defined and the builtin is not
#ifdef __CUDA_ARCH__
    return uint32_t(__clz(w));
#else
    return w ? uint32_t(__builtin_clz(w)) : 32u;
#endif
}

// map_channels (lib.rs:56-68): the output channel of each ALAC channel, for the one layout each channel count has (the
// magic cookie's layout tag must agree with its channel count, alac.rs:128-134).  Packed one nibble per channel.
SYMGPU_HD uint32_t channel_of(uint32_t channels, uint32_t k) {
    const uint32_t maps[8] = {0x00000000u, 0x00000010u, 0x00000102u, 0x00003102u, 0x00043102u, 0x00354102u, 0x03465102u, 0x37610542u};
    return (maps[(channels - 1) & 7] >> (4 * k)) & 15;
}

SYMGPU_HD int32_t sign_extend(uint32_t v, unsigned bits) { return bits ? int32_t(v << (32 - bits)) >> (32 - bits) : 0; }
SYMGPU_HD int32_t clip_msbs(uint32_t v, unsigned num) { return int32_t(v << num) >> num; }  // num <= 31
SYMGPU_HD uint32_t lg3a(uint32_t mb) { return 31 - clz32((mb >> 9) + 3); }

struct Reader {  // the reference's BitReaderLtr reads: up to 32 bits, signed, capped unary ones, a byte realignment
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
    // read_unary_ones_capped(9) (bit.rs:738-766): ones up to the first zero, which is consumed, or 9 ones, after which
    // nothing more is; running out of bits first is an error.  The window pads with zeros, so a one is always a real bit.
    SYMGPU_HD bool ones9(uint32_t& ones) {
        const uint32_t lead = clz32(~b.window());
        if (lead >= 9) {
            ones = 9, b.at += 9;
            return true;
        }
        if (size_t(lead) + 1 > b.left()) return false;
        ones = lead, b.at += lead + 1;
        return true;
    }
    SYMGPU_HD void realign() { b.at = (b.at + 7) & ~size_t(7); }  // the packet's bits start on a byte, so this never passes its end
};

// read_rice_code (lib.rs:611-647).
SYMGPU_HD bool read_rice(Reader& r, uint32_t k, uint32_t bps, uint32_t& value) {
    uint32_t prefix;
    if (!r.ones9(prefix)) return false;
    if (prefix > 8) return r.read(bps, value);
    if (k > 1) {
        value = (prefix << k) - prefix;
        uint32_t suffix;
        if (!r.read(k - 1, suffix)) return false;
        if (suffix > 0) {
            uint32_t bit;
            if (!r.read(1, bit)) return false;
            value = value + (suffix << 1) + bit - 1;
        }
        return true;
    }
    value = k == 1 ? prefix : 0;
    return true;
}

// ElementChannel::read_residuals (lib.rs:112-163) into out[0, n): zero runs are written as zeros, since the scratch plane is
// not cleared beforehand as the reference's buffer is.
SYMGPU_HD bool read_residuals(Reader& r, uint32_t mb0, uint32_t kb, uint32_t bps, uint32_t pb_factor, int32_t* out, uint32_t n) {
    uint32_t mb = mb0, sign_toggle = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t k = lg3a(mb);
        uint32_t val;
        if (!read_rice(r, k < kb ? k : kb, bps, val)) return false;
        val += sign_toggle;
        out[i] = int32_t(val >> 1) ^ -int32_t(val & 1);
        if (val > 0xffff) mb = 0xffff;
        else mb = mb + pb_factor * val - ((pb_factor * mb) >> 9);
        sign_toggle = 0;
        if (mb < 128 && i + 1 < n) {
            const uint32_t kz = clz32(mb) - 24 + ((mb + 16) >> 6);
            uint32_t zeros;
            if (!read_rice(r, kz < kb ? kz : kb, 16, zeros)) return false;
            if (zeros < 0xffff) sign_toggle = 1;
            mb = 0;
            const uint32_t end = (i + 1 + zeros) < n ? i + 1 + zeros : n;  // zeros <= 0xffff, n <= 65536: no wrap
            for (uint32_t t = i + 1; t < end; ++t) out[t] = 0;
            i = end - 1;
        }
    }
    return true;
}

// ElementChannel::try_read (lib.rs:83-110), with predict's mode rule (lib.rs:167-169) applied at once.
SYMGPU_HD bool read_channel_header(Reader& r, uint32_t pb, Channel& c, uint32_t& pb_factor) {
    uint32_t mode, shift, pbf, order;
    if (!r.read(4, mode) || !r.read(4, shift) || !r.read(3, pbf) || !r.read(5, order)) return false;
    if (mode > 0 && mode < 15) return false;
    pb_factor = (pbf * pb) >> 2;
    c.mode = uint8_t(mode), c.shift = uint8_t(shift), c.order = uint8_t(order);
    for (uint32_t j = 0; j < 32; ++j) c.coeffs[j] = 0;
    for (uint32_t j = 0; j < order; ++j) {
        int32_t v;
        if (!r.read_signed(16, v)) return false;
        c.coeffs[j] = int16_t(v);
    }
    return true;
}

// What the magic cookie fixes for a stream (symgpu_alac_group without its placement).
struct Config {
    uint32_t frame_length, bit_depth, pb, mb, kb, channels;
};

// decode_sce_or_cpe (lib.rs:471-603) for output channels a (and b for a CPE): headers, tail bits, residuals (or the
// uncompressed samples) into planes + a * slot / b * slot and tails likewise.  Returns kDecoded with *n, kRefused or kNoRoom.
SYMGPU_HD int decode_element(Reader& r, const Config& cfg, bool cpe, uint32_t a, uint32_t b, Channel* recs, int32_t* planes, uint16_t* tails,
                             uint32_t slot, uint32_t& n) {
    uint32_t v, partial, shift_code, uncompressed;
    if (!r.read(4, v) || !r.read(12, v) || v != 0) return kRefused;
    if (!r.read(1, partial) || !r.read(2, shift_code) || !r.read(1, uncompressed)) return kRefused;
    const uint32_t shift = 8 * shift_code;
    if (shift >= 24 || shift >= cfg.bit_depth) return kRefused;
    n = cfg.frame_length;
    if (partial && !r.read(32, n)) return kRefused;
    if (n > cfg.frame_length) return kRefused;
    if (n > slot) return kNoRoom;
    Channel& c0 = recs[a];
    Channel& c1 = recs[b];
    int32_t* out0 = planes + size_t(a) * slot;
    int32_t* out1 = planes + size_t(b) * slot;
    c0 = Channel{};
    c0.n = n, c0.role = cpe ? kFirst : kSce, c0.partner = uint8_t(b);
    if (cpe) c1 = Channel{}, c1.n = n, c1.role = kSecond, c1.partner = uint8_t(a);
    if (uncompressed) {
        c0.kind = kUncompressed;
        if (cpe) c1.kind = kUncompressed;
        for (uint32_t i = 0; i < n; ++i) {
            if (!r.read_signed(cfg.bit_depth, out0[i])) return kRefused;
            if (cpe && !r.read_signed(cfg.bit_depth, out1[i])) return kRefused;
        }
        return kDecoded;
    }
    const uint32_t bps = cfg.bit_depth - shift + (cpe ? 1 : 0);
    if (bps > 32) return kRefused;
    uint32_t ms_shift;
    int32_t ms_weight;
    if (!r.read(8, ms_shift) || !r.read_signed(8, ms_weight)) return kRefused;
    if (!cpe && (ms_shift != 0 || ms_weight != 0)) return kRefused;
    uint32_t pbf0, pbf1 = 0;
    if (!read_channel_header(r, cfg.pb, c0, pbf0)) return kRefused;
    if (cpe && !read_channel_header(r, cfg.pb, c1, pbf1)) return kRefused;
    if (cpe && ms_weight != 0 && ms_shift > 31) return kRefused;  // lib.rs:552-557
    c0.kind = kCompressed, c0.bps = uint8_t(bps), c0.tail = uint8_t(shift), c0.ms_shift = uint8_t(ms_shift), c0.ms_weight = int8_t(ms_weight);
    if (cpe) c1.kind = kCompressed, c1.bps = uint8_t(bps), c1.tail = uint8_t(shift), c1.ms_shift = uint8_t(ms_shift), c1.ms_weight = int8_t(ms_weight);
    if (shift > 0) {  // interleaved for a CPE
        uint16_t* t0 = tails + size_t(a) * slot;
        uint16_t* t1 = tails + size_t(b) * slot;
        for (uint32_t i = 0; i < n; ++i) {
            if (!r.read(shift, v)) return kRefused;
            t0[i] = uint16_t(v);
            if (cpe) {
                if (!r.read(shift, v)) return kRefused;
                t1[i] = uint16_t(v);
            }
        }
    }
    if (!read_residuals(r, cfg.mb, cfg.kb, bps, pbf0, out0, n)) return kRefused;
    if (cpe && !read_residuals(r, cfg.mb, cfg.kb, bps, pbf1, out1, n)) return kRefused;
    return kDecoded;
}

// decode_inner (lib.rs:315-418) up to the prediction: recs[0, channels) and the planes / tails of [channels][slot] samples.
// On kDecoded *frames is the num_samples of the last element decoded (0 when none was); a channel no element wrote keeps
// n = 0.  kRefused: the reference refuses the packet.  kNoRoom: an element has more samples than the slot.
SYMGPU_HD int decode_packet(const uint8_t* p, size_t len, const Config& cfg, Channel* recs, int32_t* planes, uint16_t* tails, uint32_t slot,
                            uint32_t* frames) {
    for (uint32_t c = 0; c < cfg.channels; ++c) recs[c] = Channel{};
    Reader r(p, len);
    uint32_t next = 0, n_frames = 0;
    for (;;) {
        uint32_t tag;
        if (!r.read(3, tag)) return kRefused;
        if (tag == 0 || tag == 3 || tag == 1) {  // SCE, LFE, CPE
            const bool cpe = tag == 1;
            if (cpe && next + 2 > cfg.channels) break;
            const uint32_t a = channel_of(cfg.channels, next), b = cpe ? channel_of(cfg.channels, next + 1) : a;
            uint32_t n = 0;
            const int e = decode_element(r, cfg, cpe, a, b, recs, planes, tails, slot, n);
            if (e != kDecoded) return e;
            n_frames = n;
            next += cpe ? 2 : 1;
        } else if (tag == 4) {  // DSE
            uint32_t t, align, count, more;
            if (!r.read(4, t) || !r.read(1, align) || !r.read(8, count)) return kRefused;
            if (count == 255) {
                if (!r.read(8, more)) return kRefused;
                count += more;
            }
            if (align) r.realign();
            if (!r.b.skip(size_t(8) * count)) return kRefused;
        } else if (tag == 6) {  // FIL
            uint32_t count, more;
            if (!r.read(4, count)) return kRefused;
            if (count == 15) {
                if (!r.read(8, more)) return kRefused;
                count = count + more - 1;
            }
            if (!r.b.skip(size_t(8) * count)) return kRefused;
        } else if (tag == 7) {  // END
            break;
        } else {  // CCE, PCE
            return kRefused;
        }
        if (next >= cfg.channels) break;
    }
    *frames = n_frames;
    return kDecoded;
}

// ElementChannel::predict (lib.rs:165-264) over out[0, c.n).  The coefficients are kept most-distant-sample first (w[j]
// multiplies out[i - order + j]), which is the order both the filter and the adaptation walk them in, so with the loops
// unrolled every index into w is a constant and w stays in registers.
SYMGPU_HD void predict_channel(const Channel& c, int32_t* out) {
    if (c.kind != kCompressed || c.order == 0 || c.n == 0) return;
    const uint32_t n = c.n, order = c.order, shift = c.shift, clip = 32 - c.bps;
    if (order == 31 || c.mode == 15)
        for (uint32_t i = 1; i < n; ++i) out[i] = clip_msbs(uint32_t(out[i]) + uint32_t(out[i - 1]), clip);
    const uint32_t warm = 1 + order < n ? 1 + order : n;
    for (uint32_t i = 1; i < warm; ++i) out[i] = clip_msbs(uint32_t(out[i]) + uint32_t(out[i - 1]), clip);
    int32_t w[32];
SYMGPU_UNROLL
    for (uint32_t j = 0; j < 32; ++j) w[j] = j < order ? int32_t(c.coeffs[order - 1 - j]) : 0;
    const uint32_t round = (1u << shift) >> 1;
    for (uint32_t i = 1 + order; i < n; ++i) {
        const int32_t* h = out + (i - order);
        int32_t res = out[i];
        const int32_t past0 = out[i - order - 1];
        uint32_t sum = 0;
SYMGPU_UNROLL
        for (uint32_t j = 0; j < 32; ++j)
            if (j < order) sum += uint32_t(w[j]) * (uint32_t(h[j]) - uint32_t(past0));
        const int32_t val = int32_t(sum + round) >> shift;
        out[i] = clip_msbs(uint32_t(out[i]) + uint32_t(past0) + uint32_t(val), clip);
        if (res != 0) {
            const bool positive = res > 0;
            bool done = false;
SYMGPU_UNROLL
            for (uint32_t j = 0; j < 32; ++j) {
                if (j < order && !done) {
                    const int32_t d = int32_t(uint32_t(past0) - uint32_t(h[j]));
                    const int32_t sign = (d > 0) - (d < 0);
                    const int32_t s = positive ? sign : -sign;
                    w[j] = int32_t(uint32_t(w[j]) - uint32_t(s));
                    const int32_t mag = int32_t(uint32_t(s) * uint32_t(d)) >> shift;
                    res = int32_t(uint32_t(res) - (j + 1) * uint32_t(mag));
                    done = positive ? res <= 0 : res >= 0;
                }
            }
        }
    }
}

// Sample t of output channel c after decode_packet and predict_channel: decorrelate_mid_side for a CPE with a non-zero weight
// (lib.rs:663-671; one sample of it needs only the pair's two samples at t), the tail-bit splice (lib.rs:563-585) and the
// final shift to 32 bits (lib.rs:409-415).  A sample past the channel's element is the reference's silence.
SYMGPU_HD int32_t finish_sample(const Channel& c, const int32_t* own, const int32_t* other, const uint16_t* tail, uint32_t t, uint32_t bit_depth) {
    if (t >= c.n) return 0;
    uint32_t v = uint32_t(own[t]);
    if (c.kind == kCompressed) {
        if (c.role != kSce && c.ms_weight != 0) {
            const uint32_t s0 = c.role == kFirst ? v : uint32_t(other[t]), s1 = c.role == kFirst ? uint32_t(other[t]) : v;
            const uint32_t mid = s0 + s1 - uint32_t(int32_t(s1 * uint32_t(int32_t(c.ms_weight))) >> c.ms_shift);
            v = c.role == kFirst ? mid : mid - s1;
        }
        if (c.tail) v = (v << c.tail) | tail[t];
    }
    return int32_t(v << ((32 - bit_depth) & 31));
}

}  // namespace alac
}  // namespace symgpu
