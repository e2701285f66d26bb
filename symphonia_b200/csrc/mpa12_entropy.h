// MPEG Layer I / II bitstream rules of ONE packet -- header, side information (bit allocation, scale-factor selection,
// scale factors) and the sample codewords -- written once for host and device.  The CPU front-end (mpa12_frontend.cpp)
// calls these functions frame after frame; the device path (mpa12_decode_kernel.cu) calls the SAME functions, the side
// read with one thread per packet and the codewords with many lanes per frame.
//
// Why the codewords can be decoded in parallel: once the side information is read, every codeword's width is known, and
// the samples of a frame are laid out granule by granule (Layer I: 12 time slots, Layer II: 12 granules of three samples),
// each granule holding the same codewords in the same order.  So the codeword of (granule gr, sub-band sb, channel ch)
// starts at  sample_start + gr * G + prefix(sb, ch),  G = the bits of one granule.  Layer I / II has no bit reservoir,
// and a frame depends on the stream only through the synthesis state and the signal specification.
//
// Reference: Layer1::decode (symphonia-bundle-mp3/src/layer1/mod.rs:73-176), Layer2::decode (layer2/mod.rs:136-369),
// scale factors layer12.rs:9-75, the decoder's packet handling decoder.rs:87-128.
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu/packetizer.hpp"
#include "mp3_entropy.h"

namespace symgpu {
namespace mpa12e {

using symgpu::mp3e::Bits;
using symgpu::packet::MpaHeader;
using symgpu::packet::MpaMode;
using symgpu::packet::MpaVersion;

struct QuantClass {
    float c, d;
    float inv_divisor;  // 2^-(bits - 1), exact
    uint8_t read_bits;  // width of one sample, or of the codeword holding three
    uint8_t bits;       // width of one sample after degrouping
    uint16_t levels;
    bool grouped;
};

// The decoders' constants.  Computed once on the host with libm (mpa12_frontend.cpp, host_constants()); the device receives
// these values and never recomputes them (the device's pow is not the host's).
struct Constants {
    float scale[64];
    float factor[16];       // Layer I
    QuantClass cls[17];     // by class: 3, 5, 7, 9, 15, 31, ... 65535 levels
};
const Constants& host_constants();  // host only

// The packet prologue is shared with Layer III (mp3_entropy.h).
using symgpu::mp3e::body_of;
using symgpu::mp3e::kDecoded;
using symgpu::mp3e::kRefused;
using symgpu::mp3e::kUnsupported;
using symgpu::mp3e::read_header;

// What the side read leaves for the sample codewords of one frame.  404 bytes.
struct Side {
    uint32_t body_at;        // byte offset of the body (after the header word and the CRC) in the packet
    uint32_t body_bytes;
    uint32_t sample_start;   // bit offset, in the body, of the first sample codeword
    uint32_t granule_bits;   // G: the bits of one granule (Layer I: one time slot of all sub-bands)
    uint8_t layer, n_ch, bound, sblimit;
    uint8_t q[2][32];        // Layer I: bits per sample; Layer II: quantisation class + 1; 0: nothing allocated.  Above the
                             // bound q[1] = q[0]: both channels take channel 0's codeword.
    uint8_t sf[2][3][32];    // scale-factor indices (Layer I: part 0 only)
    uint16_t prefix[2][32];  // bit offset of the (sb, ch) codeword inside a granule; above the bound prefix[1] = prefix[0]
};

// Allocation tables (ISO 11172-3 Tables 3-B.2a-d, 13818-3 Table B.1) as the standard lays them out: a sub-band's row is
// the list of quantiser sizes its allocation index selects (index 0: nothing allocated).
SYMGPU_HD unsigned row_nbal(int row) { return row < 2 ? 2u : row < 4 ? 3u : 4u; }
SYMGPU_HD unsigned row_levels(int row, unsigned index) {
    static constexpr uint16_t rows[8][16] = {
        {0, 3, 5, 65535},
        {0, 3, 5, 9},
        {0, 3, 5, 9, 15, 31, 63, 127},
        {0, 3, 5, 7, 9, 15, 31, 65535},
        {0, 3, 5, 7, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383},
        {0, 3, 5, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383, 32767},
        {0, 3, 5, 7, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 65535},
        {0, 3, 7, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383, 32767, 65535},
    };
    return rows[row][index];
}
// Table t's sblimit and the row of sub-band sb (sb < sblimit), as (sub-bands, row) runs.
SYMGPU_HD unsigned table_sblimit(int t) {
    static constexpr uint8_t sblimit[5] = {27, 30, 8, 12, 30};
    return sblimit[t];
}
SYMGPU_HD int table_row(int t, int sb) {
    static constexpr uint8_t runs[5][4][2] = {
        {{3, 7}, {8, 6}, {12, 3}, {4, 0}},   // 3-B.2a
        {{3, 7}, {8, 6}, {12, 3}, {7, 0}},   // 3-B.2b
        {{2, 5}, {6, 2}, {0, 0}, {0, 0}},    // 3-B.2c
        {{2, 5}, {10, 2}, {0, 0}, {0, 0}},   // 3-B.2d
        {{4, 4}, {7, 2}, {19, 1}, {0, 0}},   // 13818-3 B.1 (MPEG-2 / 2.5)
    };
    int r = 0;
    while (sb >= runs[t][r][0]) sb -= runs[t][r][0], ++r;
    return runs[t][r][1];
}
SYMGPU_HD int class_of(unsigned levels) {  // 3 5 7 9 -> 0..3, 2^k - 1 -> k
    if (levels <= 9) return int(levels - 3) / 2;
    int k = 0;
    while ((1u << k) <= levels) ++k;
    return k;
}

// layer2/mod.rs:136-166
SYMGPU_HD int table_of(const MpaHeader& h) {
    if (h.version != MpaVersion::Mpeg1) return 4;
    const uint32_t per_channel = h.bitrate / uint32_t(h.n_channels());
    if (per_channel <= 48000) return h.sample_rate == 32000 ? 3 : 2;
    if (per_channel <= 80000) return 0;
    return h.sample_rate != 48000 ? 1 : 0;
}

SYMGPU_HD int32_t centre(uint32_t raw, unsigned bits) {  // invert the top bit, sign-extend: offset binary -> two's complement
    const uint32_t inv = raw ^ (1u << (bits - 1));
    return int32_t(inv << (32 - bits)) >> (32 - bits);
}

// ---- side read ---------------------------------------------------------------------------------------------------------
// Reads allocation, scale-factor selection and scale factors from `body` (s.body_bytes long) exactly as the reference reads
// them, and fills s's codeword layout.  false where a read fails or Layer I allocation 15 appears.
SYMGPU_HD bool read_layer1_side(const uint8_t* body, const MpaHeader& h, Side& s) {
    Bits bs(body, s.body_bytes);
    const int n_ch = h.n_channels(), bound = h.mode == MpaMode::JointStereo ? h.bound : 32;
    s.n_ch = uint8_t(n_ch), s.bound = uint8_t(bound), s.sblimit = 32;
    uint32_t v;
    for (int sb = 0; sb < 32; ++sb) {
        const int readers = sb < bound ? n_ch : 1;
        for (int ch = 0; ch < readers; ++ch) {
            if (!bs.read(4, v) || v > 14) return false;
            s.q[ch][sb] = uint8_t(v ? v + 1 : 0);
        }
        if (sb >= bound) s.q[1][sb] = s.q[0][sb];
    }
    for (int sb = 0; sb < 32; ++sb)
        for (int ch = 0; ch < n_ch; ++ch)
            if (s.q[ch][sb]) {
                if (!bs.read(6, v)) return false;
                s.sf[ch][0][sb] = uint8_t(v);
            }
    uint32_t g = 0;
    for (int sb = 0; sb < 32; ++sb) {
        const int readers = sb < bound ? n_ch : 1;
        for (int ch = 0; ch < readers; ++ch) s.prefix[ch][sb] = uint16_t(g), g += s.q[ch][sb];
        if (sb >= bound) s.prefix[1][sb] = s.prefix[0][sb];
    }
    s.sample_start = uint32_t(bs.at), s.granule_bits = g;
    return true;
}

SYMGPU_HD bool read_layer2_side(const Constants& K, const uint8_t* body, const MpaHeader& h, Side& s) {
    Bits bs(body, s.body_bytes);
    const int t = table_of(h);
    const int n_ch = h.n_channels(), sblimit = int(table_sblimit(t));
    const int bound = (h.mode == MpaMode::JointStereo ? h.bound : 32) < sblimit ? (h.mode == MpaMode::JointStereo ? h.bound : 32) : sblimit;
    s.n_ch = uint8_t(n_ch), s.bound = uint8_t(bound), s.sblimit = uint8_t(sblimit);
    uint8_t alloc[2][32] = {}, scfsi[2][32] = {};
    uint32_t v;
    for (int sb = 0; sb < sblimit; ++sb) {
        const int row = table_row(t, sb), readers = sb < bound ? n_ch : 1;
        for (int ch = 0; ch < readers; ++ch) {
            if (!bs.read(row_nbal(row), v)) return false;
            alloc[ch][sb] = uint8_t(v);
            s.q[ch][sb] = uint8_t(v ? class_of(row_levels(row, v)) + 1 : 0);
        }
        if (sb >= bound) alloc[1][sb] = alloc[0][sb], s.q[1][sb] = s.q[0][sb];
    }
    for (int sb = 0; sb < sblimit; ++sb)
        for (int ch = 0; ch < n_ch; ++ch)
            if (alloc[ch][sb]) {
                if (!bs.read(2, v)) return false;
                scfsi[ch][sb] = uint8_t(v);
            }
    for (int sb = 0; sb < sblimit; ++sb)
        for (int ch = 0; ch < n_ch; ++ch)
            if (alloc[ch][sb]) {
                uint32_t a, b, c;
                if (!bs.read(6, a)) return false;
                b = c = a;
                switch (scfsi[ch][sb]) {  // which of the three parts share a scale factor (ISO 11172-3 2.4.2.5)
                    case 0:
                        if (!bs.read(6, b) || !bs.read(6, c)) return false;
                        break;
                    case 1:
                        if (!bs.read(6, c)) return false;
                        break;
                    case 2: break;
                    default:
                        if (!bs.read(6, b)) return false;
                        c = b;
                }
                s.sf[ch][0][sb] = uint8_t(a), s.sf[ch][1][sb] = uint8_t(b), s.sf[ch][2][sb] = uint8_t(c);
            }
    uint32_t g = 0;
    for (int sb = 0; sb < sblimit; ++sb) {
        const int readers = sb < bound ? n_ch : 1;
        for (int ch = 0; ch < readers; ++ch) {
            s.prefix[ch][sb] = uint16_t(g);
            if (s.q[ch][sb]) {
                const QuantClass& qc = K.cls[s.q[ch][sb] - 1];
                g += qc.grouped ? qc.read_bits : 3u * qc.read_bits;
            }
        }
        if (sb >= bound) s.prefix[1][sb] = s.prefix[0][sb];
    }
    s.sample_start = uint32_t(bs.at), s.granule_bits = g;
    return true;
}

// The side read of a packet that passed the prologue (body = the packet + s.body_at).  Zeroes the record first.
SYMGPU_HD bool read_side(const Constants& K, const uint8_t* body, const MpaHeader& h, Side& s) {
    const uint32_t at = s.body_at, bytes = s.body_bytes;
    s = Side{};
    s.body_at = at, s.body_bytes = bytes, s.layer = h.layer;
    return h.layer == 1 ? read_layer1_side(body, h, s) : read_layer2_side(K, body, h, s);
}

// ---- fit rule ----------------------------------------------------------------------------------------------------------
// The reference reads the 12 granules' codewords one after another and refuses the frame when a read runs past the body.
// Reads are sequential and each starts where the previous ended, so the end of the last read, sample_start + 12 G, is the
// furthest bit any read reaches: "some read fails" holds exactly when sample_start + 12 G > the body's bits.  (With G = 0
// there is no read, and the side read already ended inside the body.)
SYMGPU_HD bool fits(const Side& s) { return uint64_t(s.sample_start) + 12ull * s.granule_bits <= uint64_t(s.body_bytes) * 8; }

// ---- one sample codeword -----------------------------------------------------------------------------------------------
// The samples of (granule gr, sub-band sb) of output channel c: Layer I one value, Layer II three, written to out[0 ..].
// Above the joint-stereo bound the codeword is channel 0's, scaled by channel c's own scale factor.  The arithmetic is the
// reference's, operation for operation; false where the read runs past the body (never after fits()).  Nothing allocated:
// zeros.
SYMGPU_HD bool decode_codeword(const Constants& K, const Side& s, const uint8_t* body, int gr, int sb, int c, float* out) {
    const int rc = sb < s.bound ? c : 0;
    const unsigned q = s.q[rc][sb];
    if (s.layer == 1) {
        if (!q) return out[0] = 0.0f, true;
        Bits bs(body, s.body_bytes, size_t(s.sample_start) + size_t(gr) * s.granule_bits + s.prefix[rc][sb]);
        uint32_t v;
        if (!bs.read(q, v)) return false;
        const float sample = K.factor[q] * float(centre(v, q) + 1);
        out[0] = K.scale[s.sf[c][0][sb]] * sample;
        return true;
    }
    if (!q) return out[0] = out[1] = out[2] = 0.0f, true;
    const QuantClass& qc = K.cls[q - 1];
    Bits bs(body, s.body_bytes, size_t(s.sample_start) + size_t(gr) * s.granule_bits + s.prefix[rc][sb]);
    uint32_t raw[3], v;
    if (qc.grouped) {
        if (!bs.read(qc.read_bits, v)) return false;
        for (int k = 0; k < 3; ++k) raw[k] = v % qc.levels, v /= qc.levels;
    } else {
        for (int k = 0; k < 3; ++k)
            if (!bs.read(qc.read_bits, raw[k])) return false;
    }
    // The reference divides by 2^(bits - 1).  A centred sample has at most 16 significant bits, so that quotient is exact, and
    // so is the product with the exact reciprocal: the two are the same float.  The product is what is computed here, because
    // the device's correctly rounded division is a sequence of fused multiply-adds.
    const float scale = K.scale[s.sf[c][gr / 4][sb]];
    for (int k = 0; k < 3; ++k) {
        const float x = qc.c * (float(centre(raw[k], qc.bits)) * qc.inv_divisor + qc.d);
        out[k] = scale * x;
    }
    return true;
}

}  // namespace mpa12e
}  // namespace symgpu
