// ORACLE (test infrastructure, NOT product code): CPU restatement of the reference's ALAC packet decode, one packet per call.
//
//   map_channels                              symphonia-codec-alac/src/lib.rs:56-68
//   ElementChannel::try_read                  lib.rs:83-110
//   ElementChannel::read_residuals            lib.rs:112-163
//   ElementChannel::predict                   lib.rs:165-264
//   AlacDecoder::decode_inner                 lib.rs:315-418 (buffer cleared to silence, truncated to the last element)
//   decode_sce_or_cpe                         lib.rs:471-603
//   lg3a, read_rice_code, rice_code_to_signed, clip_msbs, decorrelate_mid_side   lib.rs:605-671
//   BitReaderLtr (reads past the end fail; read_unary_ones_capped)               symphonia-core/src/io/bit.rs:500-766
//
// Written in the reference's own order: residuals, then predict (which refuses modes 1..14), then the mid/side step (which
// refuses a shift above 31).  i32 arithmetic that a release build of the reference wraps is done through uint32_t here.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct Bits {  // one bit at a time: the plainest reading of BitReaderLtr
    const uint8_t* p;
    uint64_t n_bits, at = 0;
    bool bit(uint32_t& b) {
        if (at >= n_bits) return false;
        b = (p[at >> 3] >> (7 - (at & 7))) & 1;
        ++at;
        return true;
    }
    bool bits(uint32_t width, uint32_t& v) {
        v = 0;
        for (uint32_t k = 0; k < width; ++k) {
            uint32_t b;
            if (!bit(b)) return false;
            v = (v << 1) | b;
        }
        return true;
    }
    bool sbits(uint32_t width, int32_t& v) {
        uint32_t u;
        if (!bits(width, u)) return false;
        v = width == 0 ? 0 : width == 32 ? int32_t(u) : ((u >> (width - 1)) & 1 ? int32_t(u | (0xffffffffu << width)) : int32_t(u));
        return true;
    }
    bool ones_capped(uint32_t limit, uint32_t& num) {  // bit.rs:738-766
        num = 0;
        while (num < limit) {
            uint32_t b;
            if (!bit(b)) return false;
            if (!b) return true;
            ++num;
        }
        return true;
    }
    void realign() { at = (at + 7) / 8 * 8; }
    bool ignore(uint64_t count) {
        if (count > n_bits - at) return false;
        at += count;
        return true;
    }
};

uint32_t leading_zeros(uint32_t v) {
    uint32_t n = 0;
    for (int k = 31; k >= 0 && !((v >> k) & 1); --k) ++n;
    return n;
}
uint32_t lg3a(uint32_t v) { return 31 - leading_zeros((v >> 9) + 3); }
int32_t clip_msbs(int32_t v, uint32_t num) { return int32_t(uint32_t(v) << num) >> num; }
int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
int32_t wmul(int32_t a, int32_t b) { return int32_t(uint32_t(a) * uint32_t(b)); }

bool read_rice_code(Bits& bs, uint32_t k, uint32_t bps, uint32_t& value) {
    uint32_t prefix;
    if (!bs.ones_capped(9, prefix)) return false;
    if (prefix > 8) return bs.bits(bps, value);
    if (k > 1) {
        value = (prefix << k) - prefix;
        uint32_t suffix;
        if (!bs.bits(k - 1, suffix)) return false;
        if (suffix > 0) {
            uint32_t b;
            if (!bs.bit(b)) return false;
            value = value + (suffix << 1) + b - 1;
        }
        return true;
    }
    value = k == 1 ? prefix : 0;
    return true;
}

struct ElementChannel {
    uint32_t bps, kb, mb, mode, shift, pb_factor, lpc_order;
    int32_t lpc_coeffs[32];
};

bool try_read(Bits& bs, uint32_t pb, uint32_t kb, uint32_t mb, uint32_t bps, ElementChannel& e) {
    uint32_t pbf;
    if (!bs.bits(4, e.mode) || !bs.bits(4, e.shift) || !bs.bits(3, pbf) || !bs.bits(5, e.lpc_order)) return false;
    e.pb_factor = (pbf * pb) >> 2;
    e.bps = bps, e.kb = kb, e.mb = mb;
    std::memset(e.lpc_coeffs, 0, sizeof e.lpc_coeffs);
    for (uint32_t j = 0; j < e.lpc_order; ++j)
        if (!bs.sbits(16, e.lpc_coeffs[j])) return false;
    return true;
}

bool read_residuals(Bits& bs, const ElementChannel& e, int32_t* out, uint32_t out_len) {
    uint32_t mb = e.mb, sign_toggle = 0;
    uint64_t zero_run_end = 0;
    for (uint32_t i = 0; i < out_len; ++i) {
        if (i < zero_run_end) continue;  // the buffer is already silence
        const uint32_t k = lg3a(mb);
        uint32_t val;
        if (!read_rice_code(bs, k < e.kb ? k : e.kb, e.bps, val)) return false;
        val += sign_toggle;
        out[i] = int32_t(val >> 1) ^ -int32_t(val & 1);
        if (val > 0xffff) mb = 0xffff;
        else mb = mb + e.pb_factor * val - ((e.pb_factor * mb) >> 9);
        sign_toggle = 0;
        if (mb < 128 && i + 1 < out_len) {
            const uint32_t kz = leading_zeros(mb) - 24 + ((mb + 16) >> 6);
            uint32_t zeros;
            if (!read_rice_code(bs, kz < e.kb ? kz : e.kb, 16, zeros)) return false;
            if (zeros < 0xffff) sign_toggle = 1;
            mb = 0;
            zero_run_end = uint64_t(i) + 1 + zeros;
        }
    }
    return true;
}

bool predict(ElementChannel& e, int32_t* out, uint32_t len) {
    if (e.mode > 0 && e.mode < 15) return false;
    if (e.lpc_order == 0 || len == 0) return true;
    const uint32_t num_clip_bits = 32 - e.bps;
    if (e.lpc_order == 31 || e.mode == 15)
        for (uint32_t i = 1; i < len; ++i) out[i] = clip_msbs(wadd(out[i], out[i - 1]), num_clip_bits);
    const uint32_t order = e.lpc_order;
    for (uint32_t i = 1; i < (1 + order < len ? 1 + order : len); ++i) out[i] = clip_msbs(wadd(out[i], out[i - 1]), num_clip_bits);
    for (uint32_t i = 1 + order; i < len; ++i) {
        int32_t res = out[i];
        const int32_t past0 = out[i - order - 1];
        int32_t sum = 0;
        for (uint32_t j = 0; j < order; ++j)  // coefficients reversed against out[i - order .. i)
            sum = wadd(sum, wmul(e.lpc_coeffs[order - 1 - j], wsub(out[i - order + j], past0)));
        const int32_t val = wadd(sum, int32_t((1u << e.shift) >> 1)) >> e.shift;
        out[i] = clip_msbs(wadd(wadd(out[i], past0), val), num_clip_bits);
        if (res != 0) {
            for (uint32_t j = 0; j < order; ++j) {
                int32_t& coeff = e.lpc_coeffs[order - 1 - j];
                const int32_t v = wsub(past0, out[i - order + j]);
                const int32_t sign = v > 0 ? 1 : v < 0 ? -1 : 0;
                if (res > 0) {
                    coeff = wsub(coeff, sign);
                    res = wsub(res, wmul(int32_t(1 + j), wmul(sign, v) >> e.shift));
                    if (res <= 0) break;
                } else {
                    coeff = wadd(coeff, sign);
                    res = wsub(res, wmul(int32_t(1 + j), wmul(-sign, v) >> e.shift));
                    if (res >= 0) break;
                }
            }
        }
    }
    return true;
}

const uint8_t kMaps[8][8] = {{0, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 0, 0, 0, 0, 0, 0}, {2, 0, 1, 0, 0, 0, 0, 0}, {2, 0, 1, 3, 0, 0, 0, 0},
                             {2, 0, 1, 3, 4, 0, 0, 0}, {2, 0, 1, 4, 5, 3, 0, 0}, {2, 0, 1, 5, 6, 4, 3, 0}, {2, 4, 5, 0, 1, 6, 7, 3}};

// decode_sce_or_cpe; out1 null for an SCE.  Returns false on the reference's errors.
bool decode_sce_or_cpe(Bits& bs, uint32_t frame_length, uint32_t bit_depth, uint32_t pb, uint32_t mb, uint32_t kb, std::vector<uint16_t>& tail_bits,
                       int32_t* out0, int32_t* out1, uint32_t& num_samples) {
    const bool is_cpe = out1 != nullptr;
    uint32_t v, partial, shift2, uncompressed;
    if (!bs.bits(4, v)) return false;
    if (!bs.bits(12, v) || v != 0) return false;
    if (!bs.bits(1, partial) || !bs.bits(2, shift2) || !bs.bits(1, uncompressed)) return false;
    const uint32_t shift = 8 * shift2;
    if (shift >= 24 || shift >= bit_depth) return false;
    num_samples = frame_length;
    if (partial && !bs.bits(32, num_samples)) return false;
    if (num_samples > frame_length) return false;
    if (!uncompressed) {
        const uint32_t bps = bit_depth - shift + (is_cpe ? 1 : 0);
        if (bps > 32) return false;
        uint32_t mid_side_shift;
        int32_t mid_side_weight;
        if (!bs.bits(8, mid_side_shift) || !bs.sbits(8, mid_side_weight)) return false;
        if (!is_cpe && (mid_side_shift != 0 || mid_side_weight != 0)) return false;
        ElementChannel e0, e1;
        if (!try_read(bs, pb, kb, mb, bps, e0)) return false;
        if (is_cpe && !try_read(bs, pb, kb, mb, bps, e1)) return false;
        if (shift > 0) {
            const uint32_t num_tail = (is_cpe ? 2 : 1) * num_samples;
            for (uint32_t t = 0; t < num_tail; ++t) {
                if (!bs.bits(shift, v)) return false;
                tail_bits[t] = uint16_t(v);
            }
        }
        if (!read_residuals(bs, e0, out0, num_samples) || !predict(e0, out0, num_samples)) return false;
        if (is_cpe) {
            if (!read_residuals(bs, e1, out1, num_samples) || !predict(e1, out1, num_samples)) return false;
            if (mid_side_weight != 0) {
                if (mid_side_shift > 31) return false;
                for (uint32_t t = 0; t < frame_length; ++t) {  // the whole planes, as the reference passes them
                    const int32_t s0 = wsub(wadd(out0[t], out1[t]), wmul(out1[t], mid_side_weight) >> mid_side_shift);
                    out0[t] = s0;
                    out1[t] = wsub(s0, out1[t]);
                }
            }
        }
        if (shift > 0) {
            for (uint32_t t = 0; t < num_samples; ++t) {
                if (is_cpe) {
                    out0[t] = int32_t((uint32_t(out0[t]) << shift) | tail_bits[2 * t]);
                    out1[t] = int32_t((uint32_t(out1[t]) << shift) | tail_bits[2 * t + 1]);
                } else {
                    out0[t] = int32_t((uint32_t(out0[t]) << shift) | tail_bits[t]);
                }
            }
        }
    } else {
        for (uint32_t t = 0; t < num_samples; ++t) {
            if (!bs.sbits(bit_depth, out0[t])) return false;
            if (is_cpe && !bs.sbits(bit_depth, out1[t])) return false;
        }
    }
    return true;
}

}  // namespace

extern "C" {

// One packet with the stream's cookie: planes [channels][frame_length] (each channel's samples from 0; only the first *frames
// are the packet's), *frames the frame count.  0: decoded; 1: the reference refuses the packet.
int oracle_alac_packet(const uint8_t* data, size_t len, uint32_t frame_length, uint32_t bit_depth, uint32_t pb, uint32_t mb, uint32_t kb,
                       uint32_t channels, int32_t* planes, uint32_t* frames) {
    *frames = 0;
    if (channels < 1 || channels > 8) return 1;
    std::fill(planes, planes + size_t(channels) * frame_length, 0);  // render_silence
    std::vector<uint16_t> tail_bits(size_t(channels < 2 ? channels : 2) * frame_length);
    Bits bs{data, uint64_t(len) * 8};
    const uint8_t* map = kMaps[channels - 1];
    uint32_t next_channel = 0, num_frames = 0;
    for (;;) {
        uint32_t tag;
        if (!bs.bits(3, tag)) return 1;
        if (tag == 0 || tag == 3) {
            if (!decode_sce_or_cpe(bs, frame_length, bit_depth, pb, mb, kb, tail_bits, planes + size_t(map[next_channel]) * frame_length, nullptr,
                                   num_frames))
                return 1;
            next_channel += 1;
        } else if (tag == 1) {
            if (next_channel + 2 > channels) break;
            if (!decode_sce_or_cpe(bs, frame_length, bit_depth, pb, mb, kb, tail_bits, planes + size_t(map[next_channel]) * frame_length,
                                   planes + size_t(map[next_channel + 1]) * frame_length, num_frames))
                return 1;
            next_channel += 2;
        } else if (tag == 4) {
            uint32_t t, align, count, more;
            if (!bs.bits(4, t) || !bs.bits(1, align) || !bs.bits(8, count)) return 1;
            if (count == 255) {
                if (!bs.bits(8, more)) return 1;
                count += more;
            }
            if (align) bs.realign();
            if (!bs.ignore(uint64_t(8) * count)) return 1;
        } else if (tag == 6) {
            uint32_t count, more;
            if (!bs.bits(4, count)) return 1;
            if (count == 15) {
                if (!bs.bits(8, more)) return 1;
                count = count + more - 1;
            }
            if (!bs.ignore(uint64_t(8) * count)) return 1;
        } else if (tag == 2 || tag == 5) {
            return 1;
        } else {
            break;
        }
        if (next_channel >= channels) break;
    }
    *frames = num_frames;
    const uint32_t shift = 32 - bit_depth;
    if (shift > 0 && shift < 32)
        for (size_t k = 0; k < size_t(channels) * frame_length; ++k) planes[k] = int32_t(uint32_t(planes[k]) << shift);
    return 0;
}

}  // extern "C"
