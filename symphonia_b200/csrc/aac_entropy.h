// AAC-LC packet rules of ONE raw_data_block, written once for host and device: the element loop, set_pair, ics_info,
// sections, scale factors, pulse / TNS / gain-control reads, the spectrum (books 1-11, escapes, noise), common-window joint
// stereo and the line ranges of the TNS filters.  The CPU front-end (aac_frontend.cpp) keeps one state per stream and calls
// these functions packet after packet; the device decoder (aac_decode_kernel.cu) decodes every packet from a fresh state
// (decode_job) and then chains the state that carries between packets (walk_step).  The front-end's CPU tests run every rule
// of the packet; tests/cpp/aac_entropy_driver.cpp runs decode_job and walk_step in the device's schedule on the CPU.
//
// What carries from one raw_data_block to the next (aac/mod.rs, ics/mod.rs): the element layout (set_pair), one noise
// generator per element, each channel's window shape, and -- read only by a pulse in a band no section coded -- the scale
// factors an earlier block left behind.  Noise draws change values, never control flow, and a generator jumps ahead in
// O(log n); so a packet decoded from a fresh state records its set_pair attempts, draws, window-shape writes and group-0
// scale-factor writes, and walk_step turns those records, in stream order, into what the packet does in context.
//
// Pulse::synth (pulse.rs:60-105) calls powf, which the device cannot reproduce bit for bit (glibc's powf is not correctly
// rounded): pulse_lines (shared) finds the lines a pulse touches, pulse_apply (host only) computes their new values.
//
// Floating point: single IEEE operations in the reference's order; host code is compiled with -ffp-contract=off, device code
// with -fmad=false.  No libm call is made in device code: TNS reads sin() from tns_sin, noise scaling uses sqrt_rn / div_rn.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu.h"
#include "mp3_entropy.h"  // SYMGPU_HD and the bit reader: a failed read fails the packet, the window pads with zeros

namespace symgpu {
namespace aace {

using Bits = mp3e::Bits;

constexpr uint32_t kLcgSeed = 0x1f2e3d4c;  // common.rs:96-111
enum : uint8_t { ZERO_HCB = 0, RESERVED_HCB = 12, NOISE_HCB = 13, INTENSITY_HCB2 = 14, INTENSITY_HCB = 15 };

// A Huffman book as flat arrays: the next 10 bits -> value << 5 | length for codes of <= 10 bits (0 for longer ones), and the
// binary tree over the (length, code) list: pairs of children for bit 0 / bit 1, >= 0 inner node index, < 0 ~value.
struct Book {
    uint16_t lut[1024];
    int32_t node[2 * 289];
    uint32_t max_len;
};

// Everything the packet rules read, built once on the host (aac_tables_host) and copied to the device as it is.
struct Tables {
    Book book[12];                                       // spectrum books 1..11 at [0..10], scale factors at [11]
    float pow43[8192], normal_scf[256], intensity_scf[256];
    float tns_sin[2][16];                                // sinf(c / iqfac) of Tns::read by coef_res, c = -8..7 at [c + 8]
    uint16_t lng[12][52], shrt[12][16];                  // band edges by sample-rate index (common.rs:22-92, :121-172)
    uint8_t n_lng[12], n_shrt[12], tns_max_long[12], tns_max_short[12];
};

struct Bands {
    const uint16_t* v;
    uint32_t len;  // entries (bands + 1)
};

struct Lcg {
    uint32_t state = kLcgSeed;
    uint32_t draws = 0;  // this packet's draws
    SYMGPU_HD int32_t next() { return ++draws, int32_t(state = state * 1664525u + 1013904223u); }
    // The state after `n` more draws: the n-th power of the affine map x -> a x + c, by squaring (mod 2^32).
    SYMGPU_HD static uint32_t jump(uint32_t s, uint64_t n) {
        uint32_t a = 1664525u, c = 1013904223u, ra = 1, rc = 0;
        for (; n; n >>= 1) {
            if (n & 1) ra *= a, rc = rc * a + c;
            c = c * a + c, a *= a;
        }
        return ra * s + rc;
    }
};

// One channel: IcsInfo + Ics.  `coeffs` points at the channel's 1024 lines.
struct Ics {
    uint8_t window_sequence, prev_window_sequence, window_shape, prev_window_shape;
    bool long_win;
    bool grouping[8];
    uint8_t group_start[8];
    uint32_t window_groups, num_windows, max_sfb, rate_idx;
    uint32_t global_gain;
    bool has_pulse;
    uint8_t n_pulse, pulse_start, pulse_off[4], pulse_amp[4];
    uint8_t shape_written;  // this packet assigned window_shape
    uint8_t n0;             // group-0 scale factors this packet wrote
    bool zero_lines;        // decode_spectrum clears the 1024 lines first (false: the caller hands them over cleared)
    uint32_t n_tns;         // TNS filters with order > 0, resolved to line ranges
    symgpu_aac_tns tns[8];
    uint8_t sfb_cb[8][64];
    float scales[8][64];
    float* coeffs;
};

SYMGPU_HD Bands bands_of(const Tables& T, uint32_t rate_idx, bool long_win) {
    return long_win ? Bands{T.lng[rate_idx], T.n_lng[rate_idx]} : Bands{T.shrt[rate_idx], T.n_shrt[rate_idx]};
}

// Ics::reset -> IcsInfo::new (ics/mod.rs:103-117, :229-232); also the state of a channel no packet touched yet.
SYMGPU_HD void reset_info(Ics& s) {
    s.window_sequence = s.prev_window_sequence = 0;
    s.window_shape = s.prev_window_shape = 0;
    for (int i = 0; i < 8; ++i) s.grouping[i] = false, s.group_start[i] = 0;
    s.window_groups = s.num_windows = s.max_sfb = 0;
    s.long_win = true;
}

SYMGPU_HD void init_ics(Ics& s, uint32_t rate_idx, float* coeffs) {
    reset_info(s);
    s.rate_idx = rate_idx, s.coeffs = coeffs;
    s.global_gain = 0, s.has_pulse = false, s.n_pulse = s.pulse_start = 0;
    s.shape_written = 0, s.n0 = 0, s.n_tns = 0, s.zero_lines = true;
    for (int g = 0; g < 8; ++g)
        for (int b = 0; b < 64; ++b) s.sfb_cb[g][b] = 0, s.scales[g][b] = 0.0f;
}

#define SYMGPU_AACE_CHECK(cond) \
    do {                        \
        if (!(cond)) return SYMGPU_ERR_DECODE; \
    } while (0)
#define SYMGPU_AACE_READ(w, v) SYMGPU_AACE_CHECK(bs.read((w), (v)))
#define SYMGPU_AACE_TRY(call)          \
    do {                               \
        const int st_ = (call);        \
        if (st_ != SYMGPU_OK) return st_; \
    } while (0)

// bit.rs:771-808: the codeword is matched against the data padded with zeros, then must fit.
SYMGPU_HD bool codebook(Bits& bs, const Book& b, uint32_t& value) {
    const uint32_t win = bs.window();
    const uint32_t e = b.lut[win >> 22];
    if (e) {
        value = e >> 5;
        return bs.skip(e & 31);
    }
    uint32_t node = 0;
    for (uint32_t len = 1; len <= b.max_len; ++len) {
        const int32_t next = b.node[2 * node + ((win >> (32 - len)) & 1)];
        if (next < 0) {
            value = uint32_t(~next);
            return bs.skip(len);
        }
        node = uint32_t(next);
    }
    return false;  // unreachable: the books are complete prefix codes
}

SYMGPU_HD void copy_from_common(Ics& s, const Ics& o) {
    const uint8_t seq = s.window_sequence, shape = s.window_shape;
    s.window_sequence = o.window_sequence, s.window_shape = o.window_shape, s.shape_written = 1;
    for (int i = 0; i < 8; ++i) s.grouping[i] = o.grouping[i], s.group_start[i] = o.group_start[i];
    s.window_groups = o.window_groups, s.num_windows = o.num_windows, s.max_sfb = o.max_sfb, s.long_win = o.long_win;
    s.prev_window_sequence = seq, s.prev_window_shape = shape;
}

SYMGPU_HD int decode_info(Bits& bs, const Tables& T, Ics& s) {  // ics/mod.rs:120-177, :292-300
    s.prev_window_sequence = s.window_sequence, s.prev_window_shape = s.window_shape;
    uint32_t v;
    SYMGPU_AACE_READ(1, v);
    SYMGPU_AACE_CHECK(v == 0);
    SYMGPU_AACE_READ(2, v);
    s.window_sequence = uint8_t(v);
    SYMGPU_AACE_READ(1, v);
    s.window_shape = uint8_t(v), s.shape_written = 1;
    s.window_groups = 1;
    if (s.window_sequence == SYMGPU_AAC_EIGHT_SHORT) {
        s.long_win = false, s.num_windows = 8;
        SYMGPU_AACE_READ(4, v);
        s.max_sfb = v;
        for (uint32_t i = 0; i < 7; ++i) {
            SYMGPU_AACE_READ(1, v);
            s.grouping[i] = v != 0;
            if (!v) s.group_start[s.window_groups++] = uint8_t(i + 1);
        }
    } else {
        s.long_win = true, s.num_windows = 1;
        SYMGPU_AACE_READ(6, v);
        s.max_sfb = v;
        SYMGPU_AACE_READ(1, v);
        if (v) return SYMGPU_ERR_UNSUPPORTED;  // predictor data (ltp.rs:20-54)
    }
    SYMGPU_AACE_CHECK(s.max_sfb + 1 <= bands_of(T, s.rate_idx, s.long_win).len);
    return SYMGPU_OK;
}

SYMGPU_HD uint32_t group_start_of(const Ics& s, uint32_t g) {
    return g == 0 ? 0 : g >= s.window_groups ? (s.long_win ? 1u : 8u) : s.group_start[g];
}

SYMGPU_HD int decode_section_data(Bits& bs, Ics& s) {  // :234-275
    const uint32_t bits = s.long_win ? 5 : 3, esc = (1u << bits) - 1;
    for (uint32_t g = 0; g < s.window_groups; ++g) {
        uint32_t k = 0, l = 0;
        while (k < s.max_sfb) {
            SYMGPU_AACE_CHECK(l < 64);
            uint32_t cb, inc;
            SYMGPU_AACE_READ(4, cb);
            SYMGPU_AACE_CHECK(cb != RESERVED_HCB);
            uint64_t len = 0;
            for (;;) {
                SYMGPU_AACE_READ(bits, inc);
                len += inc;
                if (inc < esc) break;
            }
            SYMGPU_AACE_CHECK(k + len <= s.max_sfb);
            for (uint32_t b = k; b < k + len; ++b) s.sfb_cb[g][b] = uint8_t(cb);
            k += uint32_t(len), ++l;
        }
    }
    return SYMGPU_OK;
}

SYMGPU_HD int decode_scale_factors(Bits& bs, const Tables& T, Ics& s) {  // :302-354
    bool noise_pcm = true;
    int32_t scf_int = 155, scf_noise = int32_t(s.global_gain) - 90 + 100, scf_normal = int32_t(s.global_gain);
    uint32_t v;
    for (uint32_t g = 0; g < s.window_groups; ++g)
        for (uint32_t b = 0; b < s.max_sfb; ++b) {
            const uint8_t cb = s.sfb_cb[g][b];
            float f;
            if (cb == ZERO_HCB) {
                f = 0.0f;
            } else if (cb == INTENSITY_HCB || cb == INTENSITY_HCB2) {
                SYMGPU_AACE_CHECK(codebook(bs, T.book[11], v));
                scf_int += int32_t(v) - 60;
                SYMGPU_AACE_CHECK(scf_int >= 0 && scf_int < 256);
                f = T.intensity_scf[scf_int];
            } else if (cb == NOISE_HCB) {
                if (noise_pcm) {
                    noise_pcm = false;
                    SYMGPU_AACE_READ(9, v);
                    scf_noise += int32_t(v) - 256;
                } else {
                    SYMGPU_AACE_CHECK(codebook(bs, T.book[11], v));
                    scf_noise += int32_t(v) - 60;
                }
                SYMGPU_AACE_CHECK(scf_noise >= 0 && scf_noise < 256);
                f = T.normal_scf[scf_noise];
            } else {
                SYMGPU_AACE_CHECK(codebook(bs, T.book[11], v));
                scf_normal += int32_t(v) - 60;
                SYMGPU_AACE_CHECK(scf_normal >= 0 && scf_normal < 256);
                f = T.normal_scf[scf_normal];
            }
            s.scales[g][b] = f;
            if (g == 0) s.n0 = uint8_t(b + 1);
        }
    return SYMGPU_OK;
}

SYMGPU_HD float sign_of(uint32_t bit) { return 1.0f - 2.0f * float(bit); }

// ---- correctly rounded square root and division in integer arithmetic ------------------------------------------------------
// Noise scaling needs IEEE sqrtf and division.  nvcc's correctly rounded sequences for them use fused multiply-adds, which the
// library's kernels are kept free of (tests/test_build_and_abi.py), so the host and the device both use these: the same bits
// as IEEE round-to-nearest-even for finite, non-negative operands.
SYMGPU_HD uint32_t f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u;
    __builtin_memcpy(&u, &f, 4);
    return u;
#endif
}
SYMGPU_HD float u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    __builtin_memcpy(&f, &u, 4);
    return f;
#endif
}
SYMGPU_HD void split(float x, uint64_t& m, int& e) {  // |x| = m * 2^e, m normalised to 24 bits (x != 0, finite)
    const uint32_t b = f2u(x), ef = (b >> 23) & 255;
    m = b & 0x7fffffu, e = -149;
    if (ef) m |= 0x800000u, e = int(ef) - 150;
    while (m < 0x800000u) m <<= 1, --e;
}
SYMGPU_HD float round_rn(uint64_t r, int e, bool sticky) {  // r * 2^e (+ a sticky fraction below r's last bit), r >= 2^24
#ifdef __CUDA_ARCH__
    const int nb = 64 - __clzll((long long)r);
#else
    const int nb = 64 - __builtin_clzll(r);
#endif
    const int shift = nb - 24;
    uint64_t keep = r >> shift;
    const uint64_t rem = r & ((uint64_t(1) << shift) - 1), half = uint64_t(1) << (shift - 1);
    if (rem > half || (rem == half && (sticky || (keep & 1)))) ++keep;
    e += shift;
    if (keep >> 24) keep >>= 1, ++e;
    const int biased = e + 23 + 127;
    if (biased >= 255) return u2f(0x7f800000u);
    if (biased <= 0) return 0.0f;  // not reached: the roots and quotients of noise scaling are normal
    return u2f(uint32_t(biased) << 23 | uint32_t(keep & 0x7fffffu));
}
SYMGPU_HD float sqrt_rn(float x) {  // x >= 0, finite
    if (x == 0.0f) return x;
    uint64_t m;
    int e;
    split(x, m, e);
    if (e & 1) m <<= 1, --e;
    uint64_t n = m << 38, res = 0, one = uint64_t(1) << 62;  // digit by digit: res = floor(sqrt(n)), n = the remainder
    while (one > n) one >>= 2;
    while (one) {
        if (n >= res + one) n -= res + one, res = (res >> 1) + one;
        else res >>= 1;
        one >>= 2;
    }
    return round_rn(res, (e - 38) / 2, n != 0);
}
SYMGPU_HD float div_rn(float a, float b) {  // a, b >= 0, finite
    if (b == 0.0f) return a == 0.0f ? u2f(0x7fc00000u) : u2f(0x7f800000u);
    if (a == 0.0f) return 0.0f;
    uint64_t ma, mb;
    int ea, eb;
    split(a, ma, ea), split(b, mb, eb);
    const uint64_t n = ma << 40;
    return round_rn(n / mb, ea - eb - 40, n % mb != 0);
}

// :598-607.  n ones then a zero, n < 9 (more ones fail the packet as running out of data does), then n + 4 bits.
SYMGPU_HD bool read_escape(Bits& bs, uint32_t& out) {
    const uint32_t win = bs.window();
#ifdef __CUDA_ARCH__
    const uint32_t n = uint32_t(__clz(int(~win | 0x7fffffu)));  // the leading ones, at most 9
#else
    const uint32_t n = uint32_t(__builtin_clz(~win | 0x7fffffu));
#endif
    if (n >= 9 || !bs.skip(n + 1)) return false;
    uint32_t w;
    if (!bs.read(n + 4, w)) return false;
    out = (1u << (n + 4)) + w;
    return true;
}

SYMGPU_HD int decode_spectrum(Bits& bs, const Tables& T, Ics& s, Lcg& lcg) {  // :360-401, :466-596
    float* coeffs = s.coeffs;
    if (s.zero_lines)
        for (int i = 0; i < 1024; ++i) coeffs[i] = 0.0f;
    const Bands b = bands_of(T, s.rate_idx, s.long_win);
    uint32_t cw, bit;
    for (uint32_t g = 0; g < s.window_groups; ++g) {
        const uint32_t cur_w = group_start_of(s, g), next_w = group_start_of(s, g + 1);
        for (uint32_t sfb = 0; sfb < s.max_sfb; ++sfb) {
            const uint8_t cb = s.sfb_cb[g][sfb];
            const float scale = s.scales[g][sfb];
            if (cb == ZERO_HCB || cb == RESERVED_HCB || cb == INTENSITY_HCB || cb == INTENSITY_HCB2) continue;
            const uint32_t n = uint32_t(b.v[sfb + 1] - b.v[sfb]);
            for (uint32_t w = cur_w; w < next_w; ++w) {
                float* dst = coeffs + b.v[sfb] + 128 * w;
                if (cb == NOISE_HCB) {  // decode_noise
                    float energy = 0.0f;
                    for (uint32_t i = 0; i < n; ++i) {
                        const float x = float(int16_t(lcg.next() >> 16));
                        dst[i] = x;
                        energy += x * x;
                    }
                    const float sc = div_rn(scale, sqrt_rn(energy));
                    for (uint32_t i = 0; i < n; ++i) dst[i] *= sc;
                } else if (cb <= 2) {
                    const float iq[3] = {-scale, 0.0f, scale};
                    for (uint32_t i = 0; i + 4 <= n; i += 4) {
                        SYMGPU_AACE_CHECK(codebook(bs, T.book[cb - 1], cw));
                        dst[i] = iq[cw / 27], dst[i + 1] = iq[cw / 9 % 3], dst[i + 2] = iq[cw / 3 % 3], dst[i + 3] = iq[cw % 3];
                    }
                } else if (cb <= 4) {
                    const float iq[3] = {0.0f, scale, 2.51984209978974632953f * scale};
                    for (uint32_t i = 0; i + 4 <= n; i += 4) {
                        SYMGPU_AACE_CHECK(codebook(bs, T.book[cb - 1], cw));
                        const uint32_t d[4] = {cw / 27, cw / 9 % 3, cw / 3 % 3, cw % 3};
                        for (int k = 0; k < 4; ++k)
                            if (d[k]) {
                                SYMGPU_AACE_READ(1, bit);
                                dst[i + k] = sign_of(bit) * iq[d[k]];
                            }
                    }
                } else if (cb <= 6) {
                    for (uint32_t i = 0; i + 2 <= n; i += 2) {
                        SYMGPU_AACE_CHECK(codebook(bs, T.book[cb - 1], cw));
                        const uint32_t a = cw / 9, c = cw % 9;
                        const float x = a < 4 ? -T.pow43[4 - a] : T.pow43[a - 4], y = c < 4 ? -T.pow43[4 - c] : T.pow43[c - 4];
                        dst[i] = x * scale, dst[i + 1] = y * scale;
                    }
                } else if (cb <= 10) {
                    const uint32_t mod = cb < 9 ? 8 : 13;
                    for (uint32_t i = 0; i + 2 <= n; i += 2) {
                        SYMGPU_AACE_CHECK(codebook(bs, T.book[cb - 1], cw));
                        const float x = T.pow43[cw / mod], y = T.pow43[cw % mod];
                        float sx = 1.0f, sy = 1.0f;
                        if (x != 0.0f) {
                            SYMGPU_AACE_READ(1, bit);
                            sx = sign_of(bit);
                        }
                        if (y != 0.0f) {
                            SYMGPU_AACE_READ(1, bit);
                            sy = sign_of(bit);
                        }
                        dst[i] = sx * x * scale, dst[i + 1] = sy * y * scale;
                    }
                } else {
                    for (uint32_t i = 0; i + 2 <= n; i += 2) {
                        SYMGPU_AACE_CHECK(codebook(bs, T.book[10], cw));
                        uint32_t a = cw / 17, c = cw % 17;
                        float sx = 1.0f, sy = 1.0f;
                        if (a) {
                            SYMGPU_AACE_READ(1, bit);
                            sx = sign_of(bit);
                        }
                        if (c) {
                            SYMGPU_AACE_READ(1, bit);
                            sy = sign_of(bit);
                        }
                        if (a == 16) SYMGPU_AACE_CHECK(read_escape(bs, a));
                        if (c == 16) SYMGPU_AACE_CHECK(read_escape(bs, c));
                        dst[i] = sx * T.pow43[a] * scale, dst[i + 1] = sy * T.pow43[c] * scale;
                    }
                }
            }
        }
    }
    return SYMGPU_OK;
}

// Tns::read (tns.rs:35-147), each filter resolved at once to the line range Tns::synth walks (:149-199); order 0 left out.
SYMGPU_HD int read_tns(Bits& bs, const Tables& T, Ics& s) {
    s.n_tns = 0;
    uint32_t v;
    SYMGPU_AACE_READ(1, v);
    if (!v) return SYMGPU_OK;
    const Bands b = bands_of(T, s.rate_idx, s.long_win);
    uint32_t max_bands = s.long_win ? T.tns_max_long[s.rate_idx] : T.tns_max_short[s.rate_idx];
    if (s.max_sfb < max_bands) max_bands = s.max_sfb;
    const uint32_t max_order = s.long_win ? 12 : 7;
    for (uint32_t w = 0; w < s.num_windows; ++w) {
        uint32_t nf, coef_res = 0;
        SYMGPU_AACE_READ(s.long_win ? 2 : 1, nf);
        if (nf) SYMGPU_AACE_READ(1, coef_res);
        uint32_t bottom = b.len - 1;
        for (uint32_t f = 0; f < nf; ++f) {
            uint32_t length, order;
            SYMGPU_AACE_READ(s.long_win ? 6 : 4, length);
            SYMGPU_AACE_READ(s.long_win ? 5 : 3, order);
            SYMGPU_AACE_CHECK(order <= max_order);
            const uint32_t top = bottom;
            bottom = top > length ? top - length : 0;
            if (order == 0) continue;
            uint32_t direction, compress;
            SYMGPU_AACE_READ(1, direction);
            SYMGPU_AACE_READ(1, compress);
            const uint32_t res_bits = (coef_res ? 4u : 3u) - (compress ? 1u : 0u);
            const uint32_t sign_mask = 1u << (res_bits - 1), full = 1u << res_bits;
            float tmp[12];
            for (uint32_t k = 0; k < order; ++k) {
                SYMGPU_AACE_READ(res_bits, v);
                const int32_t c = (v & sign_mask) ? int32_t(v) - int32_t(full) : int32_t(v);
                tmp[k] = T.tns_sin[coef_res][c + 8];
            }
            symgpu_aac_tns& o = s.tns[s.n_tns++];
            o.start = uint16_t(w * 128 + b.v[bottom < max_bands ? bottom : max_bands]);
            o.end = uint16_t(w * 128 + b.v[top < max_bands ? top : max_bands]);
            o.order = uint8_t(order), o.direction = uint8_t(direction), o.reserved = 0;
            float* coef = o.lpc;
            for (int i = 0; i < 20; ++i) coef[i] = 0.0f;
            float bb[13];
            for (uint32_t m = 1; m <= order; ++m) {
                for (uint32_t i = 1; i < m; ++i) bb[i] = coef[i - 1] + tmp[m - 1] * coef[m - i - 1];
                for (uint32_t i = 1; i < m; ++i) coef[i - 1] = bb[i];
                coef[m - 1] = tmp[m - 1];
            }
        }
    }
    return SYMGPU_OK;
}

SYMGPU_HD int decode_ics(Bits& bs, const Tables& T, Ics& s, Lcg& lcg, bool common_window) {  // Ics::decode, ics/mod.rs:403-447
    uint32_t v;
    SYMGPU_AACE_READ(8, s.global_gain);
    if (!common_window) SYMGPU_AACE_TRY(decode_info(bs, T, s));
    SYMGPU_AACE_TRY(decode_section_data(bs, s));
    SYMGPU_AACE_TRY(decode_scale_factors(bs, T, s));
    SYMGPU_AACE_READ(1, v);
    s.has_pulse = v != 0;
    if (s.has_pulse) {
        SYMGPU_AACE_READ(2, v);
        s.n_pulse = uint8_t(v + 1);
        SYMGPU_AACE_READ(6, v);
        s.pulse_start = uint8_t(v);
        for (uint32_t i = 0; i < s.n_pulse; ++i) {
            SYMGPU_AACE_READ(5, v);
            s.pulse_off[i] = uint8_t(v);
            SYMGPU_AACE_READ(4, v);
            s.pulse_amp[i] = uint8_t(v);
        }
    }
    SYMGPU_AACE_CHECK(!s.has_pulse || s.long_win);
    SYMGPU_AACE_TRY(read_tns(bs, T, s));
    SYMGPU_AACE_READ(1, v);
    SYMGPU_AACE_CHECK(v == 0);  // gain control
    return decode_spectrum(bs, T, s, lcg);
}

SYMGPU_HD int decode_cpe(Bits& bs, const Tables& T, Ics& a, Ics& b, Lcg& lcg, bool (&ms_used)[8][64]) {  // cpe.rs:61-161
    uint32_t common, ms_mask_present = 0, v;
    SYMGPU_AACE_READ(1, common);
    if (common) {
        SYMGPU_AACE_TRY(decode_info(bs, T, a));
        SYMGPU_AACE_READ(2, ms_mask_present);
        SYMGPU_AACE_CHECK(ms_mask_present != 3);
        for (uint32_t g = 0; g < a.window_groups; ++g)
            for (uint32_t sfb = 0; sfb < a.max_sfb; ++sfb) {
                if (ms_mask_present == 1) {
                    SYMGPU_AACE_READ(1, v);
                    ms_used[g][sfb] = v != 0;
                } else {
                    ms_used[g][sfb] = ms_mask_present == 2;
                }
            }
        copy_from_common(b, a);
    }
    SYMGPU_AACE_TRY(decode_ics(bs, T, a, lcg, common));
    SYMGPU_AACE_TRY(decode_ics(bs, T, b, lcg, common));
    if (!common) return SYMGPU_OK;
    const Bands bd = bands_of(T, a.rate_idx, a.long_win);
    uint32_t g = 0;
    for (uint32_t w = 0; w < a.num_windows; ++w) {
        if (w > 0 && !a.grouping[w - 1]) ++g;
        for (uint32_t sfb = 0; sfb < a.max_sfb; ++sfb) {
            const uint32_t lo = w * 128 + bd.v[sfb], hi = w * 128 + bd.v[sfb + 1];
            const uint8_t c0 = a.sfb_cb[g][sfb], c1 = b.sfb_cb[g][sfb];
            if (c1 == INTENSITY_HCB || c1 == INTENSITY_HCB2) {
                const bool invert = ms_mask_present == 1 && ms_used[g][sfb];
                const float dir = c1 == INTENSITY_HCB ? 1.0f : -1.0f, factor = invert ? -1.0f : 1.0f;
                const float scale = dir * factor * b.scales[g][sfb];
                for (uint32_t i = lo; i < hi; ++i) b.coeffs[i] = scale * a.coeffs[i];
            } else if (c0 == NOISE_HCB || c1 == NOISE_HCB) {
            } else if (ms_used[g][sfb]) {
                for (uint32_t i = lo; i < hi; ++i) {
                    const float tmp = a.coeffs[i] - b.coeffs[i];
                    a.coeffs[i] += b.coeffs[i];
                    b.coeffs[i] = tmp;
                }
            }
        }
    }
    return SYMGPU_OK;
}

// AacDecoder::decode_ga (mod.rs:128-229).  S supplies the stream's side of set_pair: S::set_pair(k, channel, is_pair) -> status,
// S::ics(k, c), S::lcg(k), S::ms_used(k).
template <class S>
SYMGPU_HD int decode_ga(Bits& bs, const Tables& T, S& st, uint32_t& cur_pair, uint32_t& cur_ch) {
    uint32_t v;
    while (bs.left() > 3) {
        uint32_t id;
        SYMGPU_AACE_READ(3, id);
        switch (id) {
            case 0:
            case 3:
                SYMGPU_AACE_READ(4, v);
                SYMGPU_AACE_TRY(st.set_pair(cur_pair, cur_ch, false));
                SYMGPU_AACE_TRY(decode_ics(bs, T, st.ics(cur_pair, 0), st.lcg(cur_pair), false));
                ++cur_pair, ++cur_ch;
                break;
            case 1:
                SYMGPU_AACE_READ(4, v);
                SYMGPU_AACE_TRY(st.set_pair(cur_pair, cur_ch, true));
                SYMGPU_AACE_TRY(decode_cpe(bs, T, st.ics(cur_pair, 0), st.ics(cur_pair, 1), st.lcg(cur_pair), st.ms_used(cur_pair)));
                ++cur_pair, cur_ch += 2;
                break;
            case 2: return SYMGPU_ERR_UNSUPPORTED;
            case 4: {
                uint32_t align, count;
                SYMGPU_AACE_READ(4, v);
                SYMGPU_AACE_READ(1, align);
                SYMGPU_AACE_READ(8, count);
                if (count == 255) {
                    SYMGPU_AACE_READ(8, v);
                    count += v;
                }
                if (align) bs.at = (bs.at + 7) & ~size_t(7);
                SYMGPU_AACE_CHECK(bs.at <= bs.n_bits && bs.skip(size_t(count) * 8));
                break;
            }
            case 5: return SYMGPU_ERR_UNSUPPORTED;
            case 6: {
                uint32_t count;
                SYMGPU_AACE_READ(4, count);
                if (count == 15) {
                    SYMGPU_AACE_READ(8, v);
                    count += v - 1;
                }
                if (count > 0) {
                    SYMGPU_AACE_READ(4, v);
                    SYMGPU_AACE_CHECK(bs.skip(4));
                    SYMGPU_AACE_CHECK(bs.skip(size_t(count - 1) * 8));
                }
                break;
            }
            default: return SYMGPU_OK;  // ID_TERM
        }
    }
    return SYMGPU_OK;
}

// ---- pulses ----------------------------------------------------------------------------------------------------------------
// The lines Pulse::synth changes (pulse.rs:60-105), in its order; a line may come twice (offset 0).
struct PulseLines {
    uint8_t n, max_sfb;
    uint8_t band[4], amp[4];
    uint16_t line[4];
};

SYMGPU_HD PulseLines pulse_lines(const Tables& T, const Ics& s) {
    PulseLines p{};
    p.max_sfb = uint8_t(s.max_sfb);
    if (!s.has_pulse) return p;
    const Bands b = bands_of(T, s.rate_idx, s.long_win);
    if (s.pulse_start >= b.len - 1) return p;
    uint32_t k = b.v[s.pulse_start], band = s.pulse_start;
    for (uint32_t i = 0; i < s.n_pulse; ++i) {
        k += s.pulse_off[i];
        if (k >= 1024) break;
        while (b.v[band + 1] <= k) ++band;
        p.line[p.n] = uint16_t(k), p.band[p.n] = uint8_t(band), p.amp[p.n] = s.pulse_amp[i];
        ++p.n;
    }
    return p;
}

// Host only (C library powf, as the reference's f32::powf).  value[i]: line[i] before the pulses; scale[i]: scales[0][band[i]].
// On return value[i] is what line[i] holds after pulse i (the last pulse on a line leaves its final value).
inline void pulse_apply(const PulseLines& p, const float* scale, float* value) {
    const float p43 = 4.0f / 3.0f;
    for (uint32_t i = 0; i < p.n; ++i) {
        float cur = value[i];
        for (uint32_t j = 0; j < i; ++j)
            if (p.line[j] == p.line[i]) cur = value[j];
        float base = cur;
        if (base != 0.0f) {
            if (scale[i] == 0.0f) {
                base = 0.0f;
            } else {
                const float bval = cur / scale[i];
                base = bval >= 0.0f ? powf(cur, 0.75f) : -powf(-cur, 0.75f);
            }
        }
        if (base > 0.0f) base += float(p.amp[i]);
        else base -= float(p.amp[i]);
        const float iq = base < 0.0f ? -powf(-base, p43) : powf(base, p43);
        value[i] = iq * scale[i];
    }
}

// ---- one packet from a fresh state (the device's pass A / pass B) -----------------------------------------------------------
// What the packet does to the state that carries, as decoded from a fresh state: enough for walk_step to tell what it does in
// context.  Everything element k does touches only element k's state.
struct JobRec {
    int8_t status;          // symgpu_status of the fresh decode (SYMGPU_OK, _ERR_DECODE, _ERR_UNSUPPORTED)
    uint8_t n_att;          // set_pair attempts, in element order
    uint8_t att[3];         // channel | is_pair << 7
    uint8_t shape;          // bit c: channel c's window_shape was assigned; bit 2 + c: the value
    uint8_t n0[2];          // group-0 scale factors written, per channel
    uint8_t elem_of_ch[2];  // the element that decoded channel c, 0xff: none
    uint8_t n_tns[2];       // TNS records of channel c (a decoded packet), at tns[8 c]
    uint8_t reserved[2];
    uint32_t draws[2];      // noise draws of elements 0 and 1 (a third element never gets past set_pair)
};

// The fresh state of one packet: channel c's Ics is ics[c], element k's generator starts at lcg_start[k].
struct JobState {
    uint32_t channels;
    uint32_t lcg_start[2];
    JobRec rec;
    Lcg lcg_[2];
    Ics ics_[2];
    bool ms_[8][64];
    SYMGPU_HD int set_pair(uint32_t k, uint32_t ch, bool pair) {  // mod.rs:114-126 on a fresh layout: pair k is new
        rec.att[rec.n_att++] = uint8_t(ch | (pair ? 0x80u : 0u));
        if (k < 2) lcg_[k].state = lcg_start[k], lcg_[k].draws = 0;
        SYMGPU_AACE_CHECK((pair ? ch + 1 : ch) < channels);
        for (uint32_t c = 0; c < (pair ? 2u : 1u); ++c) rec.elem_of_ch[ch + c] = uint8_t(k);
        return SYMGPU_OK;
    }
    SYMGPU_HD Ics& ics(uint32_t k, uint32_t c) { return ics_[(rec.att[k] & 0x7f) + c]; }
    SYMGPU_HD Lcg& lcg(uint32_t k) { return lcg_[k]; }
    SYMGPU_HD bool (&ms_used(uint32_t))[8][64] { return ms_; }
};

// Where decode_job writes one packet: units [2] (prev_window_shape 0, tns_first 8 c: walk and placement fill them in), tns [16],
// coeffs [2][1024] (lines_cleared: they are zero, and only the lines the packet codes are written -- pass A after one memset of
// the whole buffer; otherwise every line of a decoded channel is written, as pass B must: joint stereo may have written lines
// of bands the spectrum skips; channels the packet does not decode are not written), pulse [2], scales0 [2][64] (group-0 scale factors: the first rec.n0[c] are written).
struct JobOut {
    symgpu_aac_unit* units;
    symgpu_aac_tns* tns;
    float* coeffs;
    PulseLines* pulse;
    float* scales0;
};

SYMGPU_HD void decode_job(const uint8_t* p, size_t n, const Tables& T, uint32_t rate_idx, uint32_t channels, const uint32_t lcg_start[2],
                          bool lines_cleared, JobState& S, JobOut o) {
    S.channels = channels;
    S.lcg_start[0] = lcg_start[0], S.lcg_start[1] = lcg_start[1];
    S.rec = JobRec{};
    S.rec.elem_of_ch[0] = S.rec.elem_of_ch[1] = 0xff;
    for (uint32_t c = 0; c < 2; ++c) {
        init_ics(S.ics_[c], rate_idx, o.coeffs + 1024 * c), S.lcg_[c] = Lcg{};
        S.ics_[c].zero_lines = !lines_cleared;
    }
    Bits bs(p, n);
    uint32_t cur_pair = 0, cur_ch = 0;
    int st = decode_ga(bs, T, S, cur_pair, cur_ch);
    if (st == SYMGPU_OK && cur_ch != channels) st = SYMGPU_ERR_UNSUPPORTED;
    JobRec& r = S.rec;
    r.status = int8_t(st);
    for (uint32_t k = 0; k < 2; ++k) r.draws[k] = S.lcg_[k].draws;
    for (uint32_t c = 0; c < 2; ++c) {
        const Ics& s = S.ics_[c];
        if (r.elem_of_ch[c] == 0xff) continue;
        r.shape |= uint8_t((s.shape_written << c) | ((s.shape_written & s.window_shape) << (2 + c)));
        r.n0[c] = s.n0;
        for (uint32_t b = 0; b < s.n0; ++b) o.scales0[64 * c + b] = s.scales[0][b];
    }
    for (uint32_t c = 0; c < 2; ++c) {
        symgpu_aac_unit u{};
        o.pulse[c] = PulseLines{};
        if (st == SYMGPU_OK && c < channels) {
            const Ics& s = S.ics_[c];
            u.window_sequence = s.window_sequence, u.window_shape = s.window_shape;
            u.n_tns = uint8_t(s.n_tns), u.tns_first = s.n_tns ? 8 * c : 0;
            r.n_tns[c] = uint8_t(s.n_tns);
            for (uint32_t f = 0; f < s.n_tns; ++f) o.tns[8 * c + f] = s.tns[f];
            o.pulse[c] = pulse_lines(T, s);
        }
        o.units[c] = u;
    }
}

// ---- the walk: one file's records in stream order --------------------------------------------------------------------------
constexpr uint32_t kNoJob = 0xffffffffu;

// Per channel, the packets whose group-0 scale factors may still be read, as a stack of (job, bands written) with the bands
// strictly decreasing from bottom to top: a packet that wrote at least as many bands as an earlier one hides it.  The last
// writer of band b is the topmost entry with more than b bands.  At most 64 entries; O(1) amortised per packet.
struct WalkState {
    uint8_t n_est;        // elements established (set_pair's layout)
    uint8_t est[3];
    uint8_t shape;        // bit c: channel c's window_shape
    uint8_t depth[2];
    uint32_t lcg[2];      // each element's generator before the next packet
    uint8_t stk_n0[2][64];
    uint32_t stk_job[2][64];
};
struct WalkOut {
    int8_t status;        // what the packet does in context
    uint8_t prev_shape;   // bit c: channel c's prev_window_shape
    uint8_t n0[2];        // group-0 scale factors the packet leaves behind, per channel
    uint32_t lcg_start[2];
    uint32_t scale_src[2][4];  // a decoded packet's pulse line i of channel c reads scales0 of this job (kNoJob: 0.0)
};

SYMGPU_HD void walk_begin(WalkState& w) {
    w.n_est = 0, w.shape = 0, w.depth[0] = w.depth[1] = 0;
    w.lcg[0] = w.lcg[1] = kLcgSeed;
}

// Job `job`'s record in context; pulse [2]: its pulse lines (read when it decodes).
SYMGPU_HD WalkOut walk_step(WalkState& w, const JobRec& r, uint32_t job, const PulseLines* pulse) {
    uint32_t refused_at = r.n_att;  // the first attempt set_pair refuses in context; the elements before it keep their effects
    for (uint32_t e = 0; e < r.n_att; ++e) {
        if (e < w.n_est) {
            if (w.est[e] != r.att[e]) {
                refused_at = e;
                break;
            }
        } else {
            w.est[e] = r.att[e], w.n_est = uint8_t(e + 1);
        }
    }
    WalkOut o{};
    o.status = int8_t(refused_at < r.n_att ? SYMGPU_ERR_DECODE : r.status);
    o.prev_shape = w.shape;
    o.lcg_start[0] = w.lcg[0], o.lcg_start[1] = w.lcg[1];
    for (uint32_t k = 0; k < 2 && k < refused_at; ++k) w.lcg[k] = Lcg::jump(w.lcg[k], r.draws[k]);
    for (uint32_t c = 0; c < 2; ++c) {
        for (uint32_t i = 0; i < 4; ++i) o.scale_src[c][i] = kNoJob;
        if (r.elem_of_ch[c] >= refused_at) continue;
        const uint8_t v = r.n0[c];
        o.n0[c] = v;
        if (r.shape >> c & 1) w.shape = uint8_t((w.shape & ~(1u << c)) | ((r.shape >> (2 + c) & 1u) << c));
        if (v) {
            while (w.depth[c] && w.stk_n0[c][w.depth[c] - 1] <= v) --w.depth[c];
            w.stk_n0[c][w.depth[c]] = v, w.stk_job[c][w.depth[c]] = job, ++w.depth[c];
        }
    }
    if (o.status == SYMGPU_OK)  // Pulse::synth runs after the whole packet: its own scale factors are the newest
        for (uint32_t c = 0; c < 2; ++c)
            for (uint32_t i = 0; i < pulse[c].n; ++i)
                for (uint32_t d = w.depth[c]; d-- > 0;)
                    if (w.stk_n0[c][d] > pulse[c].band[i]) {
                        o.scale_src[c][i] = w.stk_job[c][d];
                        break;
                    }
    return o;
}

#undef SYMGPU_AACE_CHECK
#undef SYMGPU_AACE_READ
#undef SYMGPU_AACE_TRY

}  // namespace aace

// The tables, built on the host once (aac_frontend.cpp).
const aace::Tables& aac_tables_host();
uint32_t aac_rate_index(uint32_t sample_rate);

}  // namespace symgpu
