// AAC-LC entropy front-end (include/symgpu.h "AAC entropy front-end", SURVEY §8f N1): one raw_data_block per packet ->
// what symgpu_aac_synth_* reads (two channel units, resolved TNS filters, 2 x 1024 dequantised lines).  Everything the
// reference does between BitReaderLtr::new(packet.data) and Dsp::synth, in its order:
//   AacDecoder::decode_ga / set_pair            symphonia-codec-aac/src/aac/mod.rs:114-229
//   ChannelPair::decode_ga_sce / decode_ga_cpe  aac/cpe.rs:51-161      (common window, ms mask, intensity, mid/side)
//   IcsInfo::decode, Ics::decode*               aac/ics/mod.rs:120-447 (sections, scale factors, spectrum, noise)
//   Pulse::read / synth, Tns::read (+ ranges)   aac/ics/pulse.rs:35-105, aac/ics/tns.rs:35-199
// The per-packet rules are the host/device functions of aac_entropy.h; this file keeps the stream state between packets and
// is a loop over them.  CPU only.  State is changed in place as the reference changes it: a packet that fails half way leaves
// the window history and the noise generator where the failure found them.
//
// Floating point: single IEEE operations in the reference's order (host code is compiled with -ffp-contract=off); the
// tables use the C library's powf, which is what f32::powf calls (tests/test_aac_frontend.py: the scale-factor tables are the
// correctly rounded powers of two; x^(4/3) is within one unit in the last place, 10 of 8192 entries differ under glibc).
#include <cmath>
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <thread>
#include <vector>

#include "../../include/symgpu.h"
#include "aac_entropy.h"

namespace {

namespace ae = symgpu::aace;

#include "aac_huffman_data.inc"

// ---- aac/common.rs:22-92, :121-172; tns.rs:22-24 --------------------------------------------------------------------------
const uint16_t L48[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 48, 56, 64, 72, 80, 88, 96, 108, 120, 132, 144, 160, 176, 196, 216, 240, 264, 292, 320,
                        352, 384, 416, 448, 480, 512, 544, 576, 608, 640, 672, 704, 736, 768, 800, 832, 864, 896, 928, 1024};
const uint16_t S48[] = {0, 4, 8, 12, 16, 20, 28, 36, 44, 56, 68, 80, 96, 112, 128};
const uint16_t L32[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 48, 56, 64, 72, 80, 88, 96, 108, 120, 132, 144, 160, 176, 196, 216, 240, 264, 292, 320,
                        352, 384, 416, 448, 480, 512, 544, 576, 608, 640, 672, 704, 736, 768, 800, 832, 864, 896, 928, 960, 992, 1024};
const uint16_t L8[] = {0, 12, 24, 36, 48, 60, 72, 84, 96, 108, 120, 132, 144, 156, 172, 188, 204, 220, 236, 252, 268, 288, 308, 328, 348, 372, 396, 420,
                       448, 476, 508, 544, 580, 620, 664, 712, 764, 820, 880, 944, 1024};
const uint16_t S8[] = {0, 4, 8, 12, 16, 20, 24, 28, 36, 44, 52, 60, 72, 88, 108, 128};
const uint16_t L16[] = {0, 8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 100, 112, 124, 136, 148, 160, 172, 184, 196, 212, 228, 244, 260, 280, 300, 320, 344,
                        368, 396, 424, 456, 492, 532, 572, 616, 664, 716, 772, 832, 896, 960, 1024};
const uint16_t S16[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 40, 48, 60, 72, 88, 108, 128};
const uint16_t L24[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 44, 52, 60, 68, 76, 84, 92, 100, 108, 116, 124, 136, 148, 160, 172, 188, 204, 220, 240,
                        260, 284, 308, 336, 364, 396, 432, 468, 508, 552, 600, 652, 704, 768, 832, 896, 960, 1024};
const uint16_t S24[] = {0, 4, 8, 12, 16, 20, 24, 28, 36, 44, 52, 64, 76, 92, 108, 128};
const uint16_t L64[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 44, 48, 52, 56, 64, 72, 80, 88, 100, 112, 124, 140, 156, 172, 192, 216, 240, 268, 304,
                        344, 384, 424, 464, 504, 544, 584, 624, 664, 704, 744, 784, 824, 864, 904, 944, 984, 1024};
const uint16_t S64[] = {0, 4, 8, 12, 16, 20, 24, 32, 40, 48, 64, 92, 128};
const uint16_t L96[] = {0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40, 44, 48, 52, 56, 64, 72, 80, 88, 96, 108, 120, 132, 144, 156, 172, 188, 212, 240, 276,
                        320, 384, 448, 512, 576, 640, 704, 768, 832, 896, 960, 1024};
struct BandList {
    const uint16_t* v;
    size_t len;  // entries (bands + 1)
};
#define BANDS(a) BandList{a, sizeof(a) / sizeof(a[0])}
struct SubbandInfo {
    uint32_t min_rate;
    BandList lng, shrt;
};
const SubbandInfo kInfo[12] = {{92017, BANDS(L96), BANDS(S64)}, {75132, BANDS(L96), BANDS(S64)}, {55426, BANDS(L64), BANDS(S64)}, {46009, BANDS(L48), BANDS(S48)},
                               {37566, BANDS(L48), BANDS(S48)}, {27713, BANDS(L32), BANDS(S48)}, {23004, BANDS(L24), BANDS(S24)}, {18783, BANDS(L24), BANDS(S24)},
                               {13856, BANDS(L16), BANDS(S16)}, {11502, BANDS(L16), BANDS(S16)}, {9391, BANDS(L16), BANDS(S16)},  {0, BANDS(L8), BANDS(S8)}};
const uint8_t kTnsMaxLong[12] = {31, 31, 34, 40, 42, 51, 46, 46, 42, 42, 42, 39};
const uint8_t kTnsMaxShort[12] = {9, 9, 10, 14, 14, 14, 14, 14, 14, 14, 14, 14};

// ---- the tables of aac_entropy.h ---------------------------------------------------------------------------------------------
void build_book(ae::Book& b, const uint32_t* words, size_t n) {  // the (length, code) list -> first-level LUT + binary tree
    std::memset(&b, 0, sizeof b);
    size_t n_nodes = 1;
    for (size_t v = 0; v < n; ++v) {
        const uint32_t len = words[v] >> 24, code = words[v] & 0xffffff;
        if (len > b.max_len) b.max_len = len;
        if (len <= 10)
            for (uint32_t k = 0; k < (1u << (10 - len)); ++k) b.lut[(code << (10 - len)) | k] = uint16_t(v << 5 | len);
        size_t at = 0;
        for (uint32_t bit_no = len; bit_no-- > 0;) {
            const uint32_t bit = (code >> bit_no) & 1;
            if (bit_no == 0) {
                b.node[2 * at + bit] = ~int32_t(v);
            } else {
                if (b.node[2 * at + bit] == 0) b.node[2 * at + bit] = int32_t(n_nodes++);
                at = size_t(b.node[2 * at + bit]);
            }
        }
    }
}

struct HostTables {
    ae::Tables t;
    HostTables() {
        std::memset(&t, 0, sizeof t);
        const uint32_t* w[11] = {kAacHuff_1, kAacHuff_2, kAacHuff_3, kAacHuff_4, kAacHuff_5, kAacHuff_6, kAacHuff_7, kAacHuff_8, kAacHuff_9, kAacHuff_10, kAacHuff_11};
        const size_t n[11] = {81, 81, 81, 81, 81, 81, 64, 64, 169, 169, 289};
        for (int k = 0; k < 11; ++k) build_book(t.book[k], w[k], n[k]);
        build_book(t.book[11], kAacHuff_scf, 121);
        const float p43 = 4.0f / 3.0f;
        for (int i = 0; i < 8192; ++i) t.pow43[i] = powf(float(i), p43);                              // ics/mod.rs:44-50
        for (int i = 0; i < 256; ++i) t.normal_scf[i] = powf(2.0f, 0.25f * float(i - 56 - 100));      // :58-66
        for (int i = 0; i < 256; ++i) t.intensity_scf[i] = powf(0.5f, 0.25f * float(i - 155));        // :74-82
        for (int res = 0; res < 2; ++res) {                                                            // tns.rs:84-110
            const float fac = res ? 8.0f : 4.0f;
            const float half_pi = 1.57079632679489661923132169163975144f;
            const float iqfac = (fac - 0.5f) / half_pi, iqfac_m = (fac + 0.5f) / half_pi;
            for (int i = 0; i < 16; ++i) {
                const float c = float(i - 8);
                t.tns_sin[res][i] = sinf(c >= 0.0f ? c / iqfac : c / iqfac_m);
            }
        }
        for (int r = 0; r < 12; ++r) {
            std::memcpy(t.lng[r], kInfo[r].lng.v, kInfo[r].lng.len * sizeof(uint16_t));
            std::memcpy(t.shrt[r], kInfo[r].shrt.v, kInfo[r].shrt.len * sizeof(uint16_t));
            t.n_lng[r] = uint8_t(kInfo[r].lng.len), t.n_shrt[r] = uint8_t(kInfo[r].shrt.len);
            t.tns_max_long[r] = kTnsMaxLong[r], t.tns_max_short[r] = kTnsMaxShort[r];
        }
    }
};

// ---- BitReaderLtr for the AudioSpecificConfig parser: a failed read sticks, READ_OK() checks it --------------------------
struct Bits {
    const uint8_t* p;
    size_t n_bytes, n_bits, at = 0;
    bool ok = true;  // false: a read ran past the end (end_of_bitstream_error)
    Bits(const uint8_t* d, size_t n) : p(d), n_bytes(n), n_bits(n * 8) {}
    size_t left() const { return n_bits - at; }
    // The stream from `at` on, first bit in bit 63, zeros past the end; at least 57 bits are real or padding.
    uint64_t peek() const {
        const size_t byte = at >> 3;
        uint64_t v = 0;
        if (byte + 8 <= n_bytes) {
            std::memcpy(&v, p + byte, 8);
            v = __builtin_bswap64(v);
        } else {
            for (size_t k = 0; k < 8; ++k) v = (v << 8) | (byte + k < n_bytes ? p[byte + k] : 0u);
        }
        return v << (at & 7);
    }
    uint32_t read(uint32_t w) {  // w <= 32
        if (!ok || w > left()) return ok = false, 0;
        if (w == 0) return 0;
        const uint32_t v = uint32_t(peek() >> (64 - w));
        at += w;
        return v;
    }
    bool read_bool() { return read(1) == 1; }
};


struct Pair {  // cpe.rs:25-49
    bool is_pair;
    uint32_t channel;
    bool ms_used[8][64] = {};
    ae::Ics ics[2];
    ae::Lcg lcg;
    float coeffs[2][1024];
    Pair(bool pair, uint32_t ch, uint32_t rate_idx) : is_pair(pair), channel(ch) {
        for (int c = 0; c < 2; ++c) ae::init_ics(ics[c], rate_idx, coeffs[c]);
    }
};

#define CHECK(cond) \
    do {            \
        if (!(cond)) return SYMGPU_ERR_DECODE; \
    } while (0)
#define READ_OK() CHECK(bs.ok)

}  // namespace

const symgpu::aace::Tables& symgpu::aac_tables_host() {
    static const HostTables t;
    return t.t;
}

uint32_t symgpu::aac_rate_index(uint32_t sample_rate) {
    for (uint32_t i = 0; i < 12; ++i)
        if (sample_rate >= kInfo[i].min_rate) return i;
    return 11;
}

struct symgpu_aac_fe {
    uint32_t channels, rate_idx;
    bool stale = false;               // a pulse read a scale factor an earlier block left behind
    std::vector<std::unique_ptr<Pair>> pairs;
    std::vector<uint32_t> lcg_start;  // job mode: the noise generator's state when pair k is first seen

    // the stream's side of aac_entropy.h's decode_ga
    int set_pair(uint32_t pair_no, uint32_t channel, bool pair) {  // mod.rs:114-126
        if (pairs.size() <= pair_no) {
            pairs.emplace_back(new Pair(pair, channel, rate_idx));
            if (pair_no < lcg_start.size()) pairs.back()->lcg.state = lcg_start[pair_no];
        } else {
            CHECK(pairs[pair_no]->channel == channel);
            CHECK(pairs[pair_no]->is_pair == pair);
        }
        CHECK((pair ? channel + 1 : channel) < channels);
        return SYMGPU_OK;
    }
    ae::Ics& ics(uint32_t k, uint32_t c) { return pairs[k]->ics[c]; }
    ae::Lcg& lcg(uint32_t k) { return pairs[k]->lcg; }
    bool (&ms_used(uint32_t k))[8][64] { return pairs[k]->ms_used; }

    void apply_pulse(ae::Ics& s) {  // Pulse::synth, pulse.rs:60-105
        const ae::PulseLines p = ae::pulse_lines(symgpu::aac_tables_host(), s);
        float scale[4], value[4];
        for (uint32_t i = 0; i < p.n; ++i) {
            if (p.band[i] >= s.max_sfb) stale = true;
            scale[i] = s.scales[0][p.band[i]], value[i] = s.coeffs[p.line[i]];
        }
        ae::pulse_apply(p, scale, value);
        for (uint32_t i = 0; i < p.n; ++i) s.coeffs[p.line[i]] = value[i];
    }
};

extern "C" {

symgpu_status symgpu_aac_fe_create(uint32_t sample_rate, uint32_t channels, symgpu_aac_fe** out) {
    if (!out) return SYMGPU_ERR_ARG;
    *out = nullptr;
    if (channels < 1 || channels > 2) return SYMGPU_ERR_UNSUPPORTED;  // mod.rs:101-108 "aac too complex"
    symgpu_aac_fe* fe = new (std::nothrow) symgpu_aac_fe();
    if (!fe) return SYMGPU_ERR_LIMIT;
    fe->channels = channels;
    fe->rate_idx = symgpu::aac_rate_index(sample_rate);
    *out = fe;
    return SYMGPU_OK;
}

// AudioSpecificConfig::read, symphonia-common/src/mpeg/audio/mod.rs:230-439.  Object types by their MPEG-4 index (:87-130).
symgpu_status symgpu_aac_asc_parse(const uint8_t* buf, size_t n, symgpu_aac_asc* out) {
    if ((!buf && n) || !out) return SYMGPU_ERR_ARG;
    std::memset(out, 0, sizeof *out);
    Bits bs(buf, n);
    auto object_type = [&bs]() -> uint32_t {
        uint32_t v = bs.read(5);
        if (v == 31) v = bs.read(6) + 32;
        return v;
    };
    static const uint32_t kRates[13] = {96000, 88200, 64000, 48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000, 7350};
    auto sampling_frequency = [&bs](uint32_t& rate) -> symgpu_status {
        const uint32_t idx = bs.read(4);
        READ_OK();
        if (idx <= 12) rate = kRates[idx];
        else if (idx == 15) rate = bs.read(24);
        else return SYMGPU_ERR_DECODE;
        READ_OK();
        return SYMGPU_OK;
    };
    static const uint8_t kChannels[8] = {0, 1, 2, 3, 4, 5, 6, 8};
    auto channel_config = [&bs](uint8_t& ch) -> symgpu_status {  // 0: defined in-band
        const uint32_t idx = bs.read(4);
        READ_OK();
        CHECK(idx <= 7);
        ch = kChannels[idx];
        return SYMGPU_OK;
    };
    symgpu_status st;
    uint32_t aot = object_type();
    READ_OK();
    if ((st = sampling_frequency(out->sample_rate)) != SYMGPU_OK) return st;
    CHECK(out->sample_rate != 0);
    if ((st = channel_config(out->channels)) != SYMGPU_OK) return st;
    if (aot == 5 || aot == 29) {  // SBR / PS: explicit hierarchical signalling
        out->sbr_present = 1, out->ps_present = aot == 29, out->has_ext = 1;
        if ((st = sampling_frequency(out->ext_sample_rate)) != SYMGPU_OK) return st;
        aot = object_type();
        READ_OK();
        if (aot == 22 && (st = channel_config(out->ext_channels)) != SYMGPU_OK) return st;
    }
    out->object_type = uint8_t(aot > 255 ? 255 : aot);
    switch (aot) {
        case 1: case 2: case 3: case 6: case 7: case 17: case 19: case 20: case 21: case 22: case 23: {  // GASpecificConfig
            const bool short_frame = bs.read_bool();
            READ_OK();
            out->samples = short_frame ? 960 : 1024;
            const bool depends_on_core = bs.read_bool();
            READ_OK();
            if (depends_on_core) bs.read(14);
            const bool extension_flag = bs.read_bool();
            READ_OK();
            if (out->channels == 0) return SYMGPU_ERR_UNSUPPORTED;  // program config element
            if (aot == 6 || aot == 20) bs.read(3);
            READ_OK();
            if (extension_flag) {
                if (aot == 22) bs.read(5), bs.read(11);
                if (aot == 17 || aot == 19 || aot == 20 || aot == 23) bs.read(3);
                const bool extension_flag3 = bs.read_bool();
                READ_OK();
                if (extension_flag3) return SYMGPU_ERR_UNSUPPORTED;
            }
            break;
        }
        case 8: case 9: case 12: case 13: case 14: case 15: case 16: case 24: case 25: case 26: case 27: case 28: case 30: case 32: case 33: case 34:
        case 35: case 36: case 37: case 38: case 39: case 40: case 41:
            return SYMGPU_ERR_UNSUPPORTED;
        default: break;
    }
    if (aot == 17 || aot == 19 || aot == 20 || aot == 21 || aot == 22 || aot == 23) {  // (the other error-resilient types returned above)
        const uint32_t ep_config = bs.read(2);
        READ_OK();
        if (ep_config >= 2) return SYMGPU_ERR_UNSUPPORTED;
    }
    if (out->has_ext && bs.left() >= 16) {  // backward-compatible signalling behind the configuration
        const uint32_t sync = bs.read(11);
        if (sync == 0x2b7) {
            const uint32_t ext = object_type();
            READ_OK();
            if (ext == 5) {
                out->sbr_present = bs.read_bool();
                READ_OK();
                if (out->sbr_present) {
                    uint32_t r;
                    if ((st = sampling_frequency(r)) != SYMGPU_OK) return st;
                    if (bs.left() >= 12) {
                        if (bs.read(11) == 0x548) out->ps_present = bs.read_bool();
                        READ_OK();
                    }
                }
            }
            if (ext == 29) {
                out->sbr_present = bs.read_bool();
                READ_OK();
                if (out->sbr_present) {
                    uint32_t r;
                    if ((st = sampling_frequency(r)) != SYMGPU_OK) return st;
                }
                bs.read(4);
                READ_OK();
            }
        }
    }
    return SYMGPU_OK;
}

// AacDecoder::try_new with extra data (aac/mod.rs:59-108)
symgpu_status symgpu_aac_fe_create_asc(const uint8_t* extra, size_t n, symgpu_aac_fe** out, symgpu_aac_asc* asc_out) {
    if (!out || (!extra && n)) return SYMGPU_ERR_ARG;
    *out = nullptr;
    if (n < 2) return SYMGPU_ERR_DECODE;
    symgpu_aac_asc asc;
    const symgpu_status st = symgpu_aac_asc_parse(extra, n, &asc);
    if (asc_out) *asc_out = asc;
    if (st != SYMGPU_OK) return st;
    if (asc.channels == 0) return SYMGPU_ERR_UNSUPPORTED;  // "channels or channel layout is required"
    if (asc.object_type != 2 || asc.sbr_present || asc.channels > 2 || asc.samples != 1024) return SYMGPU_ERR_UNSUPPORTED;  // "aac too complex"
    return symgpu_aac_fe_create(asc.sample_rate, asc.channels, out);
}

void symgpu_aac_fe_destroy(symgpu_aac_fe* fe) { delete fe; }

void symgpu_aac_fe_reset(symgpu_aac_fe* fe) {  // AudioDecoder::reset -> ChannelPair::reset (the delay lines live with the synthesis stage)
    if (!fe) return;
    for (auto& p : fe->pairs) ae::reset_info(p->ics[0]), ae::reset_info(p->ics[1]);
}

symgpu_status symgpu_aac_fe_decode(symgpu_aac_fe* fe, const uint8_t* packet, size_t n, uint32_t tns_base, symgpu_aac_unit* units,
                                   symgpu_aac_tns* tns, uint32_t* n_tns, float* coeffs) {
    if (!fe || (!packet && n) || !units || !tns || !n_tns || !coeffs) return SYMGPU_ERR_ARG;
    *n_tns = 0;
    symgpu::mp3e::Bits bs(packet, n);
    uint32_t cur_pair = 0, cur_ch = 0;
    const int st = ae::decode_ga(bs, symgpu::aac_tables_host(), *fe, cur_pair, cur_ch);
    if (st != SYMGPU_OK) return symgpu_status(st);
    // the reference renders the channels its elements covered and leaves the others alone; the batch format carries every channel
    if (cur_ch != fe->channels) return SYMGPU_ERR_UNSUPPORTED;
    std::memset(units, 0, 2 * sizeof(symgpu_aac_unit));
    std::memset(coeffs, 0, 2 * 1024 * sizeof(float));
    uint32_t total = 0;
    for (size_t k = 0; k < cur_pair; ++k) {
        Pair& p = *fe->pairs[k];
        for (uint32_t c = 0; c < (p.is_pair ? 2u : 1u); ++c) {
            ae::Ics& ics = p.ics[c];
            const uint32_t ch = p.channel + c;
            fe->apply_pulse(ics);
            symgpu_aac_unit& u = units[ch];
            u.window_sequence = ics.window_sequence, u.window_shape = ics.window_shape, u.prev_window_shape = ics.prev_window_shape;
            std::memcpy(tns + total, ics.tns, ics.n_tns * sizeof(symgpu_aac_tns));
            u.n_tns = uint8_t(ics.n_tns), u.tns_first = ics.n_tns ? tns_base + total : 0;
            total += ics.n_tns;
            std::memcpy(coeffs + 1024 * ch, ics.coeffs, 1024 * sizeof(float));
        }
    }
    *n_tns = total;
    return SYMGPU_OK;
}

symgpu_status symgpu_aac_fe_decode_packets(symgpu_aac_fe* fe, const uint8_t* data, size_t n, const symgpu_piece* packets, size_t n_packets,
                                           uint32_t tns_base, symgpu_aac_unit* units, symgpu_aac_tns* tns, size_t tns_cap, float* coeffs,
                                           uint32_t* frame_of, size_t* n_good, size_t* n_tns) {
    if (!fe || (!data && n) || (n_packets && (!packets || !units || !coeffs || !frame_of)) || !n_good || !n_tns || (tns_cap && !tns)) return SYMGPU_ERR_ARG;
    size_t good = 0, total = 0;
    symgpu_aac_tns scratch[16];
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].len > n - packets[i].offset) continue;  // not inside the data: no packet
        uint32_t nt = 0;
        const symgpu_status st = symgpu_aac_fe_decode(fe, data + packets[i].offset, packets[i].len, uint32_t(tns_base + total), units + 2 * good, scratch,
                                                      &nt, coeffs + 2048 * good);
        if (st != SYMGPU_OK) continue;  // the caller of the reference drops the packet and goes on
        if (total + nt > tns_cap) return SYMGPU_ERR_LIMIT;
        std::memcpy(tns + total, scratch, nt * sizeof(symgpu_aac_tns));
        total += nt;
        frame_of[good++] = uint32_t(i);
    }
    *n_good = good, *n_tns = total;
    return SYMGPU_OK;
}

// Blocks of ONE stream as independent jobs (DESIGN 10.9): between raw_data_blocks only the previous window shape, the element layout
// and the noise generators carry over.  Pass A decodes every block with a fresh state on `n_threads` threads and counts each
// pair's noise draws; the generators' states at every block follow by jumping ahead over the prefix sums; pass B decodes again the
// blocks that drew noise, from the right states; window history is chained afterwards.  Exact for streams every block of which
// decodes with one element layout; anything else (a refused block, a changed layout, a pulse reading a scale an earlier block left
// behind) is SYMGPU_ERR_RESET: the caller takes the serial path, which keeps the reference's state across failures.
symgpu_status symgpu_aac_fe_decode_packets_jobs(uint32_t sample_rate, uint32_t channels, const uint8_t* data, size_t n, const symgpu_piece* packets,
                                                size_t n_packets, uint32_t tns_base, symgpu_aac_unit* units, symgpu_aac_tns* tns, size_t tns_cap,
                                                float* coeffs, size_t* n_tns, uint32_t n_threads) {
    if ((!data && n) || (n_packets && (!packets || !units || !coeffs)) || !n_tns || (tns_cap && !tns)) return SYMGPU_ERR_ARG;
    if (channels < 1 || channels > 2) return SYMGPU_ERR_UNSUPPORTED;
    n_threads = std::max<uint32_t>(1, std::min<uint32_t>({n_threads, 64u, std::max(1u, std::thread::hardware_concurrency()),
                                                           uint32_t(std::min<size_t>(std::max<size_t>(n_packets, 1), 64))}));
    try { // no C++ exception crosses the ABI (vector / thread creation may throw)
    struct Job {
        symgpu_status st = SYMGPU_OK;
        uint32_t n_pairs = 0, n_tns = 0;
        bool is_pair[2] = {false, false}, stale = false;
        uint64_t draws[2] = {0, 0};
        uint32_t start[2] = {0x1f2e3d4c, 0x1f2e3d4c};
        symgpu_aac_tns tns[16];
    };
    std::vector<Job> jobs(n_packets);
    auto run = [&](size_t i, bool with_start) {
        Job& j = jobs[i];
        symgpu_aac_fe* fe = nullptr;
        if (symgpu_aac_fe_create(sample_rate, channels, &fe) != SYMGPU_OK) return void(j.st = SYMGPU_ERR_LIMIT);
        if (with_start) fe->lcg_start.assign(j.start, j.start + 2);
        if (packets[i].offset > n || packets[i].len > n - packets[i].offset) j.st = SYMGPU_ERR_DECODE;
        else j.st = symgpu_aac_fe_decode(fe, data + packets[i].offset, packets[i].len, 0, units + 2 * i, j.tns, &j.n_tns, coeffs + 2048 * i);
        j.n_pairs = uint32_t(fe->pairs.size() < 2 ? fe->pairs.size() : 2);
        for (uint32_t k = 0; k < j.n_pairs; ++k) {
            const Pair& p = *fe->pairs[k];
            j.is_pair[k] = p.is_pair, j.draws[k] = p.lcg.draws;
        }
        j.stale = fe->stale;
        symgpu_aac_fe_destroy(fe);
    };
    auto parallel = [&](bool second) {
        std::vector<std::thread> pool;
        for (uint32_t t = 0; t < n_threads; ++t)
            pool.emplace_back([&, t] {
                for (size_t i = t; i < n_packets; i += n_threads)
                    if (!second || jobs[i].draws[0] || jobs[i].draws[1]) run(i, second);
            });
        for (auto& th : pool) th.join();
    };
    parallel(false);
    uint64_t total[2] = {0, 0};
    for (size_t i = 0; i < n_packets; ++i) {
        const Job& j = jobs[i];
        if (j.st != SYMGPU_OK || j.stale || j.n_pairs != jobs[0].n_pairs || j.is_pair[0] != jobs[0].is_pair[0] || j.is_pair[1] != jobs[0].is_pair[1])
            return SYMGPU_ERR_RESET;
        for (int k = 0; k < 2; ++k) jobs[i].start[k] = ae::Lcg::jump(ae::kLcgSeed, total[k]), total[k] += j.draws[k];
    }
    parallel(true);
    size_t at = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        Job& j = jobs[i];
        if (j.st != SYMGPU_OK) return SYMGPU_ERR_RESET;
        if (at + j.n_tns > tns_cap) return SYMGPU_ERR_LIMIT;
        uint32_t local = 0;
        for (uint32_t c = 0; c < 2; ++c) {
            symgpu_aac_unit& u = units[2 * i + c];
            u.prev_window_shape = i ? units[2 * (i - 1) + c].window_shape : 0;
            u.tns_first = u.n_tns ? uint32_t(tns_base + at + local) : 0;
            local += u.n_tns;
        }
        std::memcpy(tns + at, j.tns, j.n_tns * sizeof(symgpu_aac_tns));
        at += j.n_tns;
    }
    *n_tns = at;
    return SYMGPU_OK;
    } catch (...) {
        return SYMGPU_ERR_LIMIT;
    }
}

void symgpu_aac_fe_tables(float* pow43, float* normal_scf, float* intensity_scf) {
    const ae::Tables& T = symgpu::aac_tables_host();
    if (pow43) std::memcpy(pow43, T.pow43, sizeof T.pow43);
    if (normal_scf) std::memcpy(normal_scf, T.normal_scf, sizeof T.normal_scf);
    if (intensity_scf) std::memcpy(intensity_scf, T.intensity_scf, sizeof T.intensity_scf);
}

}  // extern "C"
