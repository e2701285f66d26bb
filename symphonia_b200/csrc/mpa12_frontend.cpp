// MPEG Layer I / II sample decoders (include/symgpu.h, SURVEY §8f N1): bit allocation, scale factors, (de)grouping and
// dequantisation -- everything Layer1::decode / Layer2::decode do before they call the polyphase synthesis
// (symphonia-bundle-mp3/src/layer1/mod.rs:73-176, layer2/mod.rs:214-369).  The rules themselves are mpa12_entropy.h, shared
// with the device decoder (mpa12_decode_kernel.cu); this file is the CPU loop over them and the constants' computation.
//
// The arithmetic is the reference's, operation for operation (f32, no contraction: the Makefile passes
// -ffp-contract=off): Layer I  sample = scalefactor * (factor[nb] * (a + 1)),  factor = (2^nb / (2^nb - 1)) * (1 / 2^(nb-1));
// Layer II sample = scalefactor * (C * (a / 2^(b-1) + D)).  The constants are closed forms that reproduce the reference's
// decimal literals bit for bit (tests/golden/mpa12_constants.json): scalefactor[i] = (float)2^(1 - i/3); C = (float)(2^b / L)
// for L quantisation levels, b = ceil(log2(L + 1)); D = 1/2 for the grouped classes, else 2^-(b-1) as the 11-decimal
// number the standard's table prints (which for b = 15, 16 is one ulp above the power of two).
#include <cmath>
#include <cstring>

#include "../../include/symgpu.h"
#include "mpa12_entropy.h"

namespace symgpu {
namespace mpa12e {

const Constants& host_constants() {
    static const Constants K = [] {
        Constants c{};
        for (int i = 0; i < 63; ++i) c.scale[i] = float(std::pow(2.0, 1.0 - i / 3.0));
        c.scale[63] = 0.0f;  // not in the standard; files use it (layer12.rs:71-74)
        for (int nb = 0; nb < 16; ++nb) c.factor[nb] = 0.0f;
        for (int nb = 2; nb < 16; ++nb) {
            const int a = 1 << nb, b = 1 << (nb - 1);
            c.factor[nb] = (float(a) / float(a - 1)) * (1.0f / float(b));
        }
        static const uint16_t levels[17] = {3, 5, 7, 9, 15, 31, 63, 127, 255, 511, 1023, 2047, 4095, 8191, 16383, 32767, 65535};
        for (int k = 0; k < 17; ++k) {
            QuantClass& q = c.cls[k];
            q.levels = levels[k];
            int b = 0;
            while ((1u << b) < unsigned(levels[k]) + 1) ++b;
            q.bits = uint8_t(b);
            q.inv_divisor = float(std::ldexp(1.0, -(b - 1)));
            q.grouped = levels[k] == 3 || levels[k] == 5 || levels[k] == 9;
            q.read_bits = uint8_t(q.grouped ? (levels[k] == 3 ? 5 : levels[k] == 5 ? 7 : 10) : b);
            q.c = float(double(1u << b) / double(levels[k]));
            q.d = q.grouped ? 0.5f : float(std::round(std::ldexp(1.0, -(b - 1)) * 1e11) / 1e11);
        }
        return c;
    }();
    return K;
}

}  // namespace mpa12e
}  // namespace symgpu

namespace {

using namespace symgpu::mpa12e;

struct Spec {
    bool have = false;
    uint32_t rate = 0;
    int channels = 0;
};

// The packet rules of mpa12_entropy.h in the reference's order; the samples are decoded granule by granule, each codeword at
// its closed-form position.
symgpu_status decode_packet(Spec* spec, const uint8_t* frame, size_t n, int layer, float* subbands, symgpu_mp3_frame_info* info) {
    MpaHeader h{};
    size_t q = 0;
    const int hs = read_header(frame, n, h, q);
    if (hs != kDecoded) return hs == kUnsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE;
    if (spec) {
        if (!spec->have) spec->have = true, spec->rate = h.sample_rate, spec->channels = h.n_channels();
        else if (spec->rate != h.sample_rate || spec->channels != h.n_channels()) return SYMGPU_ERR_DECODE;
    }
    Side s;
    if (!body_of(h, layer, n, q, s.body_at, s.body_bytes)) return SYMGPU_ERR_DECODE;
    const int n_slots = layer == 1 ? 12 : 36, per = layer == 1 ? 1 : 3;
    std::memset(subbands, 0, sizeof(float) * 2 * 32 * n_slots);
    const Constants& K = host_constants();
    const uint8_t* body = frame + s.body_at;
    if (!read_side(K, body, h, s) || !fits(s)) return SYMGPU_ERR_DECODE;
    for (int gr = 0; gr < 12; ++gr)
        for (int sb = 0; sb < s.sblimit; ++sb)
            for (int c = 0; c < s.n_ch; ++c)
                if (!decode_codeword(K, s, body, gr, sb, c, subbands + (c * 32 + sb) * n_slots + gr * per)) return SYMGPU_ERR_DECODE;
    if (info) {
        *info = symgpu_mp3_frame_info{};
        info->sample_rate = h.sample_rate, info->channels = uint8_t(h.n_channels()), info->granules = 1;
        info->sample_rate_idx = h.sample_rate_idx, info->version = uint8_t(h.version);
    }
    return SYMGPU_OK;
}

}  // namespace

extern "C" symgpu_status symgpu_mpa12_fe_decode(const uint8_t* frame, size_t n, int layer, float* subbands, symgpu_mp3_frame_info* info) {
    if ((!frame && n) || !subbands || (layer != 1 && layer != 2)) return SYMGPU_ERR_ARG;
    return decode_packet(nullptr, frame, n, layer, subbands, info);
}

extern "C" symgpu_status symgpu_mpa12_fe_decode_packets(const uint8_t* data, size_t n, const symgpu_mpa_packet* packets, size_t n_packets, int layer,
                                                        float* subbands, uint32_t* frame_of, size_t* n_good, symgpu_mp3_frame_info* info) {
    if ((!data && n) || !n_good || (layer != 1 && layer != 2) || (n_packets && (!packets || !subbands || !frame_of))) return SYMGPU_ERR_ARG;
    const size_t per_frame = size_t(2) * 32 * (layer == 1 ? 12 : 36);
    Spec spec;
    size_t good = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].size > n - packets[i].offset) return SYMGPU_ERR_ARG;
        symgpu_mp3_frame_info fi;
        if (decode_packet(&spec, data + packets[i].offset, packets[i].size, layer, subbands + good * per_frame, &fi) != SYMGPU_OK) continue;
        if (good == 0 && info) *info = fi;
        frame_of[good++] = uint32_t(i);
    }
    *n_good = good;
    return SYMGPU_OK;
}

extern "C" size_t symgpu_mpa12_constants(float* out, size_t cap) {
    const Constants& K = host_constants();
    float all[98];
    std::memcpy(all, K.scale, sizeof K.scale);
    for (int k = 0; k < 17; ++k) all[64 + k] = K.cls[k].c, all[81 + k] = K.cls[k].d;
    if (out) std::memcpy(out, all, sizeof(float) * std::min<size_t>(cap, 98));
    return 98;
}
