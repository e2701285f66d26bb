// ALAC front-end (include/symgpu.h "ALAC"): a stream's packets decoded on the CPU with the very functions the device decoder
// runs (alac_entropy.h) -- decode_packet, predict_channel per channel, finish_sample per sample -- so that the packet rules can
// be tested, plainly and under sanitizers, without a GPU.
#include <vector>

#include "../../include/symgpu.h"
#include "alac_entropy.h"

extern "C" symgpu_status symgpu_alac_fe_decode_packets(const uint8_t* data, size_t n, const symgpu_piece* packets, size_t n_packets,
                                                       const symgpu_alac_group* group, uint8_t* status, uint32_t* frames, int32_t* samples,
                                                       size_t samples_cap, size_t* n_samples) {
    if ((!data && n) || !group || !n_samples || (n_packets && (!packets || !status || !frames)) || (samples_cap && !samples)) return SYMGPU_ERR_ARG;
    if (group->channels < 1 || group->channels > 8 || group->bit_depth > 32 || group->frame_length > 65536) return SYMGPU_ERR_ARG;
    using namespace symgpu::alac;
    const Config cfg{group->frame_length, group->bit_depth, group->pb, group->mb, group->kb, group->channels};
    const uint32_t ch = cfg.channels, slot = cfg.frame_length;
    std::vector<int32_t> planes(size_t(ch) * slot);
    std::vector<uint16_t> tails(size_t(ch) * slot);
    Channel recs[8];
    size_t at = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].len > n - packets[i].offset) return SYMGPU_ERR_ARG;
        uint32_t got = 0;
        const int r = decode_packet(data + packets[i].offset, packets[i].len, cfg, recs, planes.data(), tails.data(), slot, &got);
        status[i] = uint8_t(r), frames[i] = 0;
        if (r != kDecoded) continue;
        if (size_t(got) * ch > samples_cap - at) return SYMGPU_ERR_LIMIT;
        for (uint32_t c = 0; c < ch; ++c) predict_channel(recs[c], planes.data() + size_t(c) * slot);
        for (uint32_t t = 0; t < got; ++t)
            for (uint32_t c = 0; c < ch; ++c) {
                const Channel& rc = recs[c];
                samples[at + size_t(t) * ch + c] = finish_sample(rc, planes.data() + size_t(c) * slot, planes.data() + size_t(rc.partner) * slot,
                                                                 tails.data() + size_t(c) * slot, t, cfg.bit_depth);
            }
        frames[i] = got;
        at += size_t(got) * ch;
    }
    *n_samples = at;
    return SYMGPU_OK;
}
