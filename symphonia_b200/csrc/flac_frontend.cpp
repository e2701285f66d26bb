// FLAC front-end (include/symgpu.h "FLAC front-end", SURVEY §8f N1 for the FLAC row): frame header, sub-frame headers,
// warm-up samples, quantised predictor coefficients and Rice-coded residuals -- everything FlacDecoder::decode_inner
// reads from the bitstream (symphonia-bundle-flac/src/frame.rs, decoder.rs:139-640) -- into the descriptor tables and the
// sample buffer of symgpu_flac_restore_*.  The per-packet rules live in flac_entropy.h, shared with the device decoder
// (flac_decode_kernel.cu); this loop packs the accepted packets densely.  Prediction, wasted-bit shifts, decorrelation
// and scaling are NOT done here: they are the data-parallel half (flac_kernel.cu / oracle_flac.cpp).
#include "../../include/symgpu.h"
#include "flac_entropy.h"

extern "C" symgpu_status symgpu_flac_fe_decode_packets(const uint8_t* data, size_t n, const symgpu_piece* packets, size_t n_packets,
                                                       uint32_t stream_bps, uint32_t stream_channels, uint32_t max_block,
                                                       symgpu_flac_frame* frames, symgpu_flac_frame_info* infos, uint32_t* frame_of,
                                                       symgpu_flac_subframe* subs, size_t subs_cap, int32_t* samples, size_t samples_cap,
                                                       size_t* n_good, size_t* n_subs, size_t* n_samples) {
    if ((!data && n) || !n_good || !n_subs || !n_samples || (n_packets && (!packets || !frames || !infos || !frame_of || !subs || !samples)))
        return SYMGPU_ERR_ARG;
    size_t good = 0, sub_at = 0, smp_at = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].len > n - packets[i].offset) return SYMGPU_ERR_ARG;
        const int r = symgpu::flace::decode_packet(data + packets[i].offset, packets[i].len, stream_bps, stream_channels, max_block, uint32_t(sub_at),
                                                   subs + sub_at, subs_cap - sub_at, samples + smp_at, smp_at, samples_cap - smp_at, ~0u,
                                                   frames + good, infos + good);
        if (r == symgpu::flace::kNoRoom) return SYMGPU_ERR_LIMIT;
        if (r != symgpu::flace::kDecoded) continue;
        const uint32_t channels = frames[good].channels, block = infos[good].block_size;
        frame_of[good++] = uint32_t(i);
        sub_at += channels, smp_at += size_t(channels) * block;
    }
    *n_good = good, *n_subs = sub_at, *n_samples = smp_at;
    return SYMGPU_OK;
}
