// The C records of the FLAC index (include/symgpu.h symgpu_flac_stream_info / symgpu_flac_packet) from packetizer.hpp's
// FlacStreamInfo and FlacPacket, shared by symgpu_flac_index (packetizer.cpp) and symgpu_flac_index_dev (flac_index_kernel.cu), so
// both write the same bytes.
#pragma once
#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

namespace symgpu_detail {

SYMGPU_PACKET_HD inline symgpu_flac_stream_info flac_info_record(const symgpu::packet::FlacStreamInfo& si, uint64_t first_frame_pos) {
    symgpu_flac_stream_info r{};
    r.n_samples = si.n_samples, r.first_frame_pos = first_frame_pos, r.sample_rate = si.sample_rate;
    r.frame_min = si.frame_min, r.frame_max = si.frame_max, r.block_min = si.block_min, r.block_max = si.block_max;
    r.channels = si.channels, r.bits_per_sample = si.bits_per_sample, r.has_md5 = si.has_md5;
    for (int k = 0; k < 16; ++k) r.md5[k] = si.md5[k];
    return r;
}

SYMGPU_PACKET_HD inline symgpu_flac_packet flac_packet_record(const symgpu::packet::FlacPacket& p) { return symgpu_flac_packet{p.offset, p.ts, p.size, p.dur}; }

}  // namespace symgpu_detail
