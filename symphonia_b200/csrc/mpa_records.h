// The C records of the MPEG index (include/symgpu.h symgpu_mpa_track / symgpu_mpa_packet) from packetizer.hpp's MpaTrack and
// MpaPacket, shared by symgpu_mpa_index (packetizer.cpp) and symgpu_mpa_index_dev (mpa_index_kernel.cu), so both write the same
// bytes.
#pragma once
#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

namespace symgpu_detail {

SYMGPU_PACKET_HD inline symgpu_mpa_track mpa_track_record(const symgpu::packet::MpaTrack& t) {
    symgpu_mpa_track r{};
    r.first_header = t.first_word, r.sample_rate = t.first.sample_rate;
    r.version = uint8_t(t.first.version), r.layer = t.first.layer, r.channels = uint8_t(t.first.n_channels());
    r.tag = uint8_t(t.tag), r.has_delay = t.has_delay, r.has_num_frames = t.has_num_frames;
    r.delay = t.delay, r.padding = t.padding, r.num_frames = t.num_frames, r.first_packet_pos = t.first_packet_pos;
    return r;
}

// `frame`: the packet's bytes, for main_data_begin.
SYMGPU_PACKET_HD inline symgpu_mpa_packet mpa_packet_record(const symgpu::packet::MpaPacket& p, const uint8_t* frame) {
    using namespace symgpu::packet;
    symgpu_mpa_packet o{};
    o.offset = p.offset, o.size = p.size, o.header = p.header, o.pts = p.pts, o.dur = p.dur, o.trim_start = p.trim_start, o.trim_end = p.trim_end;
    MpaHeader h{};
    mpa_parse_header(p.header, h);
    o.main_data_begin = h.layer == 3 ? mpa_main_data_begin(frame, p.size, h) : -1;
    return o;
}

}  // namespace symgpu_detail
