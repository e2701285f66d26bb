// The symgpu_caf_info record of an opened (or refused) CAF file, shared by the host index (packetizer.cpp) and the device index
// (caf_index_kernel.cu) so that their records are equal byte for byte.
#pragma once
#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

namespace symgpu_detail {

// n_packets is left 0: the caller counts the packets that fit.
SYMGPU_PACKET_HD inline symgpu_caf_info caf_info_record(const symgpu::packet::CafAlac& a, symgpu::packet::Status s) {
    using symgpu::packet::Status;
    symgpu_caf_info r{};
    r.open = uint8_t(s == Status::Ok ? SYMGPU_OK : s == Status::Unsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE);
    r.reason = a.reason;
    if (s != Status::Ok) return r;
    r.data_start = a.data_start, r.table_at = a.table_at, r.table_bytes = a.table_bytes, r.table_packets = a.table_packets;
    r.valid_frames = a.valid_frames, r.priming_frames = a.priming_frames, r.remainder_frames = a.remainder_frames;
    r.frames_per_packet = a.frames_per_packet, r.frame_length = a.frame_length, r.max_frame_bytes = a.max_frame_bytes;
    r.avg_bit_rate = a.avg_bit_rate, r.sample_rate = a.sample_rate, r.max_run = a.max_run, r.compatible_version = a.compatible_version;
    r.bit_depth = a.bit_depth, r.pb = a.pb, r.mb = a.mb, r.kb = a.kb, r.channels = a.channels;
    return r;
}

}  // namespace symgpu_detail
