// Device helpers of the calls that build jobs from the tables of symgpu_ogg_index_dev (vorbis_jobs_kernel.cu, ogg_flac_jobs_kernel.cu):
// which file owns a packet, whether a file's tables were written, a packet's pieces copied by one warp, and the argument rules and
// grid sizes those calls share.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/symgpu.h"

namespace symgpu_detail {
namespace ogg_dev {

// The file that owns packet p of the table: the last whose first_packet <= p (an empty file shares first_packet with the next).
__device__ inline uint32_t file_of_packet(const symgpu_ogg_file_index* index, uint32_t n_files, uint64_t p) {
    uint32_t lo = 0, hi = n_files;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (index[mid].first_packet <= p) lo = mid;
        else hi = mid;
    }
    return lo;
}

// A file's tables are usable when they were written and lie inside the table of n_packets.
__device__ inline bool tables_ok(const symgpu_ogg_file_index& ix, uint64_t n_packets) {
    return !(ix.status & SYMGPU_OGG_NOT_WRITTEN) && ix.first_packet + ix.n_packets <= n_packets;
}

// One warp copies a packet's pieces back to back to dst.
__device__ inline void warp_copy_packet(uint8_t* dst, const uint8_t* d, const symgpu_piece* pc, uint32_t n_pieces) {
    const uint32_t lane = threadIdx.x & 31;
    uint64_t at = 0;
    for (uint32_t k = 0; k < n_pieces; ++k) {
        const symgpu_piece q = pc[k];
        for (uint32_t b = lane; b < q.len; b += 32) dst[at + b] = d[q.offset + b];
        at += q.len;
    }
}

// The argument rules the calls share with symgpu_ogg_index_dev.
inline symgpu_status check_files(const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files) {
    if ((n_bytes && !data) || (n_files && !files)) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_OGG_MAX_FILES) return SYMGPU_ERR_LIMIT;
    for (size_t i = 0; i < n_files; ++i)
        if (files[i].offset > n_bytes || files[i].len > n_bytes - files[i].offset) return SYMGPU_ERR_ARG;
    return SYMGPU_OK;
}

inline unsigned blocks_for(uint64_t threads, unsigned per_block) {
    const uint64_t b = (threads + per_block - 1) / per_block;
    return unsigned(b == 0 ? 1 : b < 65535 * 8 ? b : 65535 * 8);
}

}  // namespace ogg_dev
}  // namespace symgpu_detail
