// FLAC-in-Ogg jobs built on the device from the tables of symgpu_ogg_index_dev (DESIGN §5b / §5e, include/symgpu.h): what
// decode.ogg_flac_index chooses for each file, as the job table symgpu_flac_decode_fmt_dev takes.  The per-file and per-packet
// rules are functions of include/symgpu/packetizer.hpp that tests/cpp/ogg_flac_jobs_driver.cpp also runs on the CPU
// (ogg_first_stream_len, ogg_flac_ident, ogg_flac_is_audio, ogg_flac_packet_block).  What a host walk does packet after packet is
// done here by a scan:
//   symgpu_ogg_flac_heads_dev  1. ogg_flac_heads_kernel, one thread per file: the stream's end and its identification packet;
//                              2. ogg_flac_audio_kernel, one thread per packet: is it an audio packet, and its block size;
//                              3. exclusive_scan_kernel (block_scan.cuh), one block: audio packets, bytes and slots before each;
//                              4. ogg_flac_totals_kernel, one thread per file: its audio packets, bytes and slots.
//   symgpu_ogg_flac_jobs_dev   ogg_flac_job_kernel, one warp per packet: bytes gathered, job written.
#include <cuda_runtime.h>

#include "../../include/symgpu/packetizer.hpp"
#include "batch_call.h"
#include "block_scan.cuh"
#include "flac_records.h"
#include "ogg_device.cuh"

namespace {

using namespace symgpu::packet;
using namespace symgpu_detail;
using namespace symgpu_detail::ogg_dev;

__global__ void ogg_flac_heads_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                      const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets, const symgpu_piece* __restrict__ pieces,
                                      const symgpu_ogg_file_index* __restrict__ index, const uint32_t* __restrict__ group_of, uint32_t n_groups,
                                      symgpu_ogg_flac_file* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files || group_of[i] >= n_groups) return;
    const symgpu_ogg_file_index ix = index[i];
    symgpu_ogg_flac_file h{};
    if (ix.n_packets == 0 || !tables_ok(ix, n_packets)) {
        h.status = SYMGPU_OGG_FLAC_NO_PACKETS;
    } else {
        const symgpu_ogg_packet* pk = packets + ix.first_packet;
        const symgpu_piece* pc = pieces + ix.first_piece;
        h.n_stream = ogg_first_stream_len(pk, ix.n_packets);
        uint8_t id[kOggFlacIdentLen];
        FlacStreamInfo si{};
        const uint32_t got = pk[0].len == kOggFlacIdentLen ? ogg_packet_head(data + files[i].offset, pc + pk[0].first_piece, pk[0].n_pieces, id, kOggFlacIdentLen) : 0;
        const Status s = got == kOggFlacIdentLen ? ogg_flac_ident(id, got, si) : Status::Unsupported;
        if (s == Status::Ok) h.info = symgpu_detail::flac_info_record(si, 0);
        else h.status = s == Status::Unsupported ? SYMGPU_OGG_FLAC_NOT_FLAC : SYMGPU_OGG_FLAC_BAD_STREAMINFO;
    }
    heads[group_of[i]] = h;
}

// ranks[p]: audio, slot, and the values the scan sums in place (1, the packet's length, its slot for an audio packet).
__global__ void ogg_flac_audio_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                      const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets, const symgpu_piece* __restrict__ pieces,
                                      const symgpu_ogg_file_index* __restrict__ index, const uint32_t* __restrict__ group_of, uint32_t n_groups,
                                      const symgpu_ogg_flac_file* __restrict__ heads, symgpu_ogg_flac_packet_rank* ranks) {
    for (uint64_t p = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < n_packets; p += uint64_t(gridDim.x) * blockDim.x) {
        const uint32_t f = file_of_packet(index, n_files, p);
        const symgpu_ogg_file_index ix = index[f];
        const uint32_t g = group_of[f];
        symgpu_ogg_flac_packet_rank r{};
        if (g < n_groups && p >= ix.first_packet && p - ix.first_packet < ix.n_packets) {
            const symgpu_ogg_flac_file h = heads[g];
            const uint32_t k = uint32_t(p - ix.first_packet);
            const symgpu_ogg_packet pk = packets[p];
            const uint8_t* d = data + files[f].offset;
            const symgpu_piece* pc = pieces + ix.first_piece + pk.first_piece;
            uint8_t b0 = 0;
            if (h.status == 0 && k > 0 && k < h.n_stream && ogg_packet_head(d, pc, pk.n_pieces, &b0, 1) == 1 && ogg_flac_is_audio(uint32_t(pk.len), b0)) {
                r.audio = 1, r.rank = 1, r.byte_at = pk.len;
                r.slot = ogg_flac_packet_block(d, pc, pk.n_pieces);
                r.samples_at = r.slot;
            }
        }
        ranks[p] = r;
    }
}

// Exclusive sums of audio packets, their bytes and their slots over the whole table (each field holds its own value before).
struct RankSums {
    static constexpr int kN = 3;
    __device__ uint64_t get(const symgpu_ogg_flac_packet_rank& r, int k) const { return k == 0 ? r.rank : k == 1 ? r.byte_at : r.samples_at; }
    __device__ void put(symgpu_ogg_flac_packet_rank& r, int k, uint64_t before) const { (k == 0 ? r.rank : k == 1 ? r.byte_at : r.samples_at) = before; }
};

__global__ void ogg_flac_totals_kernel(const symgpu_ogg_file_index* __restrict__ index, uint32_t n_files, const uint32_t* __restrict__ group_of,
                                       uint32_t n_groups, const symgpu_ogg_flac_packet_rank* __restrict__ ranks, const symgpu_ogg_packet* __restrict__ packets,
                                       symgpu_ogg_flac_file* heads) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files || group_of[i] >= n_groups) return;
    symgpu_ogg_flac_file& h = heads[group_of[i]];
    if (h.status) return;
    const symgpu_ogg_file_index ix = index[i];
    const uint64_t first = ix.first_packet, last = first + ix.n_packets - 1;
    const symgpu_ogg_flac_packet_rank a = ranks[first], z = ranks[last];
    h.n_audio = uint32_t(z.rank + z.audio - a.rank);
    h.audio_bytes = z.byte_at + (z.audio ? packets[last].len : 0) - a.byte_at;
    h.samples = z.samples_at + z.slot - a.samples_at;
}

__global__ void ogg_flac_job_kernel(const uint8_t* __restrict__ data, const symgpu_file_range* __restrict__ files, uint32_t n_files,
                                    const symgpu_ogg_packet* __restrict__ packets, uint64_t n_packets, const symgpu_piece* __restrict__ pieces,
                                    const symgpu_ogg_file_index* __restrict__ index, const uint32_t* __restrict__ group_of,
                                    const symgpu_ogg_flac_packet_rank* __restrict__ ranks, uint8_t* out, uint64_t out_cap, symgpu_flac_job* jobs,
                                    uint64_t n_jobs) {
    const uint64_t warps = uint64_t(gridDim.x) * (blockDim.x / 32);
    for (uint64_t p = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) / 32; p < n_packets; p += warps) {
        const symgpu_ogg_flac_packet_rank rk = ranks[p];
        if (!rk.audio) continue;
        const symgpu_ogg_packet pk = packets[p];
        if (rk.rank >= n_jobs || rk.byte_at > out_cap || pk.len > out_cap - rk.byte_at) continue;
        const uint32_t f = file_of_packet(index, n_files, p);
        const symgpu_ogg_file_index ix = index[f];
        warp_copy_packet(out + rk.byte_at, data + files[f].offset, pieces + ix.first_piece + pk.first_piece, pk.n_pieces);
        if ((threadIdx.x & 31) == 0) jobs[rk.rank] = symgpu_flac_job{rk.byte_at, uint32_t(pk.len), group_of[f], rk.slot, 0};
    }
}

// The files and their groups staged; SYMGPU_ERR_ARG for groups that do not rise with the file index or pass n_groups.
symgpu_status stage_files(symgpu_ctx* ctx, const symgpu_file_range* files, size_t n_files, const uint32_t* group_of, size_t n_groups,
                          symgpu_file_range** d_files, uint32_t** d_group_of) {
    uint64_t next = 0;
    for (size_t i = 0; i < n_files; ++i) {
        if (group_of[i] == SYMGPU_OGG_FLAC_NO_GROUP) continue;
        if (group_of[i] < next || group_of[i] >= n_groups) return SYMGPU_ERR_ARG;
        next = uint64_t(group_of[i]) + 1;
    }
    Carver c;
    const size_t at_files = c.take(n_files * sizeof(symgpu_file_range)), at_groups = c.take(n_files * 4);
    symgpu_status e = ensure_stage(ctx, c.at);
    if (e != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    *d_files = reinterpret_cast<symgpu_file_range*>(stage + at_files);
    *d_group_of = reinterpret_cast<uint32_t*>(stage + at_groups);
    CU(ctx, cudaMemcpyAsync(*d_files, files, n_files * sizeof(symgpu_file_range), cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaMemcpyAsync(*d_group_of, group_of, n_files * 4, cudaMemcpyHostToDevice, ctx->stream));
    return SYMGPU_OK;
}

}  // namespace

extern "C" symgpu_status symgpu_ogg_flac_heads_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                                   const symgpu_ogg_packet* packets, size_t n_packets, const symgpu_piece* pieces,
                                                   const symgpu_ogg_file_index* index, const uint32_t* group_of, size_t n_groups,
                                                   symgpu_ogg_flac_file* heads, symgpu_ogg_flac_packet_rank* ranks) {
    if (!ctx || (n_files && (!index || !group_of)) || (n_groups && !heads) || (n_packets && (!packets || !pieces || !ranks))) return SYMGPU_ERR_ARG;
    symgpu_status e = check_files(data, n_bytes, files, n_files);
    if (e != SYMGPU_OK) return e;
    if (n_groups > SYMGPU_OGG_MAX_FILES) return SYMGPU_ERR_LIMIT;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    symgpu_file_range* d_files;
    uint32_t* d_groups;
    if ((e = stage_files(ctx, files, n_files, group_of, n_groups, &d_files, &d_groups)) != SYMGPU_OK) return e;
    cudaStream_t st = ctx->stream;
    const uint32_t nf = uint32_t(n_files), ng = uint32_t(n_groups);
    ogg_flac_heads_kernel<<<(nf + 127) / 128, 128, 0, st>>>(data, d_files, nf, packets, n_packets, pieces, index, d_groups, ng, heads);
    CU(ctx, cudaGetLastError());
    ogg_flac_audio_kernel<<<blocks_for(n_packets, 256), 256, 0, st>>>(data, d_files, nf, packets, n_packets, pieces, index, d_groups, ng, heads, ranks);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(ranks, uint64_t(n_packets), RankSums{});
    CU(ctx, cudaGetLastError());
    ogg_flac_totals_kernel<<<(nf + 127) / 128, 128, 0, st>>>(index, nf, d_groups, ng, ranks, packets, heads);
    CU(ctx, cudaGetLastError());
    ctx->launches += 4;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_ogg_flac_jobs_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                                  const symgpu_ogg_packet* packets, size_t n_packets, const symgpu_piece* pieces,
                                                  const symgpu_ogg_file_index* index, const uint32_t* group_of,
                                                  const symgpu_ogg_flac_packet_rank* ranks, uint8_t* out, size_t out_cap, symgpu_flac_job* jobs,
                                                  size_t n_jobs) {
    if (!ctx || (n_files && (!index || !group_of)) || (n_packets && (!packets || !pieces || !ranks)) || (out_cap && !out) || (n_jobs && !jobs))
        return SYMGPU_ERR_ARG;
    symgpu_status e = check_files(data, n_bytes, files, n_files);
    if (e != SYMGPU_OK) return e;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    symgpu_file_range* d_files;
    uint32_t* d_groups;
    if ((e = stage_files(ctx, files, n_files, group_of, SYMGPU_OGG_MAX_FILES, &d_files, &d_groups)) != SYMGPU_OK) return e;
    ogg_flac_job_kernel<<<blocks_for(uint64_t(n_packets) * 32, 256), 256, 0, ctx->stream>>>(data, d_files, uint32_t(n_files), packets, n_packets, pieces,
                                                                                            index, d_groups, ranks, out, out_cap, jobs, n_jobs);
    CU(ctx, cudaGetLastError());
    ++ctx->launches;
    return SYMGPU_OK;
}
