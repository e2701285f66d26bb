// symgpu_mpa_index_dev: the MPEG audio frame index of many files already in device memory (DESIGN §5b, include/symgpu.h).  Every
// per-candidate step is a function of include/symgpu/packetizer.hpp that tests/cpp/mpa_index_driver.cpp also runs on the CPU, and
// MpaIndexer (symgpu_mpa_index) is a loop over the same functions.  The files' bytes form one virtual byte space, cut into tiles of
// 4096 bytes, one block each:
//   1. candidate_count_kernel (candidate_tiles.cuh): the sync candidates of each tile;
//   2. exclusive_scan_kernel (block_scan.cuh): each tile's first candidate, and the total, which is read back (the one host wait)
//      to size the per-candidate scratch;
//   3. candidates_kernel: each candidate's virtual position and node word (mpa_node), in order;
//   4. mpa_successor_kernel: the packet successor S (mpa_successor) and the first-frame hunt step G (mpa_hunt);
//   5. H x mpa_hunt_kernel, H = mpa_hunt_rounds(longest file): G^(2^H) by pointer jumping;
//   6. mpa_track_kernel, one thread per file: the root its first candidate's hunt ends at is its first frame A (rank 0), whose
//      track open() reads (mpa_open_track: the tag, the estimate -- bounded work);
//   7. K x chain_double_kernel, K = mpa_chain_rounds(longest file): every node of each S-chain from A ranked by pointer doubling;
//   8. mpa_dur_kernel: each candidate's packet samples (mpa_packet_dur, 0 for no packet), summed per tile of 4096 candidates;
//   9. exclusive_scan_kernel: each candidate tile's first packet and samples;
//  10. mpa_rank_kernel: each candidate's packet index and samples before it, over all files (exclusive scans over candidate order:
//      a chain rises in position, so this is chain order);
//  11. mpa_record_kernel: each file's first packet and packet count from the scans at its first candidates, and the capacity check;
//  12. mpa_packet_kernel: the packets and jobs, one thread per packet, its pts -delay + the samples before it in its file.
#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/symgpu/packetizer.hpp"
#include "candidate_tiles.cuh"
#include "mpa_records.h"

namespace {

using namespace symgpu::packet;
using namespace symgpu_detail;

static_assert(sizeof(symgpu_mpa_file_index) == 16, "record sizes are ABI");
static_assert(sizeof(symgpu_mp3_job) == sizeof(symgpu_mpa12_job) && offsetof(symgpu_mp3_job, offset) == offsetof(symgpu_mpa12_job, offset) &&
                  offsetof(symgpu_mp3_job, len) == offsetof(symgpu_mpa12_job, len) &&
                  offsetof(symgpu_mp3_job, trim_start) == offsetof(symgpu_mpa12_job, trim_start) &&
                  offsetof(symgpu_mp3_job, trim_end) == offsetof(symgpu_mpa12_job, trim_end),
              "one job table feeds the Layer III and the Layer I / II decoders");

__constant__ detail::Crc16Table kCrc16;  // the LAME tag's CRC-16 table

struct MpaRule {
    __device__ static bool is_candidate(const uint8_t* d, size_t n, size_t q) { return mpa_is_candidate(d, n, q); }
    __device__ static uint32_t node(const uint8_t* d, size_t n, size_t q) { return mpa_node(d, n, q); }
};

constexpr uint32_t kCandPerThread = 16, kCandTile = kTileThreads * kCandPerThread;

__global__ void mpa_successor_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                     const uint64_t* __restrict__ vpos, uint32_t n_cand, const uint32_t* __restrict__ node, uint32_t* __restrict__ jump,
                                     uint32_t* __restrict__ hunt, uint32_t* __restrict__ rank) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) {
        const FileDev f = files[file_of(files, n_files, vpos[c])];
        const uint64_t end = f.vbase + f.len;
        const uint32_t nd = node[c], s = mpa_successor(vpos, n_cand, c, nd, end);
        jump[c] = s;
        hunt[c] = mpa_hunt(vpos, n_cand, c, nd, mpa_first_rejected(data + f.offset, size_t(f.len), size_t(vpos[c] - f.vbase), nd), s, end);
        rank[c] = kAdtsUnranked;
    }
}

__global__ void mpa_hunt_kernel(const uint32_t* __restrict__ hunt, uint32_t* __restrict__ next, uint32_t n_cand) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) mpa_hunt_jump(hunt, next, c);
}

// fcand[i]: file i's first candidate (fcand[n_files] = n_cand); the file's track, and its first frame ranked 0.
__global__ void mpa_track_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos,
                                 uint32_t n_cand, const uint32_t* __restrict__ node, const uint32_t* __restrict__ hunt, bool seekable,
                                 uint32_t* __restrict__ fcand, uint32_t* __restrict__ rank, MpaTrack* __restrict__ ftrack, symgpu_mpa_track* __restrict__ tracks,
                                 symgpu_mpa_file_index* __restrict__ index) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_files; i += gridDim.x * blockDim.x) {
        const FileDev f = files[i];
        const uint32_t c0 = detail::first_at_or_after(vpos, 0, n_cand, f.vbase);
        fcand[i] = c0;
        if (i == 0) fcand[n_files] = n_cand;
        const uint32_t root = c0 < n_cand && vpos[c0] < f.vbase + f.len ? hunt[c0] : kMpaEnd;
        MpaTrack t{};
        if (root == kMpaEnd || mpa_node_kind(node[root]) != kMpaFrame) {
            index[i].status = SYMGPU_MPA_NO_FRAME;
            ftrack[i] = t;
            tracks[i] = symgpu_mpa_track{};
            continue;
        }
        mpa_open_track(kCrc16.t, data + f.offset, size_t(f.len), size_t(vpos[root] - f.vbase), seekable, t);
        rank[root] = 0;
        ftrack[i] = t;
        tracks[i] = mpa_track_record(t);
    }
}

struct CandTile {
    uint64_t packets, samples;
};
struct CandFirsts {
    static constexpr int kN = 2;
    __device__ uint64_t get(const CandTile& r, int k) const { return k ? r.samples : r.packets; }
    __device__ void put(CandTile& r, int k, uint64_t before) const { (k ? r.samples : r.packets) = before; }
};

__global__ void __launch_bounds__(kTileThreads) mpa_dur_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                                               const uint64_t* __restrict__ vpos, uint32_t n_cand, const uint32_t* __restrict__ node,
                                                               const uint32_t* __restrict__ rank, const MpaTrack* __restrict__ ftrack,
                                                               uint32_t* __restrict__ dur, uint64_t n_tiles, CandTile* __restrict__ tiles) {
    if (blockIdx.x == 0 && threadIdx.x == 0) tiles[n_tiles] = CandTile{0, 0};  // scanned into the totals
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t v[2] = {0, 0}, before[2], sum[2];
        const uint64_t c0 = t * kCandTile + uint64_t(threadIdx.x) * kCandPerThread;
        for (uint64_t c = c0; c < c0 + kCandPerThread && c < n_cand; ++c) {
            uint32_t d = 0;
            if (rank[c] != kAdtsUnranked) {
                const uint32_t i = file_of(files, n_files, vpos[c]);
                const FileDev f = files[i];
                d = mpa_packet_dur(kCrc16.t, data + f.offset, size_t(vpos[c] - f.vbase), node[c], rank[c], uint8_t(ftrack[i].tag));
            }
            dur[c] = d;
            v[0] += d != 0, v[1] += d;
        }
        block_exclusive_sums<2>(v, before, sum);
        if (threadIdx.x == 0) tiles[t] = CandTile{sum[0], sum[1]};
    }
}

// pidx[c] / before[c]: the packets / samples of the candidates before c, over all files; pidx[n_cand] / before[n_cand]: the totals.
__global__ void __launch_bounds__(kTileThreads) mpa_rank_kernel(uint32_t n_cand, const uint32_t* __restrict__ dur, uint64_t n_tiles,
                                                                const CandTile* __restrict__ tiles, uint32_t* __restrict__ pidx,
                                                                uint64_t* __restrict__ samples_before) {
    if (blockIdx.x == 0 && threadIdx.x == 0) pidx[n_cand] = uint32_t(tiles[n_tiles].packets), samples_before[n_cand] = tiles[n_tiles].samples;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t v[2] = {0, 0}, before[2], sum[2];
        const uint64_t c0 = t * kCandTile + uint64_t(threadIdx.x) * kCandPerThread;
        for (uint64_t c = c0; c < c0 + kCandPerThread && c < n_cand; ++c) v[0] += dur[c] != 0, v[1] += dur[c];
        block_exclusive_sums<2>(v, before, sum);
        uint64_t p = tiles[t].packets + before[0], s = tiles[t].samples + before[1];
        for (uint64_t c = c0; c < c0 + kCandPerThread && c < n_cand; ++c) {
            pidx[c] = uint32_t(p), samples_before[c] = s;
            p += dur[c] != 0, s += dur[c];
        }
    }
}

__global__ void mpa_record_kernel(uint32_t n_files, const uint32_t* __restrict__ fcand, const uint32_t* __restrict__ pidx, uint64_t cap,
                                  symgpu_mpa_file_index* __restrict__ index) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_files; i += gridDim.x * blockDim.x) {
        const uint32_t first = pidx[fcand[i]], n = pidx[fcand[i + 1]] - first;
        symgpu_mpa_file_index& ix = index[i];
        ix.first_packet = first, ix.n_packets = n;
        if (uint64_t(first) + n > cap) ix.status |= SYMGPU_MPA_NOT_WRITTEN;
    }
}

__global__ void mpa_packet_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos,
                                  uint32_t n_cand, const uint32_t* __restrict__ dur, const uint32_t* __restrict__ pidx,
                                  const uint64_t* __restrict__ samples_before, const uint32_t* __restrict__ fcand, const MpaTrack* __restrict__ ftrack,
                                  const symgpu_mpa_file_index* __restrict__ index, symgpu_mpa_packet* packets, symgpu_mp3_job* jobs) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) {
        if (dur[c] == 0) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        if (index[i].status & SYMGPU_MPA_NOT_WRITTEN) continue;
        const FileDev f = files[i];
        const MpaTrack& t = ftrack[i];
        const uint64_t q = vpos[c] - f.vbase;
        const uint8_t* d = data + f.offset;
        const int64_t ts = int64_t(samples_before[c] - samples_before[fcand[i]]) - int64_t(t.delay);
        const MpaPacket p = mpa_frame_packet(detail::be32(d + q), q, ts, t);
        const uint32_t at = pidx[c];
        if (packets) packets[at] = mpa_packet_record(p, d + q);
        if (jobs) jobs[at] = symgpu_mp3_job{f.offset + q, p.size, p.trim_start, p.trim_end > 0xffffffffu ? 0xffffffffu : uint32_t(p.trim_end), 0};
    }
}

}  // namespace

extern "C" symgpu_status symgpu_mpa_index_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                              int seekable, symgpu_mpa_packet* packets, symgpu_mp3_job* jobs, size_t cap_packets,
                                              symgpu_mpa_file_index* index, symgpu_mpa_track* tracks) {
    if (!ctx || (n_bytes && !data) || (n_files && (!files || !index || !tracks))) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_MPA_MAX_FILES) return SYMGPU_ERR_LIMIT;
    std::vector<FileDev> dev;
    uint64_t total, longest;
    symgpu_status e = file_layout(files, n_files, n_bytes, dev, total, longest);
    if (e != SYMGPU_OK) return e;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const uint32_t nf = uint32_t(n_files), hunt_rounds = mpa_hunt_rounds(longest), chain_rounds = mpa_chain_rounds(longest);
    const uint64_t n_tiles = (total + kTile - 1) / kTile;
    Carver c;
    size_t at_files, at_tiles;
    uint64_t n_cand;
    if ((e = count_candidates<MpaRule>(ctx, data, dev, total, c, at_files, at_tiles, n_cand)) != SYMGPU_OK) return e;
    const size_t keep = c.at;
    if (n_cand >= kMpaEnd) return SYMGPU_ERR_LIMIT;
    const uint32_t nc = uint32_t(n_cand);
    const uint64_t n_ctiles = (n_cand + kCandTile - 1) / kCandTile;
    const size_t at_vpos = c.take(n_cand * 8), at_node = c.take(n_cand * 4), at_rank = c.take(n_cand * 4), at_dur = c.take(n_cand * 4);
    const size_t at_jump[2] = {c.take(n_cand * 4), c.take(n_cand * 4)}, at_hunt[2] = {c.take(n_cand * 4), c.take(n_cand * 4)};
    const size_t at_pidx = c.take((n_cand + 1) * 4), at_before = c.take((n_cand + 1) * 8), at_fcand = c.take((n_files + 1) * 4);
    const size_t at_ftrack = c.take(n_files * sizeof(MpaTrack)), at_ctiles = c.take((n_ctiles + 1) * sizeof(CandTile));
    if ((e = ensure_stage_keep(ctx, c.at, keep)) != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    auto u32 = [&](size_t at) { return reinterpret_cast<uint32_t*>(stage + at); };
    const FileDev* d_files = reinterpret_cast<const FileDev*>(stage + at_files);
    const uint64_t* d_tiles = reinterpret_cast<const uint64_t*>(stage + at_tiles);
    uint64_t* vpos = reinterpret_cast<uint64_t*>(stage + at_vpos);
    uint64_t* before = reinterpret_cast<uint64_t*>(stage + at_before);
    uint32_t *node = u32(at_node), *rank = u32(at_rank), *dur = u32(at_dur), *pidx = u32(at_pidx), *fcand = u32(at_fcand);
    uint32_t* jump[2] = {u32(at_jump[0]), u32(at_jump[1])};
    uint32_t* hunt[2] = {u32(at_hunt[0]), u32(at_hunt[1])};
    MpaTrack* ftrack = reinterpret_cast<MpaTrack*>(stage + at_ftrack);
    CandTile* ctiles = reinterpret_cast<CandTile*>(stage + at_ctiles);
    cudaStream_t st = ctx->stream;
    const unsigned cand_blocks = blocks_for(nc, 256), file_blocks = blocks_for(nf, 256), ctile_blocks = blocks_for(n_ctiles, 1);
    candidates_kernel<MpaRule><<<blocks_for(n_tiles, 1), kTileThreads, 0, st>>>(data, d_files, nf, total, n_tiles, d_tiles, vpos, node);
    CU(ctx, cudaGetLastError());
    mpa_successor_kernel<<<cand_blocks, 256, 0, st>>>(data, d_files, nf, vpos, nc, node, jump[0], hunt[0], rank);
    CU(ctx, cudaGetLastError());
    for (uint32_t k = 0; k < hunt_rounds; ++k) {
        mpa_hunt_kernel<<<cand_blocks, 256, 0, st>>>(hunt[k & 1], hunt[(k + 1) & 1], nc);
        CU(ctx, cudaGetLastError());
    }
    CU(ctx, cudaMemsetAsync(index, 0, n_files * sizeof(symgpu_mpa_file_index), st));
    mpa_track_kernel<<<file_blocks, 256, 0, st>>>(data, d_files, nf, vpos, nc, node, hunt[hunt_rounds & 1], seekable != 0, fcand, rank, ftrack, tracks,
                                                  index);
    CU(ctx, cudaGetLastError());
    for (uint32_t k = 0; k < chain_rounds; ++k) {
        chain_double_kernel<<<cand_blocks, 256, 0, st>>>(rank, jump[k & 1], jump[(k + 1) & 1], nc, k);
        CU(ctx, cudaGetLastError());
    }
    mpa_dur_kernel<<<ctile_blocks, kTileThreads, 0, st>>>(data, d_files, nf, vpos, nc, node, rank, ftrack, dur, n_ctiles, ctiles);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(ctiles, n_ctiles + 1, CandFirsts{});
    CU(ctx, cudaGetLastError());
    mpa_rank_kernel<<<ctile_blocks, kTileThreads, 0, st>>>(nc, dur, n_ctiles, ctiles, pidx, before);
    CU(ctx, cudaGetLastError());
    mpa_record_kernel<<<file_blocks, 256, 0, st>>>(nf, fcand, pidx, cap_packets, index);
    CU(ctx, cudaGetLastError());
    mpa_packet_kernel<<<cand_blocks, 256, 0, st>>>(data, d_files, nf, vpos, nc, dur, pidx, before, fcand, ftrack, index, packets, jobs);
    CU(ctx, cudaGetLastError());
    ctx->launches += 8 + hunt_rounds + chain_rounds;
    return SYMGPU_OK;
}
