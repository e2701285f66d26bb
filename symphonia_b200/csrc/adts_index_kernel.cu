// symgpu_adts_index_dev: the ADTS frame index of many files already in device memory (DESIGN §5b, include/symgpu.h).  Every
// per-candidate step is a function of include/symgpu/packetizer.hpp that tests/cpp/adts_index_driver.cpp also runs on the CPU;
// the header rules are the code symgpu_adts_index runs on the host.  The files' bytes form one virtual byte space, cut into
// tiles of 4096 bytes, one block each:
//   1. candidate_count_kernel (candidate_tiles.cuh): the sync candidates of each tile;
//   2. exclusive_scan_kernel (block_scan.cuh): each tile's first candidate, and the total, which is read back (the one host wait)
//      to size the per-candidate scratch;
//   3. candidates_kernel: each candidate's virtual position and node word (adts_node), in order;
//   4. adts_successor_kernel: successors (adts_successor) and the chain heads (adts_initial_rank);
//   5. K x chain_double_kernel (candidate_tiles.cuh), K = adts_rounds(longest file): every chain node's rank by pointer doubling;
//   6. adts_record_kernel: each file's packet count and stop from its last node, its stream parameters from its first frame;
//   7. exclusive_scan_kernel: each file's first packet, and whether its packets fit the capacity;
//   8. adts_packet_kernel: the packets and jobs, one thread per chain Frame.
#include <cuda_runtime.h>

#include "../../include/symgpu/packetizer.hpp"
#include "candidate_tiles.cuh"

namespace {

using namespace symgpu::packet;
using namespace symgpu_detail;

static_assert(kAdtsStopOk == uint32_t(SYMGPU_OK) && kAdtsStopDecode == uint32_t(SYMGPU_ERR_DECODE) &&
                  kAdtsStopUnsupported == uint32_t(SYMGPU_ERR_UNSUPPORTED) && kAdtsStopLimit == uint32_t(SYMGPU_ERR_LIMIT),
              "a Stop's kind is the stop symgpu_adts_index reports");
static_assert(sizeof(symgpu_adts_file_index) == 24, "record sizes are ABI");

struct AdtsRule {
    __device__ static bool is_candidate(const uint8_t* d, size_t n, size_t q) { return adts_is_candidate(d, n, q); }
    __device__ static uint32_t node(const uint8_t* d, size_t n, size_t q) { return adts_node(d, n, q); }
};

__global__ void adts_successor_kernel(const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos, uint32_t n_cand,
                                      uint32_t* __restrict__ node, uint32_t* __restrict__ jump, uint32_t* __restrict__ rank) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) {
        const FileDev f = files[file_of(files, n_files, vpos[c])];
        const uint32_t nd = node[c], s = adts_successor(vpos, n_cand, c, nd, f.vbase + f.len);
        jump[c] = s;
        if (s == kAdtsEnd) node[c] = nd | kAdtsLast;
        rank[c] = adts_initial_rank(vpos, c, f.vbase);
    }
}

__global__ void adts_record_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos,
                                   uint32_t n_cand, const uint32_t* __restrict__ node, const uint32_t* __restrict__ rank, symgpu_adts_file_index* index) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) {
        const uint32_t r = rank[c], nd = node[c];
        if (r == kAdtsUnranked) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        symgpu_adts_file_index& ix = index[i];
        if (nd & kAdtsLast) {
            uint32_t n, stop;
            adts_file_end(nd, r, &n, &stop);
            ix.n_packets = n, ix.stop = uint8_t(stop);
        }
        if (r == 0 && (nd & 7) == kAdtsFrame) {
            const FileDev f = files[i];
            const AdtsPacket p = adts_frame_packet(data + f.offset, size_t(f.len), size_t(vpos[c] - f.vbase), 0);
            ix.sample_rate = p.sample_rate, ix.channels = p.channels, ix.profile = p.profile;
        }
    }
}

// Each file's first packet, and SYMGPU_ADTS_NOT_WRITTEN when its packets pass the capacity.
struct FileFirsts {
    static constexpr int kN = 1;
    uint64_t cap;
    __device__ uint64_t get(const symgpu_adts_file_index& r, int) const { return r.n_packets; }
    __device__ void put(symgpu_adts_file_index& r, int, uint64_t before) const {
        r.first_packet = before;
        r.status = before + r.n_packets > cap ? SYMGPU_ADTS_NOT_WRITTEN : 0;
    }
};

__global__ void adts_packet_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos,
                                   uint32_t n_cand, const uint32_t* __restrict__ node, const uint32_t* __restrict__ rank,
                                   const symgpu_adts_file_index* __restrict__ index, symgpu_adts_packet* packets, symgpu_piece* jobs) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) {
        const uint32_t r = rank[c];
        if (r == kAdtsUnranked || (node[c] & 7) != kAdtsFrame) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        const symgpu_adts_file_index& ix = index[i];
        if (ix.status & SYMGPU_ADTS_NOT_WRITTEN) continue;
        const FileDev f = files[i];
        const AdtsPacket p = adts_frame_packet(data + f.offset, size_t(f.len), size_t(vpos[c] - f.vbase), r);
        const uint64_t at = ix.first_packet + r;
        if (packets) {
            symgpu_adts_packet o{};
            o.offset = p.offset, o.size = p.size, o.sample_rate = p.sample_rate, o.pts = p.pts, o.channels = p.channels, o.profile = p.profile;
            packets[at] = o;
        }
        if (jobs) jobs[at] = symgpu_piece{f.offset + p.offset, p.size, 0};
    }
}

}  // namespace

using namespace symgpu_detail;

extern "C" symgpu_status symgpu_adts_index_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                               symgpu_adts_packet* packets, symgpu_piece* jobs, size_t cap_packets, symgpu_adts_file_index* index) {
    if (!ctx || (n_bytes && !data) || (n_files && (!files || !index))) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_ADTS_MAX_FILES) return SYMGPU_ERR_LIMIT;
    std::vector<FileDev> dev;
    uint64_t total, longest;
    symgpu_status e = file_layout(files, n_files, n_bytes, dev, total, longest);
    if (e != SYMGPU_OK) return e;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const uint32_t nf = uint32_t(n_files), rounds = adts_rounds(longest);
    const uint64_t n_tiles = (total + kTile - 1) / kTile;
    Carver c;
    size_t at_files, at_tiles;
    uint64_t n_cand;
    if ((e = count_candidates<AdtsRule>(ctx, data, dev, total, c, at_files, at_tiles, n_cand)) != SYMGPU_OK) return e;
    const size_t keep = c.at;
    cudaStream_t st = ctx->stream;
    if (n_cand >= kAdtsEnd) return SYMGPU_ERR_LIMIT;
    const size_t at_vpos = c.take(n_cand * sizeof(uint64_t)), at_node = c.take(n_cand * 4), at_rank = c.take(n_cand * 4);
    const size_t at_jump[2] = {c.take(n_cand * 4), c.take(n_cand * 4)};
    if ((e = ensure_stage_keep(ctx, c.at, keep)) != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    uint64_t* vpos = reinterpret_cast<uint64_t*>(stage + at_vpos);
    uint32_t *node = reinterpret_cast<uint32_t*>(stage + at_node), *rank = reinterpret_cast<uint32_t*>(stage + at_rank);
    uint32_t* jump[2] = {reinterpret_cast<uint32_t*>(stage + at_jump[0]), reinterpret_cast<uint32_t*>(stage + at_jump[1])};
    const uint32_t nc = uint32_t(n_cand);
    const unsigned cand_blocks = blocks_for(nc, 256);
    FileDev* d_files = reinterpret_cast<FileDev*>(stage + at_files);
    const uint64_t* d_tiles = reinterpret_cast<const uint64_t*>(stage + at_tiles);
    candidates_kernel<AdtsRule><<<blocks_for(n_tiles, 1), kTileThreads, 0, st>>>(data, d_files, nf, total, n_tiles, d_tiles, vpos, node);
    CU(ctx, cudaGetLastError());
    adts_successor_kernel<<<cand_blocks, 256, 0, st>>>(d_files, nf, vpos, nc, node, jump[0], rank);
    CU(ctx, cudaGetLastError());
    for (uint32_t k = 0; k < rounds; ++k) {
        chain_double_kernel<<<cand_blocks, 256, 0, st>>>(rank, jump[k & 1], jump[(k + 1) & 1], nc, k);
        CU(ctx, cudaGetLastError());
    }
    CU(ctx, cudaMemsetAsync(index, 0, n_files * sizeof(symgpu_adts_file_index), st));
    adts_record_kernel<<<cand_blocks, 256, 0, st>>>(data, d_files, nf, vpos, nc, node, rank, index);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(index, n_files, FileFirsts{cap_packets});
    CU(ctx, cudaGetLastError());
    adts_packet_kernel<<<cand_blocks, 256, 0, st>>>(data, d_files, nf, vpos, nc, node, rank, index, packets, jobs);
    CU(ctx, cudaGetLastError());
    ctx->launches += 5 + rounds;
    return SYMGPU_OK;
}
