// The sync-candidate scan the device frame indexes share (adts_index_kernel.cu, mpa_index_kernel.cu).  The files' bytes form one
// virtual byte space, in call order, cut into tiles of 4096 bytes, one block each: candidate_count_kernel counts each tile's
// candidates, exclusive_scan_kernel (block_scan.cuh) gives each tile's first and the total, which the host reads back once to size
// the per-candidate scratch, and candidates_kernel writes every candidate's virtual position and node word, in order.  A Rule has
// static host / device functions is_candidate(d, n, q) and node(d, n, q) over one file's bytes d[0 .. n).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/symgpu/packetizer.hpp"
#include "batch_call.h"
#include "block_scan.cuh"

namespace symgpu_detail {

struct FileDev {
    uint64_t offset, len;
    uint64_t vbase;  // the file's first virtual byte: the lengths of the files before it
};

constexpr uint32_t kTileThreads = 256, kBytesPerThread = 16, kTile = kTileThreads * kBytesPerThread;
constexpr unsigned kMaxBlocks = 65535 * 8;

inline unsigned blocks_for(uint64_t n, uint32_t per_block) {
    const uint64_t b = (n + per_block - 1) / per_block;
    return unsigned(b == 0 ? 1 : b < kMaxBlocks ? b : kMaxBlocks);
}

// The file that owns virtual byte v < the files' total: the last whose vbase <= v (an empty file owns no byte).
__device__ inline uint32_t file_of(const FileDev* files, uint32_t n_files, uint64_t v) {
    uint32_t lo = 0, hi = n_files;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (files[mid].vbase <= v) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The candidates among this thread's 16 virtual bytes of the tile, in order: on(v, file, q) for each; returns their number.
template <class Rule, class On>
__device__ inline uint32_t thread_candidates(const uint8_t* data, const FileDev* files, uint32_t n_files, uint64_t total, uint64_t tile, On&& on) {
    const uint64_t v0 = tile * kTile + uint64_t(threadIdx.x) * kBytesPerThread;
    if (v0 >= total) return 0;
    const uint64_t v1 = v0 + kBytesPerThread < total ? v0 + kBytesPerThread : total;
    uint32_t f = file_of(files, n_files, v0), count = 0;
    for (uint64_t v = v0; v < v1; ++v) {
        while (v >= files[f].vbase + files[f].len) ++f;
        const FileDev& fd = files[f];
        const uint64_t q = v - fd.vbase;
        if (Rule::is_candidate(data + fd.offset, size_t(fd.len), size_t(q))) on(v, f, q), ++count;
    }
    return count;
}

template <class Rule>
__global__ void __launch_bounds__(kTileThreads) candidate_count_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                                                       uint64_t total, uint64_t n_tiles, uint64_t* __restrict__ tile_count) {
    if (blockIdx.x == 0 && threadIdx.x == 0) tile_count[n_tiles] = 0;  // scanned into the total
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint64_t v[1] = {thread_candidates<Rule>(data, files, n_files, total, t, [](uint64_t, uint32_t, uint64_t) {})};
        uint64_t before[1], sum[1];
        block_exclusive_sums<1>(v, before, sum);
        if (threadIdx.x == 0) tile_count[t] = sum[0];
    }
}

struct TileFirsts {
    static constexpr int kN = 1;
    __device__ uint64_t get(const uint64_t& r, int) const { return r; }
    __device__ void put(uint64_t& r, int, uint64_t before) const { r = before; }
};

template <class Rule>
__global__ void __launch_bounds__(kTileThreads) candidates_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                                                  uint64_t total, uint64_t n_tiles, const uint64_t* __restrict__ tile_first,
                                                                  uint64_t* __restrict__ vpos, uint32_t* __restrict__ node) {
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint64_t v[1] = {thread_candidates<Rule>(data, files, n_files, total, t, [](uint64_t, uint32_t, uint64_t) {})};
        uint64_t before[1], sum[1];
        block_exclusive_sums<1>(v, before, sum);
        uint64_t at = tile_first[t] + before[0];
        thread_candidates<Rule>(data, files, n_files, total, t, [&](uint64_t pos, uint32_t f, uint64_t q) {
            vpos[at] = pos;
            node[at++] = Rule::node(data + files[f].offset, size_t(files[f].len), size_t(q));
        });
    }
}

// One round of chain ranking by pointer doubling (adts_double in packetizer.hpp) over every candidate.
static __global__ void chain_double_kernel(uint32_t* rank, const uint32_t* __restrict__ jump, uint32_t* __restrict__ next, uint32_t n_cand, uint32_t k) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_cand; c += gridDim.x * blockDim.x) symgpu::packet::adts_double(rank, jump, next, c, k);
}

// The files' virtual layout from the caller's ranges: SYMGPU_ERR_ARG for a range outside data[0 .. n_bytes), SYMGPU_ERR_LIMIT for
// a file of 2^32 bytes or more.  total: the files' lengths summed; longest: the longest.
inline symgpu_status file_layout(const symgpu_file_range* files, size_t n_files, size_t n_bytes, std::vector<FileDev>& dev, uint64_t& total,
                                 uint64_t& longest) {
    dev.resize(n_files);
    total = longest = 0;
    for (size_t i = 0; i < n_files; ++i) {
        const symgpu_file_range& r = files[i];
        if (r.offset > n_bytes || r.len > n_bytes - r.offset) return SYMGPU_ERR_ARG;
        if (r.len >> 32) return SYMGPU_ERR_LIMIT;
        dev[i] = FileDev{r.offset, r.len, total};
        total += r.len;
        longest = r.len > longest ? r.len : longest;
    }
    return SYMGPU_OK;
}

// The files' table and the tile counts at the start of the staging buffer (carved from `c`), the count and scan launches, and the
// one host wait, for the number of candidates.
template <class Rule>
symgpu_status count_candidates(symgpu_ctx* ctx, const uint8_t* data, const std::vector<FileDev>& dev, uint64_t total, Carver& c, size_t& at_files,
                               size_t& at_tiles, uint64_t& n_cand) {
    const uint64_t n_tiles = (total + kTile - 1) / kTile;
    at_files = c.take(dev.size() * sizeof(FileDev)), at_tiles = c.take((n_tiles + 1) * sizeof(uint64_t));
    symgpu_status e = ensure_stage(ctx, c.at);
    if (e != SYMGPU_OK) return e;
    cudaStream_t st = ctx->stream;
    FileDev* d_files = reinterpret_cast<FileDev*>(static_cast<char*>(ctx->d_stage) + at_files);
    uint64_t* d_tiles = reinterpret_cast<uint64_t*>(static_cast<char*>(ctx->d_stage) + at_tiles);
    // (a copy from pageable memory returns once the source is staged, so `dev` may go out of scope without a wait)
    CU(ctx, cudaMemcpyAsync(d_files, dev.data(), dev.size() * sizeof(FileDev), cudaMemcpyHostToDevice, st));
    candidate_count_kernel<Rule><<<blocks_for(n_tiles, 1), kTileThreads, 0, st>>>(data, d_files, uint32_t(dev.size()), total, n_tiles, d_tiles);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(d_tiles, n_tiles + 1, TileFirsts{});
    CU(ctx, cudaGetLastError());
    ctx->launches += 2;
    n_cand = 0;
    CU(ctx, cudaMemcpyAsync(&n_cand, d_tiles + n_tiles, sizeof n_cand, cudaMemcpyDeviceToHost, st));
    CU(ctx, cudaStreamSynchronize(st));
    return SYMGPU_OK;
}

}  // namespace symgpu_detail
