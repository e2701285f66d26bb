// symgpu_flac_index_dev: the native FLAC frame index of many files already in device memory (DESIGN §5b, include/symgpu.h).  Every
// per-node step is a function of include/symgpu/packetizer.hpp that tests/cpp/flac_index_driver.cpp also runs on the CPU, and
// FlacIndexer (symgpu_flac_index) is a loop over the same rules.  The files' bytes form one virtual byte space, cut into tiles of
// 4096 bytes, one block each, 16 bytes per thread.  The nodes are the sync positions and one end node per file (flac_is_node):
//   1. flac_open_kernel, one thread per file: open()'s metadata walk (flac_open), the stream info record and the open status;
//   2. candidate_count_kernel + exclusive_scan_kernel (candidate_tiles.cuh): each tile's first node, and the total, which is read
//      back (the one host wait) to size the per-node scratch;
//   3. flac_key_tile_kernel: each tile's share of the CRC keys (the xor of flac_key_part over its threads' spans);
//   4. flac_key_scan_kernel: the exclusive xor-scan of the tiles' shares;
//   5. flac_nodes_kernel: each node's virtual position, node word and global key prefix, and each file's prefix at its first byte;
//   6. flac_head_kernel: each file's first node; each node's header (flac_head), its file-relative key and its end-search value;
//   7. 4 x (flac_digit_kernel, exclusive_scan_kernel, flac_scatter_kernel): a stable radix sort of the nodes by key, 4 bits a pass;
//   8. flac_sorted_kernel and T x flac_level_kernel, T = flac_tree_levels(longest file): the end-search tree over the sorted nodes;
//   9. flac_end_kernel: each plausible node's end (flac_end) and so whether it is good;
//  10. T x flac_level_kernel: the tree over the good nodes' sequence values, in node order;
//  11. flac_succ_kernel: each good node's successor (flac_successor) and each file's first frame, ranked 0 (flac_first_frame);
//  12. R x chain_double_kernel, R = flac_chain_rounds(longest file): every node of each chain ranked by pointer doubling;
//  13. flac_dur_kernel, exclusive_scan_kernel, flac_rank_kernel: each chain node's packet index and the samples before it;
//  14. flac_record_kernel: each file's first packet, packet count, samples and the capacity check;
//  15. flac_packet_kernel: the packets and jobs, one thread per chain node.
// 28 + 2 T + R launches in all.
#include <cuda_runtime.h>

#include <cstddef>

#include "../../include/symgpu/packetizer.hpp"
#include "candidate_tiles.cuh"
#include "flac_records.h"

namespace {

using namespace symgpu::packet;
using namespace symgpu_detail;

static_assert(sizeof(symgpu_flac_file_index) == 24, "record sizes are ABI");
static_assert(kFlacNone == kAdtsEnd && kFlacNone == kAdtsUnranked, "one 'none' for the chain steps");

__constant__ detail::Crc16Msb kCrc16Msb;  // the frame CRC-16's table (constant-initialised, as mpa_index_kernel.cu's)

struct FlacRule {
    __device__ static bool is_candidate(const uint8_t* d, size_t n, size_t q) { return flac_is_node(d, n, q); }
};

// What open() learned about a file.
struct FlacFile {
    FlacStreamInfo info;
    uint64_t first_frame;
    uint32_t opened;
};

constexpr uint32_t kPerThread = 16, kNodeTile = kTileThreads * kPerThread;

__global__ void flac_open_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, FlacFile* __restrict__ ffile,
                                 symgpu_flac_stream_info* __restrict__ infos, symgpu_flac_file_index* __restrict__ index) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_files; i += gridDim.x * blockDim.x) {
        FlacFile f{};
        size_t first = 0;
        const Status s = flac_open(data + files[i].offset, size_t(files[i].len), f.info, &first);
        f.first_frame = first, f.opened = s == Status::Ok;
        ffile[i] = f;
        infos[i] = f.opened ? flac_info_record(f.info, first) : symgpu_flac_stream_info{};
        symgpu_flac_file_index ix{};
        ix.open = uint8_t(s == Status::Ok ? SYMGPU_OK : s == Status::Unsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE);
        index[i] = ix;
    }
}

// The xor of flac_key_part over this thread's 16 virtual bytes of the tile, one part per file they touch.
__device__ inline uint32_t thread_key_share(const uint8_t* data, const FileDev* files, uint32_t n_files, uint64_t total, uint64_t tile) {
    const uint64_t v0 = tile * kTile + uint64_t(threadIdx.x) * kBytesPerThread;
    if (v0 >= total) return 0;
    const uint64_t v1 = v0 + kBytesPerThread < total ? v0 + kBytesPerThread : total;
    uint32_t f = file_of(files, n_files, v0), x = 0;
    for (uint64_t v = v0; v < v1;) {
        while (v >= files[f].vbase + files[f].len) ++f;
        const FileDev& fd = files[f];
        const uint64_t e = fd.vbase + fd.len < v1 ? fd.vbase + fd.len : v1;
        x ^= flac_key_part(kCrc16Msb.t, data + fd.offset, size_t(fd.len), size_t(v - fd.vbase), size_t(e - fd.vbase));
        v = e;
    }
    return x;
}

// An exclusive xor-scan over the block: before = the xor of the lower threads' values, returns the block's.
__device__ inline uint32_t block_exclusive_xor(uint32_t v, uint32_t& before) {
    __shared__ uint32_t warp_x[32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    uint32_t s = v;
    for (int o = 1; o < 32; o *= 2) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= uint32_t(o)) s ^= u;
    }
    if (lane == 31) warp_x[warp] = s;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < n_warps ? warp_x[lane] : 0;
        for (int o = 1; o < 32; o *= 2) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= uint32_t(o)) w ^= u;
        }
        warp_x[lane] = w;
    }
    __syncthreads();
    before = (warp ? warp_x[warp - 1] : 0) ^ s ^ v;
    const uint32_t all = warp_x[n_warps - 1];
    __syncthreads();
    return all;
}

__global__ void __launch_bounds__(kTileThreads) flac_key_tile_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files,
                                                                     uint32_t n_files, uint64_t total, uint64_t n_tiles, uint32_t* __restrict__ tile_x) {
    if (blockIdx.x == 0 && threadIdx.x == 0) tile_x[n_tiles] = 0;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint32_t before;
        const uint32_t all = block_exclusive_xor(thread_key_share(data, files, n_files, total, t), before);
        if (threadIdx.x == 0) tile_x[t] = all;
    }
}

__global__ void __launch_bounds__(1024) flac_key_scan_kernel(uint32_t* x, uint64_t n) {
    uint32_t carry = 0;
    for (uint64_t base = 0; base < n; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        uint32_t before;
        const uint32_t all = block_exclusive_xor(i < n ? x[i] : 0, before);
        if (i < n) x[i] = carry ^ before;
        carry ^= all;
    }
}

// Each node's virtual position, node word and key prefix (the xor-scan over every byte before it, from the start of the virtual
// space; an end node's includes its file's last byte), and fx0[f], the prefix at file f's first byte.
__global__ void __launch_bounds__(kTileThreads) flac_nodes_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                                                  uint64_t total, uint64_t n_tiles, const uint64_t* __restrict__ tile_first,
                                                                  const uint32_t* __restrict__ tile_x, uint64_t* __restrict__ vpos,
                                                                  uint32_t* __restrict__ node, uint32_t* __restrict__ key, uint32_t* __restrict__ fx0) {
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const uint64_t cnt[1] = {thread_candidates<FlacRule>(data, files, n_files, total, t, [](uint64_t, uint32_t, uint64_t) {})};
        uint64_t before[1], sum[1];
        block_exclusive_sums<1>(cnt, before, sum);
        uint32_t xb;
        block_exclusive_xor(thread_key_share(data, files, n_files, total, t), xb);
        uint64_t at = tile_first[t] + before[0];
        uint32_t pre = tile_x[t] ^ xb;  // the prefix at this thread's first byte
        const uint64_t v0 = t * kTile + uint64_t(threadIdx.x) * kBytesPerThread;
        if (v0 >= total) continue;
        const uint64_t v1 = v0 + kBytesPerThread < total ? v0 + kBytesPerThread : total;
        uint32_t f = file_of(files, n_files, v0);
        for (uint64_t v = v0; v < v1;) {  // one span per file touched
            while (v >= files[f].vbase + files[f].len) ++f;
            const FileDev& fd = files[f];
            const uint8_t* d = data + fd.offset;
            const size_t n = size_t(fd.len);
            const uint64_t e = fd.vbase + fd.len < v1 ? fd.vbase + fd.len : v1;
            uint16_t s = 0;  // CRC state over [v, here)
            for (uint64_t u = v; u < e; ++u) {
                const size_t q = size_t(u - fd.vbase);
                if (q == 0) fx0[f] = pre;
                if (flac_is_node(d, n, q)) {
                    const bool end = flac_node(n, q) & kFlacEndNode;
                    const uint16_t s_at = end ? crc16_ansi_update_with(kCrc16Msb.t, s, d + q, 1) : s;
                    vpos[at] = u, node[at] = flac_node(n, q);
                    key[at++] = pre ^ flac_key_inside(s_at, n, end ? n : q);
                }
                s = crc16_ansi_update_with(kCrc16Msb.t, s, d + q, 1);
            }
            pre ^= flac_key_inside(s, n, size_t(e - fd.vbase));
            v = e;
        }
    }
}

// fnode[i]: file i's first node (fnode[n_files] = n_nodes); per node its header, its file-relative key (the sort key, with the
// node as its value) and its end-search value.
__global__ void flac_head_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, const FlacFile* __restrict__ ffile,
                                 const uint64_t* __restrict__ vpos, const uint32_t* __restrict__ node, uint32_t n_nodes, const uint32_t* __restrict__ key,
                                 const uint32_t* __restrict__ fx0, uint32_t* __restrict__ fnode, FlacHead* __restrict__ head, uint32_t* __restrict__ skey,
                                 uint32_t* __restrict__ sid, uint64_t* __restrict__ ev) {
    const uint32_t n = n_nodes > n_files ? n_nodes : n_files;
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        if (c < n_files) {
            fnode[c] = detail::first_at_or_after(vpos, 0, n_nodes, files[c].vbase);
            if (c == 0) fnode[n_files] = n_nodes;
        }
        if (c >= n_nodes) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        const FileDev f = files[i];
        const FlacFile& ff = ffile[i];
        const FlacHead h = flac_head(data + f.offset, size_t(f.len), size_t(vpos[c] - f.vbase), node[c], ff.opened != 0, size_t(ff.first_frame), ff.info);
        head[c] = h;
        skey[c] = (key[c] ^ fx0[i]) & 0xffff, sid[c] = c;
        ev[c] = flac_end_value(h, node[c]);
    }
}

// ---- the radix sort: stable, 4 bits a pass, as counts per tile of 4096 nodes and an exclusive scan over the tiles ---------------
struct DigitTile {
    uint64_t c[16];
};
struct DigitFirsts {
    static constexpr int kN = 16;
    __device__ uint64_t get(const DigitTile& r, int k) const { return r.c[k]; }
    __device__ void put(DigitTile& r, int k, uint64_t before) const { r.c[k] = before; }
};

__device__ inline void thread_digits(const uint32_t* k_in, uint32_t n, uint64_t t, uint32_t shift, uint64_t (&cnt)[16]) {
    for (int d = 0; d < 16; ++d) cnt[d] = 0;
    const uint64_t c0 = t * kNodeTile + uint64_t(threadIdx.x) * kPerThread;
    for (uint64_t c = c0; c < c0 + kPerThread && c < n; ++c) {
        const uint32_t dg = (k_in[c] >> shift) & 15;
        for (int d = 0; d < 16; ++d) cnt[d] += dg == uint32_t(d);
    }
}

__global__ void __launch_bounds__(kTileThreads) flac_digit_kernel(const uint32_t* __restrict__ k_in, uint32_t n, uint32_t shift, uint64_t n_tiles,
                                                                  DigitTile* __restrict__ tiles) {
    if (blockIdx.x == 0 && threadIdx.x == 0) tiles[n_tiles] = DigitTile{};
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t cnt[16], before[16], sum[16];
        thread_digits(k_in, n, t, shift, cnt);
        block_exclusive_sums<16>(cnt, before, sum);
        if (threadIdx.x < 16) tiles[t].c[threadIdx.x] = sum[threadIdx.x];
    }
}

__global__ void __launch_bounds__(kTileThreads) flac_scatter_kernel(const uint32_t* __restrict__ k_in, const uint32_t* __restrict__ i_in, uint32_t n,
                                                                    uint32_t shift, uint64_t n_tiles, const DigitTile* __restrict__ tiles,
                                                                    uint32_t* __restrict__ k_out, uint32_t* __restrict__ i_out) {
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t cnt[16], before[16], sum[16], at[16];
        thread_digits(k_in, n, t, shift, cnt);
        block_exclusive_sums<16>(cnt, before, sum);
        uint64_t base = 0;  // the nodes of smaller digits, over all tiles (the scanned record past the end holds the totals)
        for (int d = 0; d < 16; ++d) at[d] = base + tiles[t].c[d] + before[d], base += tiles[n_tiles].c[d];
        const uint64_t c0 = t * kNodeTile + uint64_t(threadIdx.x) * kPerThread;
        for (uint64_t c = c0; c < c0 + kPerThread && c < n; ++c) {
            const uint32_t dg = (k_in[c] >> shift) & 15;
            uint64_t p = 0;
            for (int d = 0; d < 16; ++d)
                if (dg == uint32_t(d)) p = at[d]++;
            k_out[p] = k_in[c], i_out[p] = i_in[c];
        }
    }
}

__global__ void flac_sorted_kernel(const uint32_t* __restrict__ sid, const uint64_t* __restrict__ ev, uint32_t n, uint64_t* __restrict__ sv) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) sv[i] = ev[sid[i]];
}

__global__ void flac_level_kernel(const uint64_t* __restrict__ below, uint64_t n_below, uint64_t* __restrict__ out, uint64_t n_out) {
    for (uint64_t j = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; j < n_out; j += uint64_t(gridDim.x) * blockDim.x) out[j] = flac_tree_max(below, n_below, j);
}

__global__ void flac_end_kernel(const FileDev* __restrict__ files, uint32_t n_files, const uint64_t* __restrict__ vpos, const uint32_t* __restrict__ node,
                                uint32_t n_nodes, const uint32_t* __restrict__ fnode, const FlacHead* __restrict__ head, const uint32_t* __restrict__ key,
                                const uint32_t* __restrict__ fx0, const uint32_t* __restrict__ skey, const uint32_t* __restrict__ sid, FlacTree tree,
                                uint32_t* __restrict__ ends, uint64_t* __restrict__ gv, uint32_t* __restrict__ rank) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_nodes; c += gridDim.x * blockDim.x) {
        const FlacHead h = head[c];
        uint32_t e = kFlacNone;
        if (h.plausible) {
            const uint32_t i = file_of(files, n_files, vpos[c]);
            e = flac_end(vpos, node, c, fnode[i + 1], files[i].vbase, h, (key[c] ^ fx0[i]) & 0xffff, skey, sid, tree);
        }
        ends[c] = e;
        gv[c] = e == kFlacNone ? 0 : flac_value(h.seq);
        rank[c] = kAdtsUnranked;
    }
}

__global__ void flac_succ_kernel(const FileDev* __restrict__ files, uint32_t n_files, const FlacFile* __restrict__ ffile, const uint64_t* __restrict__ vpos,
                                 const uint32_t* __restrict__ node, uint32_t n_nodes, const uint32_t* __restrict__ fnode,
                                 const FlacHead* __restrict__ head, const uint32_t* __restrict__ ends, FlacTree good, uint32_t* __restrict__ jump,
                                 uint32_t* __restrict__ rank) {
    const uint32_t n = n_nodes > n_files ? n_nodes : n_files;
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        if (c < n_files && ffile[c].opened) {
            const uint32_t a = flac_first_frame(vpos, node, fnode[c], fnode[c + 1], files[c].vbase, size_t(ffile[c].first_frame), good);
            if (a != kFlacNone) rank[a] = 0;
        }
        if (c >= n_nodes) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        jump[c] = flac_successor(node, ends[c], fnode[i + 1], head[c].seq, good);
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

// dur[c]: the samples of chain node c's packet, 0 off the chain (a block is at least 1 sample); summed per tile of 4096 nodes.
__global__ void __launch_bounds__(kTileThreads) flac_dur_kernel(uint32_t n_nodes, const FlacHead* __restrict__ head, const uint32_t* __restrict__ rank,
                                                                uint32_t* __restrict__ dur, uint64_t n_tiles, CandTile* __restrict__ tiles) {
    if (blockIdx.x == 0 && threadIdx.x == 0) tiles[n_tiles] = CandTile{0, 0};
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t v[2] = {0, 0}, before[2], sum[2];
        const uint64_t c0 = t * kNodeTile + uint64_t(threadIdx.x) * kPerThread;
        for (uint64_t c = c0; c < c0 + kPerThread && c < n_nodes; ++c) {
            const uint32_t d = rank[c] == kAdtsUnranked ? 0 : head[c].block;
            dur[c] = d;
            v[0] += d != 0, v[1] += d;
        }
        block_exclusive_sums<2>(v, before, sum);
        if (threadIdx.x == 0) tiles[t] = CandTile{sum[0], sum[1]};
    }
}

__global__ void __launch_bounds__(kTileThreads) flac_rank_kernel(uint32_t n_nodes, const uint32_t* __restrict__ dur, uint64_t n_tiles,
                                                                 const CandTile* __restrict__ tiles, uint32_t* __restrict__ pidx,
                                                                 uint64_t* __restrict__ samples_before) {
    if (blockIdx.x == 0 && threadIdx.x == 0) pidx[n_nodes] = uint32_t(tiles[n_tiles].packets), samples_before[n_nodes] = tiles[n_tiles].samples;
    for (uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        uint64_t v[2] = {0, 0}, before[2], sum[2];
        const uint64_t c0 = t * kNodeTile + uint64_t(threadIdx.x) * kPerThread;
        for (uint64_t c = c0; c < c0 + kPerThread && c < n_nodes; ++c) v[0] += dur[c] != 0, v[1] += dur[c];
        block_exclusive_sums<2>(v, before, sum);
        uint64_t p = tiles[t].packets + before[0], s = tiles[t].samples + before[1];
        for (uint64_t c = c0; c < c0 + kPerThread && c < n_nodes; ++c) {
            pidx[c] = uint32_t(p), samples_before[c] = s;
            p += dur[c] != 0, s += dur[c];
        }
    }
}

__global__ void flac_record_kernel(uint32_t n_files, const uint32_t* __restrict__ fnode, const uint32_t* __restrict__ pidx,
                                   const uint64_t* __restrict__ samples_before, uint64_t cap, symgpu_flac_file_index* __restrict__ index) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_files; i += gridDim.x * blockDim.x) {
        const uint32_t first = pidx[fnode[i]], n = pidx[fnode[i + 1]] - first;
        symgpu_flac_file_index& ix = index[i];
        ix.first_packet = first, ix.n_packets = n, ix.samples = samples_before[fnode[i + 1]] - samples_before[fnode[i]];
        ix.status = uint64_t(first) + n > cap ? SYMGPU_FLAC_NOT_WRITTEN : 0;
    }
}

__global__ void flac_packet_kernel(const FileDev* __restrict__ files, uint32_t n_files, const FlacFile* __restrict__ ffile, const uint64_t* __restrict__ vpos,
                                   const uint32_t* __restrict__ node, uint32_t n_nodes, const FlacHead* __restrict__ head, const uint32_t* __restrict__ ends,
                                   const uint32_t* __restrict__ dur, const uint32_t* __restrict__ pidx, const symgpu_flac_file_index* __restrict__ index,
                                   symgpu_flac_packet* packets, symgpu_flac_job* jobs) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_nodes; c += gridDim.x * blockDim.x) {
        if (dur[c] == 0) continue;
        const uint32_t i = file_of(files, n_files, vpos[c]);
        if (index[i].status & SYMGPU_FLAC_NOT_WRITTEN) continue;
        const FileDev f = files[i];
        const FlacPacket p = flac_chain_packet(vpos[c] - f.vbase, flac_npos(vpos, node, ends[c], f.vbase), head[c], ffile[i].info);
        const uint32_t at = pidx[c];
        if (packets) packets[at] = flac_packet_record(p);
        if (jobs) jobs[at] = symgpu_flac_job{f.offset + p.offset, p.size, i, p.dur, 0};
    }
}

FlacTree tree_of(uint64_t* level0, uint64_t* levels, uint32_t n, uint32_t top) {
    FlacTree t{};
    t.n = n, t.top = top, t.level[0] = level0;
    uint64_t at = 0, len = n;
    for (uint32_t k = 1; k <= top; ++k) {
        len = (len + 1) / 2;
        t.level[k] = levels + at;
        at += len;
    }
    return t;
}

// The words the levels above level 0 of a tree over n values take.
uint64_t tree_words(uint64_t n, uint32_t top) {
    uint64_t words = 0, len = n;
    for (uint32_t k = 1; k <= top; ++k) len = (len + 1) / 2, words += len;
    return words;
}

}  // namespace

extern "C" symgpu_status symgpu_flac_index_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                               symgpu_flac_packet* packets, symgpu_flac_job* jobs, size_t cap_packets, symgpu_flac_file_index* index,
                                               symgpu_flac_stream_info* infos) {
    if (!ctx || (n_bytes && !data) || (n_files && (!files || !index || !infos))) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_FLAC_MAX_FILES) return SYMGPU_ERR_LIMIT;
    std::vector<FileDev> dev;
    uint64_t total, longest;
    symgpu_status e = file_layout(files, n_files, n_bytes, dev, total, longest);
    if (e != SYMGPU_OK) return e;
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    const uint32_t nf = uint32_t(n_files), top = flac_tree_levels(longest), rounds = flac_chain_rounds(longest);
    const uint64_t n_tiles = (total + kTile - 1) / kTile;
    Carver c;
    const size_t at_ffile = c.take(n_files * sizeof(FlacFile));
    size_t at_files, at_tiles;
    uint64_t n_nodes;
    cudaStream_t st = ctx->stream;
    const unsigned file_blocks = blocks_for(nf, 256);
    if ((e = count_candidates<FlacRule>(ctx, data, dev, total, c, at_files, at_tiles, n_nodes)) != SYMGPU_OK) return e;
    const size_t keep = c.at;
    if (n_nodes >= kFlacNone) return SYMGPU_ERR_LIMIT;
    const uint32_t nn = uint32_t(n_nodes);
    const uint64_t n_ntiles = (n_nodes + kNodeTile - 1) / kNodeTile, lw = tree_words(n_nodes, top);
    const size_t at_tx = c.take((n_tiles + 1) * 4), at_vpos = c.take(n_nodes * 8), at_node = c.take(n_nodes * 4), at_key = c.take(n_nodes * 4);
    const size_t at_fx0 = c.take(n_files * 4), at_fnode = c.take((n_files + 1) * 4), at_head = c.take(n_nodes * sizeof(FlacHead));
    const size_t at_sk[2] = {c.take(n_nodes * 4), c.take(n_nodes * 4)}, at_si[2] = {c.take(n_nodes * 4), c.take(n_nodes * 4)};
    const size_t at_ev = c.take(n_nodes * 8), at_sv = c.take(n_nodes * 8), at_lv = c.take(lw * 8), at_gv = c.take(n_nodes * 8), at_gl = c.take(lw * 8);
    const size_t at_ends = c.take(n_nodes * 4), at_rank = c.take(n_nodes * 4), at_jump[2] = {c.take(n_nodes * 4), c.take(n_nodes * 4)};
    const size_t at_dur = c.take(n_nodes * 4), at_pidx = c.take((n_nodes + 1) * 4), at_before = c.take((n_nodes + 1) * 8);
    const size_t at_dt = c.take((n_ntiles + 1) * sizeof(DigitTile)), at_ct = c.take((n_ntiles + 1) * sizeof(CandTile));
    if ((e = ensure_stage_keep(ctx, c.at, keep)) != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    auto u32 = [&](size_t at) { return reinterpret_cast<uint32_t*>(stage + at); };
    auto u64 = [&](size_t at) { return reinterpret_cast<uint64_t*>(stage + at); };
    const FileDev* d_files = reinterpret_cast<const FileDev*>(stage + at_files);
    const uint64_t* d_tiles = reinterpret_cast<const uint64_t*>(stage + at_tiles);
    FlacFile* ffile = reinterpret_cast<FlacFile*>(stage + at_ffile);
    FlacHead* head = reinterpret_cast<FlacHead*>(stage + at_head);
    DigitTile* dtiles = reinterpret_cast<DigitTile*>(stage + at_dt);
    CandTile* ctiles = reinterpret_cast<CandTile*>(stage + at_ct);
    uint64_t *vpos = u64(at_vpos), *ev = u64(at_ev), *sv = u64(at_sv), *gv = u64(at_gv), *before = u64(at_before);
    uint32_t *tile_x = u32(at_tx), *node = u32(at_node), *key = u32(at_key), *fx0 = u32(at_fx0), *fnode = u32(at_fnode);
    uint32_t *ends = u32(at_ends), *rank = u32(at_rank), *dur = u32(at_dur), *pidx = u32(at_pidx);
    uint32_t* sk[2] = {u32(at_sk[0]), u32(at_sk[1])};
    uint32_t* si[2] = {u32(at_si[0]), u32(at_si[1])};
    uint32_t* jump[2] = {u32(at_jump[0]), u32(at_jump[1])};
    const unsigned node_blocks = blocks_for(nn, 256), both_blocks = blocks_for(nn > nf ? nn : nf, 256), ntile_blocks = blocks_for(n_ntiles, 1);
    const unsigned tile_blocks = blocks_for(n_tiles, 1);
    flac_open_kernel<<<file_blocks, 256, 0, st>>>(data, d_files, nf, ffile, infos, index);
    CU(ctx, cudaGetLastError());
    flac_key_tile_kernel<<<tile_blocks, kTileThreads, 0, st>>>(data, d_files, nf, total, n_tiles, tile_x);
    CU(ctx, cudaGetLastError());
    flac_key_scan_kernel<<<1, 1024, 0, st>>>(tile_x, n_tiles + 1);
    CU(ctx, cudaGetLastError());
    flac_nodes_kernel<<<tile_blocks, kTileThreads, 0, st>>>(data, d_files, nf, total, n_tiles, d_tiles, tile_x, vpos, node, key, fx0);
    CU(ctx, cudaGetLastError());
    flac_head_kernel<<<both_blocks, 256, 0, st>>>(data, d_files, nf, ffile, vpos, node, nn, key, fx0, fnode, head, sk[0], si[0], ev);
    CU(ctx, cudaGetLastError());
    for (uint32_t p = 0; p < 4; ++p) {  // keys of 16 bits; after 4 passes the sorted nodes are back in sk[0] / si[0]
        flac_digit_kernel<<<ntile_blocks, kTileThreads, 0, st>>>(sk[p & 1], nn, 4 * p, n_ntiles, dtiles);
        CU(ctx, cudaGetLastError());
        exclusive_scan_kernel<<<1, 1024, 0, st>>>(dtiles, n_ntiles + 1, DigitFirsts{});
        CU(ctx, cudaGetLastError());
        flac_scatter_kernel<<<ntile_blocks, kTileThreads, 0, st>>>(sk[p & 1], si[p & 1], nn, 4 * p, n_ntiles, dtiles, sk[(p + 1) & 1], si[(p + 1) & 1]);
        CU(ctx, cudaGetLastError());
    }
    flac_sorted_kernel<<<node_blocks, 256, 0, st>>>(si[0], ev, nn, sv);
    CU(ctx, cudaGetLastError());
    const FlacTree ends_tree = tree_of(sv, u64(at_lv), nn, top), good_tree = tree_of(gv, u64(at_gl), nn, top);
    auto build = [&](const FlacTree& t) {
        uint64_t len = n_nodes;
        for (uint32_t k = 1; k <= top; ++k) {
            const uint64_t out = (len + 1) / 2;
            flac_level_kernel<<<blocks_for(out, 256), 256, 0, st>>>(t.level[k - 1], len, const_cast<uint64_t*>(t.level[k]), out);
            len = out;
        }
        return cudaGetLastError();
    };
    CU(ctx, build(ends_tree));
    flac_end_kernel<<<node_blocks, 256, 0, st>>>(d_files, nf, vpos, node, nn, fnode, head, key, fx0, sk[0], si[0], ends_tree, ends, gv, rank);
    CU(ctx, cudaGetLastError());
    CU(ctx, build(good_tree));
    flac_succ_kernel<<<both_blocks, 256, 0, st>>>(d_files, nf, ffile, vpos, node, nn, fnode, head, ends, good_tree, jump[0], rank);
    CU(ctx, cudaGetLastError());
    for (uint32_t k = 0; k < rounds; ++k) {
        chain_double_kernel<<<node_blocks, 256, 0, st>>>(rank, jump[k & 1], jump[(k + 1) & 1], nn, k);
        CU(ctx, cudaGetLastError());
    }
    flac_dur_kernel<<<ntile_blocks, kTileThreads, 0, st>>>(nn, head, rank, dur, n_ntiles, ctiles);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(ctiles, n_ntiles + 1, CandFirsts{});
    CU(ctx, cudaGetLastError());
    flac_rank_kernel<<<ntile_blocks, kTileThreads, 0, st>>>(nn, dur, n_ntiles, ctiles, pidx, before);
    CU(ctx, cudaGetLastError());
    flac_record_kernel<<<file_blocks, 256, 0, st>>>(nf, fnode, pidx, before, cap_packets, index);
    CU(ctx, cudaGetLastError());
    flac_packet_kernel<<<node_blocks, 256, 0, st>>>(d_files, nf, ffile, vpos, node, nn, head, ends, dur, pidx, index, packets, jobs);
    CU(ctx, cudaGetLastError());
    ctx->launches += 26 + 2 * top + rounds;  // (+ the count and its scan, counted by count_candidates)
    return SYMGPU_OK;
}
