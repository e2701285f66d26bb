// symgpu_ogg_index_dev: the Ogg page index of many files already in device memory (DESIGN §5b, include/symgpu.h).  Every step
// is a function of include/symgpu/packetizer.hpp that tests/cpp/ogg_index_driver.cpp also runs on the CPU; the page check and
// the logical-stream step are the code symgpu_ogg_index runs on the host.  Five launches:
//   1. ogg_successor_kernel, one thread per 4 file bytes: ogg_successor_word;
//   2. ogg_chain_kernel, one thread per file: the chain of pages that verify (ogg_next_page), then those pages ordered by serial
//      (ogg_sort_by_serial);
//   3. ogg_walk_kernel<false>, one thread per file: the logical streams (ogg_walk_streams), packets and pieces counted;
//   4. exclusive_scan_kernel (block_scan.cuh), one block: each file's first packet and first piece;
//   5. ogg_walk_kernel<true>: the same walk, writing the tables of every file that fits the capacities.
// Each per-file step is linear in the file's words and pages.
#include <cuda_runtime.h>

#include "../../include/symgpu/packetizer.hpp"
#include "batch_call.h"
#include "block_scan.cuh"

namespace {

using namespace symgpu::packet;
using symgpu_detail::Carver;

struct FileDev {
    uint64_t offset, len;
    uint64_t word_base;  // the file's first word in each per-word array: 4-byte groups of the files before it
};

struct Chain {
    uint32_t* succ;      // successor words; after the chain is built, the sort's spare keys
    uint32_t* serial;    // the chain's pages, sorted by serial
    uint32_t* offset;
    uint32_t* spare;     // the sort's spare offsets
    uint32_t* n_pages;   // per file
};

__global__ void __launch_bounds__(256) ogg_successor_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files,
                                                            uint64_t n_words, uint32_t* __restrict__ succ) {
    __shared__ uint32_t crc[8][256];
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i << 24;
        for (int k = 0; k < 8; ++k) c = (c & 0x80000000u) ? (c << 1) ^ 0x04c11db7u : c << 1;
        crc[0][i] = c;
    }
    __syncthreads();
    for (int k = 1; k < 8; ++k) {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) crc[k][i] = (crc[k - 1][i] << 8) ^ crc[0][crc[k - 1][i] >> 24];
        __syncthreads();
    }
    for (uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; w < n_words; w += uint64_t(gridDim.x) * blockDim.x) {
        uint32_t lo = 0, hi = n_files;  // the last file whose word_base <= w (empty files own no word)
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) / 2;
            if (files[mid].word_base <= w) lo = mid;
            else hi = mid;
        }
        const FileDev f = files[lo];
        succ[w] = ogg_successor_word(data + f.offset, size_t(f.len), size_t(w - f.word_base), crc);
    }
}

__global__ void ogg_chain_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, Chain c) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files) return;
    const FileDev f = files[i];
    const uint8_t* d = data + f.offset;
    uint32_t *succ = c.succ + f.word_base, *serial = c.serial + f.word_base, *offset = c.offset + f.word_base;
    uint32_t n = 0;  // a page starts in a word of its own, so a file has at most as many pages as words
    for (uint64_t pos = 0, q; ogg_next_page(succ, f.len, &pos, &q); ++n) serial[n] = detail::le32(d + q + 14), offset[n] = uint32_t(q);
    ogg_sort_by_serial(serial, offset, succ, c.spare + f.word_base, n);
    c.n_pages[i] = n;
}

struct WalkSink {
    bool write;
    symgpu_ogg_packet* packets;  // the file's (write only)
    symgpu_piece* pieces;
    uint64_t n_pieces_file;      // the file's total: a trailing open packet's pieces past it are not stored
    uint64_t piece_base = 0;     // pieces of the file's earlier streams
    uint64_t n_packets = 0, bytes = 0;
    uint32_t max_len = 0, used = 0, serial = 0;
    __device__ void begin_stream(uint32_t s) { serial = s, used = 0; }
    __device__ void end_stream() { piece_base += used; }
    __device__ void piece(uint32_t i, uint64_t offset, uint32_t len) {
        if (write && piece_base + i < n_pieces_file) pieces[piece_base + i] = symgpu_piece{offset, len, 0};
    }
    __device__ void packet(uint32_t first, uint32_t count, uint64_t len, const OggPageHead& pg) {
        if (write) {
            symgpu_ogg_packet& o = packets[n_packets];
            o.serial = serial, o.page_sequence = pg.sequence, o.page_absgp = pg.absgp, o.len = len;
            o.first_piece = uint32_t(piece_base + first), o.n_pieces = count, o.last_on_page = 0;
            for (int k = 0; k < 7; ++k) o.reserved[k] = 0;
        }
        ++n_packets, bytes += len;
        max_len = len > max_len ? uint32_t(len) : max_len;
        used = first + count;
    }
    __device__ void last_on_page() {
        if (write) packets[n_packets - 1].last_on_page = 1;
    }
};

template <bool kWrite>
__global__ void ogg_walk_kernel(const uint8_t* __restrict__ data, const FileDev* __restrict__ files, uint32_t n_files, Chain c,
                                symgpu_ogg_packet* packets, uint64_t cap_packets, symgpu_piece* pieces, uint64_t cap_pieces, symgpu_ogg_file_index* index) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_files) return;
    const FileDev f = files[i];
    symgpu_ogg_file_index& ix = index[i];
    WalkSink sink{kWrite, nullptr, nullptr, 0};
    if (kWrite) {
        if (ix.first_packet + ix.n_packets > cap_packets || ix.first_piece + ix.n_pieces > cap_pieces) {
            ix.status |= SYMGPU_OGG_NOT_WRITTEN;
            return;
        }
        sink.packets = packets + ix.first_packet, sink.pieces = pieces + ix.first_piece, sink.n_pieces_file = ix.n_pieces;
    }
    const bool cap_hit = ogg_walk_streams(data + f.offset, c.serial + f.word_base, c.offset + f.word_base, c.n_pages[i], sink);
    if (!kWrite) {
        ix.n_packets = uint32_t(sink.n_packets), ix.n_pieces = uint32_t(sink.piece_base), ix.packet_bytes = sink.bytes;
        ix.max_packet_len = sink.max_len, ix.status = cap_hit ? SYMGPU_OGG_CAP_HIT : 0;
        ix.reserved[0] = ix.reserved[1] = ix.reserved[2] = 0;
    }
}

// Each file's first packet and first piece: exclusive sums of n_packets and n_pieces (exclusive_scan_kernel).
struct FileFirsts {
    static constexpr int kN = 2;
    __device__ uint64_t get(const symgpu_ogg_file_index& r, int k) const { return k ? r.n_pieces : r.n_packets; }
    __device__ void put(symgpu_ogg_file_index& r, int k, uint64_t before) const { (k ? r.first_piece : r.first_packet) = before; }
};

}  // namespace

using namespace symgpu_detail;

extern "C" symgpu_status symgpu_ogg_index_dev(symgpu_ctx* ctx, const uint8_t* data, size_t n_bytes, const symgpu_file_range* files, size_t n_files,
                                              symgpu_ogg_packet* packets, size_t cap_packets, symgpu_piece* pieces, size_t cap_pieces,
                                              symgpu_ogg_file_index* index) {
    if (!ctx || (n_bytes && !data) || (n_files && (!files || !index)) || (cap_packets && !packets) || (cap_pieces && !pieces)) return SYMGPU_ERR_ARG;
    if (n_files > SYMGPU_OGG_MAX_FILES) return SYMGPU_ERR_LIMIT;
    std::vector<FileDev> dev(n_files);
    uint64_t words = 0;
    for (size_t i = 0; i < n_files; ++i) {
        const symgpu_file_range& r = files[i];
        if (r.offset > n_bytes || r.len > n_bytes - r.offset) return SYMGPU_ERR_ARG;
        if (r.len >> 32) return SYMGPU_ERR_LIMIT;
        dev[i] = FileDev{r.offset, r.len, words};
        words += (r.len + 3) / 4;
    }
    if (n_files == 0) return SYMGPU_OK;
    DeviceGuard guard(ctx->device);
    Carver c;
    const size_t at_files = c.take(n_files * sizeof(FileDev)), at_n = c.take(n_files * sizeof(uint32_t));
    size_t at_words[4];
    for (size_t& a : at_words) a = c.take(words * sizeof(uint32_t));
    symgpu_status e = ensure_stage(ctx, c.at);
    if (e != SYMGPU_OK) return e;
    char* stage = static_cast<char*>(ctx->d_stage);
    FileDev* d_files = reinterpret_cast<FileDev*>(stage + at_files);
    auto words_at = [&](int k) { return reinterpret_cast<uint32_t*>(stage + at_words[k]); };
    const Chain chain{words_at(0), words_at(1), words_at(2), words_at(3), reinterpret_cast<uint32_t*>(stage + at_n)};
    cudaStream_t st = ctx->stream;
    // (a copy from pageable memory returns once the source is staged, so `dev` may go out of scope without a wait)
    CU(ctx, cudaMemcpyAsync(d_files, dev.data(), n_files * sizeof(FileDev), cudaMemcpyHostToDevice, st));
    const uint32_t nf = uint32_t(n_files), file_blocks = (nf + 127) / 128;
    if (words) {
        const uint64_t blocks = (words + 255) / 256;
        ogg_successor_kernel<<<unsigned(blocks < 65535 * 8 ? blocks : 65535 * 8), 256, 0, st>>>(data, d_files, nf, words, chain.succ);
        CU(ctx, cudaGetLastError());
        ++ctx->launches;
    }
    ogg_chain_kernel<<<file_blocks, 128, 0, st>>>(data, d_files, nf, chain);
    CU(ctx, cudaGetLastError());
    ogg_walk_kernel<false><<<file_blocks, 128, 0, st>>>(data, d_files, nf, chain, packets, cap_packets, pieces, cap_pieces, index);
    CU(ctx, cudaGetLastError());
    exclusive_scan_kernel<<<1, 1024, 0, st>>>(index, nf, FileFirsts{});
    CU(ctx, cudaGetLastError());
    ogg_walk_kernel<true><<<file_blocks, 128, 0, st>>>(data, d_files, nf, chain, packets, cap_packets, pieces, cap_pieces, index);
    CU(ctx, cudaGetLastError());
    ctx->launches += 4;
    return SYMGPU_OK;
}
