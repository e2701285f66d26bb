// The FLAC-in-Ogg job build of symgpu_ogg_flac_heads_dev / symgpu_ogg_flac_jobs_dev (symphonia_b200/csrc/ogg_flac_jobs_kernel.cu)
// run on the CPU through the same functions of include/symgpu/packetizer.hpp the kernels call: per file the stream's end and
// its identification packet, per packet the audio decision and the slot, the exclusive scan over one table holding every file's
// packets, per file the totals, and per audio packet its bytes gathered and its job.  Input on stdin: one line
//   <n> (<data> <packets> <pieces>)*n    (each file's bytes and its symgpu_ogg_packet / symgpu_piece records)
// Output, per file: "F status n_stream block_min block_max sample_rate channels bps n_audio audio_bytes samples", then per job
// of the table "J group len slot offset" and the gathered bytes written to <data of file 0>.out.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

using namespace symgpu::packet;

namespace {

std::vector<uint8_t> slurp(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
template <class T>
std::vector<T> records(const std::string& path) {
    const std::vector<uint8_t> b = slurp(path);
    std::vector<T> out(b.size() / sizeof(T));
    if (!out.empty()) std::memcpy(out.data(), b.data(), out.size() * sizeof(T));
    return out;
}

struct File {
    std::vector<uint8_t> data;
    size_t first_packet = 0, first_piece = 0;
    uint32_t n_packets = 0;
};

struct Head {
    uint8_t status = 0;
    uint32_t n_stream = 0, n_audio = 0;
    uint64_t audio_bytes = 0, samples = 0;
    FlacStreamInfo info{};
};
struct Rank {
    uint64_t rank = 0, byte_at = 0, samples_at = 0;
    uint32_t slot = 0;
    bool audio = false;
};

}  // namespace

int main() {
    std::string line;
    if (!std::getline(std::cin, line)) return 1;
    std::istringstream in(line);
    size_t n = 0;
    in >> n;
    std::vector<File> files(n);
    std::vector<symgpu_ogg_packet> packets;
    std::vector<symgpu_piece> pieces;
    std::string first_path;
    for (size_t i = 0; i < n; ++i) {
        std::string d, p, q;
        in >> d >> p >> q;
        if (i == 0) first_path = d;
        files[i].data = slurp(d);
        const auto pk = records<symgpu_ogg_packet>(p);
        const auto pc = records<symgpu_piece>(q);
        files[i].first_packet = packets.size(), files[i].first_piece = pieces.size(), files[i].n_packets = uint32_t(pk.size());
        packets.insert(packets.end(), pk.begin(), pk.end());
        pieces.insert(pieces.end(), pc.begin(), pc.end());
    }
    // 1. one thread per file: the stream and the identification packet (ogg_flac_heads_kernel)
    std::vector<Head> heads(n);
    for (size_t i = 0; i < n; ++i) {
        const File& f = files[i];
        Head& h = heads[i];
        if (f.n_packets == 0) {
            h.status = SYMGPU_OGG_FLAC_NO_PACKETS;
            continue;
        }
        const symgpu_ogg_packet* pk = packets.data() + f.first_packet;
        const symgpu_piece* pc = pieces.data() + f.first_piece;
        h.n_stream = ogg_first_stream_len(pk, f.n_packets);
        uint8_t id[kOggFlacIdentLen];
        const uint32_t got = pk[0].len == kOggFlacIdentLen ? ogg_packet_head(f.data.data(), pc + pk[0].first_piece, pk[0].n_pieces, id, kOggFlacIdentLen) : 0;
        const Status s = got == kOggFlacIdentLen ? ogg_flac_ident(id, got, h.info) : Status::Unsupported;
        if (s != Status::Ok) h.status = s == Status::Unsupported ? SYMGPU_OGG_FLAC_NOT_FLAC : SYMGPU_OGG_FLAC_BAD_STREAMINFO;
    }
    // 2. one thread per packet: audio and slot (ogg_flac_audio_kernel)
    std::vector<Rank> ranks(packets.size());
    std::vector<uint32_t> owner(packets.size());
    for (size_t i = 0; i < n; ++i)
        for (uint32_t k = 0; k < files[i].n_packets; ++k) {
            const size_t p = files[i].first_packet + k;
            owner[p] = uint32_t(i);
            const symgpu_ogg_packet& pk = packets[p];
            const symgpu_piece* pc = pieces.data() + files[i].first_piece + pk.first_piece;
            uint8_t b0 = 0;
            if (heads[i].status == 0 && k > 0 && k < heads[i].n_stream && ogg_packet_head(files[i].data.data(), pc, pk.n_pieces, &b0, 1) == 1 &&
                ogg_flac_is_audio(uint32_t(pk.len), b0))
                ranks[p].audio = true, ranks[p].slot = ogg_flac_packet_block(files[i].data.data(), pc, pk.n_pieces);
        }
    // 3. the exclusive scan over the whole table (exclusive_scan_kernel)
    uint64_t c_rank = 0, c_bytes = 0, c_samples = 0;
    for (size_t p = 0; p < packets.size(); ++p) {
        Rank& r = ranks[p];
        r.rank = c_rank, r.byte_at = c_bytes, r.samples_at = c_samples;
        if (r.audio) c_rank += 1, c_bytes += packets[p].len, c_samples += r.slot;
    }
    // 4. one thread per file: totals (ogg_flac_totals_kernel)
    for (size_t i = 0; i < n; ++i) {
        Head& h = heads[i];
        if (h.status) continue;
        const size_t first = files[i].first_packet, last = first + files[i].n_packets - 1;
        const Rank &a = ranks[first], &z = ranks[last];
        h.n_audio = uint32_t(z.rank + z.audio - a.rank);
        h.audio_bytes = z.byte_at + (z.audio ? packets[last].len : 0) - a.byte_at;
        h.samples = z.samples_at + z.slot - a.samples_at;
    }
    // 5. one warp per audio packet: bytes and job (ogg_flac_job_kernel)
    std::vector<uint8_t> out(c_bytes);
    std::vector<symgpu_flac_job> jobs(c_rank);
    for (size_t p = 0; p < packets.size(); ++p) {
        const Rank& r = ranks[p];
        if (!r.audio) continue;
        const uint32_t i = owner[p];
        const symgpu_ogg_packet& pk = packets[p];
        const symgpu_piece* pc = pieces.data() + files[i].first_piece + pk.first_piece;
        uint64_t at = r.byte_at;
        for (uint32_t k = 0; k < pk.n_pieces; ++k)
            for (uint32_t b = 0; b < pc[k].len; ++b) out[at++] = files[i].data[pc[k].offset + b];
        jobs[r.rank] = symgpu_flac_job{r.byte_at, uint32_t(pk.len), i, r.slot, 0};
    }
    for (size_t i = 0; i < n; ++i) {
        const Head& h = heads[i];
        std::printf("F %u %u %u %u %u %u %u %u %llu %llu\n", h.status, h.n_stream, h.status ? 0 : h.info.block_min, h.status ? 0 : h.info.block_max,
                    h.status ? 0 : h.info.sample_rate, h.status ? 0 : h.info.channels, h.status ? 0 : h.info.bits_per_sample, h.n_audio,
                    (unsigned long long)h.audio_bytes, (unsigned long long)h.samples);
    }
    for (const symgpu_flac_job& j : jobs) std::printf("J %u %u %u %llu\n", j.group, j.len, j.slot, (unsigned long long)j.offset);
    std::ofstream(first_path + ".out", std::ios::binary).write(reinterpret_cast<const char*>(out.data()), std::streamsize(out.size()));
    return 0;
}
