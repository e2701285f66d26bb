// The schedule of symgpu_ogg_index_dev (symphonia_b200/csrc/ogg_index_kernel.cu) run on the CPU through the same functions of
// include/symgpu/packetizer.hpp the kernels call: a successor word for every 4-byte group, the chain from byte 0, its pages
// sorted by serial, the logical streams walked.  Also the shared page end trims and
// Vorbis packet timer.  Input on stdin, one request per line:
//   index <path>                      -> "P serial seq absgp len first_piece n_pieces last" per packet, "Q offset len" per
//                                        piece, then "S status"
//   trims <n> (seq absgp dur discard)*n -> the n trim_end values
//   durs <bs0> <bs1> <n_modes> <mask> <n> (head head_len)*n -> "dur discard" per packet
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/symgpu/packetizer.hpp"

using namespace symgpu::packet;

namespace {

struct Sink {
    std::vector<std::string> packets, pieces;
    std::vector<std::pair<uint64_t, uint32_t>> open;  // the current stream's pieces, indexed from 0
    uint32_t serial = 0, used = 0;
    uint64_t base = 0;                                 // pieces of the file's earlier streams
    void begin_stream(uint32_t s) { serial = s, used = 0, open.clear(); }
    void end_stream() {
        for (uint32_t k = 0; k < used; ++k) pieces.push_back("Q " + std::to_string(open[k].first) + " " + std::to_string(open[k].second));
        base += used;
    }
    void piece(uint32_t i, uint64_t offset, uint32_t len) {
        open.resize(i);
        open.emplace_back(offset, len);
    }
    void packet(uint32_t first, uint32_t count, uint64_t len, const OggPageHead& pg) {
        char line[160];
        std::snprintf(line, sizeof line, "P %u %u %llu %llu %llu %u 0", serial, pg.sequence, (unsigned long long)pg.absgp, (unsigned long long)len,
                      (unsigned long long)(base + first), count);
        packets.push_back(line);
        used = first + count;
    }
    void last_on_page() { packets.back().back() = '1'; }
};

// The device schedule, step by step, through the shared functions.
void index(const std::vector<uint8_t>& d) {
    static constexpr detail::Crc32Table tab{};
    const size_t n = d.size(), n_words = (n + 3) / 4;
    std::vector<uint32_t> succ(n_words), serial(n_words), offset(n_words), spare(n_words);
    for (size_t w = 0; w < n_words; ++w) succ[w] = ogg_successor_word(d.data(), n, w, tab.t);
    size_t pages = 0;
    for (uint64_t pos = 0, q; ogg_next_page(succ.data(), n, &pos, &q); ++pages) serial[pages] = detail::le32(d.data() + q + 14), offset[pages] = uint32_t(q);
    ogg_sort_by_serial(serial.data(), offset.data(), succ.data(), spare.data(), pages);
    Sink sink;
    const bool cap_hit = ogg_walk_streams(d.data(), serial.data(), offset.data(), pages, sink);
    for (const auto& p : sink.packets) std::printf("%s\n", p.c_str());
    for (const auto& p : sink.pieces) std::printf("%s\n", p.c_str());
    std::printf("S %d\n", int(cap_hit));
}

}  // namespace

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string mode;
        in >> mode;
        if (mode == "index") {
            std::string path;
            in >> path;
            std::ifstream f(path, std::ios::binary);
            std::vector<uint8_t> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
            index(d);
        } else if (mode == "trims") {
            size_t n;
            in >> n;
            std::vector<uint32_t> seq(n), dur(n), disc(n), out(n);
            std::vector<uint64_t> gp(n);
            for (size_t i = 0; i < n; ++i) in >> seq[i] >> gp[i] >> dur[i] >> disc[i];
            ogg_page_end_trims(seq.data(), gp.data(), dur.data(), disc.data(), n, out.data());
            for (size_t i = 0; i < n; ++i) std::printf("%u\n", out[i]);
        } else if (mode == "durs") {
            unsigned bs0, bs1, n_modes;
            unsigned long long mask;
            size_t n;
            in >> bs0 >> bs1 >> n_modes >> mask >> n;
            VorbisIdent id{2, 44100, uint8_t(bs0), uint8_t(bs1)};
            VorbisPacketTimer timer(id, uint8_t(n_modes), mask);
            for (size_t i = 0; i < n; ++i) {
                unsigned head, head_len;
                in >> head >> head_len;
                const uint8_t b[2] = {uint8_t(head & 0xff), uint8_t(head >> 8)};
                uint64_t dur, discard;
                timer.next(b, head_len, dur, discard);
                std::printf("%llu %llu\n", (unsigned long long)dur, (unsigned long long)discard);
            }
        }
        std::printf("end\n");
        std::fflush(stdout);
    }
    return 0;
}
