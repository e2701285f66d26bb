// The schedule of symgpu_adts_index_dev (symphonia_b200/csrc/adts_index_kernel.cu) run on the CPU through the same functions of
// include/symgpu/packetizer.hpp the kernels call, over many files in one buffer: the candidates in virtual byte order, their
// successors, K doubling rounds with ping-pong jump arrays, the per-file records from the chains' ends, the exclusive sum of the
// packet counts, the packets.  Input on stdin, one request per line:
//   index <path> <rounds> <n> (offset len)*n   -> "K k" (the rounds adts_rounds gives for these ranges), then per file "P offset
//                                               size sample_rate pts channels profile" per packet and "S stop sample_rate channels
//                                               profile"; rounds < 0 runs K rounds, else that many
//   extra <path> <n> (offset len)*n           -> "X m": the ranks a further round would add after K rounds (0: K rounds suffice)
#include <algorithm>
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

struct File {
    uint64_t offset, len, vbase;
};

struct Schedule {
    std::vector<File> files;
    std::vector<uint64_t> vpos;
    std::vector<uint32_t> node, rank, jump[2];
    uint32_t rounds_run = 0;

    size_t file_of(uint64_t v) const {  // the last file whose vbase <= v
        size_t lo = 0, hi = files.size();
        while (hi - lo > 1) {
            const size_t mid = (lo + hi) / 2;
            if (files[mid].vbase <= v) lo = mid;
            else hi = mid;
        }
        return lo;
    }

    Schedule(const std::vector<uint8_t>& d, const std::vector<std::pair<uint64_t, uint64_t>>& ranges) {
        uint64_t total = 0;
        for (const auto& r : ranges) files.push_back(File{r.first, r.second, total}), total += r.second;
        size_t f = 0;
        for (uint64_t v = 0; v < total; ++v) {
            while (v >= files[f].vbase + files[f].len) ++f;
            const File& fd = files[f];
            const size_t q = size_t(v - fd.vbase);
            if (adts_is_candidate(d.data() + fd.offset, size_t(fd.len), q)) vpos.push_back(v), node.push_back(adts_node(d.data() + fd.offset, size_t(fd.len), q));
        }
        const uint32_t n = uint32_t(vpos.size());
        rank.resize(n), jump[0].resize(n), jump[1].resize(n);
        for (uint32_t c = 0; c < n; ++c) {
            const File& fd = files[file_of(vpos[c])];
            const uint32_t s = adts_successor(vpos.data(), n, c, node[c], fd.vbase + fd.len);
            jump[0][c] = s;
            if (s == kAdtsEnd) node[c] |= kAdtsLast;
            rank[c] = adts_initial_rank(vpos.data(), c, fd.vbase);
        }
    }

    void round() {
        const uint32_t k = rounds_run++;
        for (uint32_t c = 0; c < vpos.size(); ++c) adts_double(rank.data(), jump[k & 1].data(), jump[(k + 1) & 1].data(), c, k);
    }

    uint64_t max_len() const {
        uint64_t m = 0;
        for (const File& f : files) m = std::max(m, f.len);
        return m;
    }

    size_t ranked() const { return size_t(std::count_if(rank.begin(), rank.end(), [](uint32_t r) { return r != kAdtsUnranked; })); }

    void print(const std::vector<uint8_t>& d) const {
        const size_t nf = files.size();
        std::vector<uint32_t> n_packets(nf, 0), stop(nf, kAdtsStopOk), rate(nf, 0), ch(nf, 0), profile(nf, 0);
        for (uint32_t c = 0; c < vpos.size(); ++c) {
            if (rank[c] == kAdtsUnranked) continue;
            const size_t i = file_of(vpos[c]);
            if (node[c] & kAdtsLast) adts_file_end(node[c], rank[c], &n_packets[i], &stop[i]);
            if (rank[c] == 0 && (node[c] & 7) == kAdtsFrame) {
                const AdtsPacket p = adts_frame_packet(d.data() + files[i].offset, size_t(files[i].len), size_t(vpos[c] - files[i].vbase), 0);
                rate[i] = p.sample_rate, ch[i] = p.channels, profile[i] = p.profile;
            }
        }
        std::vector<uint64_t> first(nf, 0);
        for (size_t i = 1; i < nf; ++i) first[i] = first[i - 1] + n_packets[i - 1];
        std::vector<AdtsPacket> packets(nf ? first[nf - 1] + n_packets[nf - 1] : 0);
        for (uint32_t c = 0; c < vpos.size(); ++c) {
            if (rank[c] == kAdtsUnranked || (node[c] & 7) != kAdtsFrame) continue;
            const size_t i = file_of(vpos[c]);
            const uint64_t at = first[i] + rank[c];
            if (at >= first[i] + n_packets[i]) continue;  // ranked past its file's end: only when too few rounds ran
            packets[at] = adts_frame_packet(d.data() + files[i].offset, size_t(files[i].len), size_t(vpos[c] - files[i].vbase), rank[c]);
        }
        for (size_t i = 0; i < nf; ++i) {
            for (uint64_t k = first[i]; k < first[i] + n_packets[i]; ++k) {
                const AdtsPacket& p = packets[k];
                std::printf("P %llu %u %u %lld %u %u\n", (unsigned long long)p.offset, p.size, p.sample_rate, (long long)p.pts, p.channels, p.profile);
            }
            std::printf("S %u %u %u %u\n", stop[i], rate[i], ch[i], profile[i]);
        }
    }
};

}  // namespace

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string mode, path;
        in >> mode >> path;
        long rounds = -1;
        if (mode == "index") in >> rounds;
        size_t n;
        in >> n;
        std::vector<std::pair<uint64_t, uint64_t>> ranges(n);
        for (auto& r : ranges) in >> r.first >> r.second;
        std::ifstream f(path, std::ios::binary);
        const std::vector<uint8_t> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        Schedule s(d, ranges);
        const uint32_t k = adts_rounds(s.max_len());
        if (mode == "index") {
            std::printf("K %u\n", k);
            for (long r = 0; r < (rounds < 0 ? long(k) : rounds); ++r) s.round();
            s.print(d);
        } else if (mode == "extra") {
            for (uint32_t r = 0; r < k; ++r) s.round();
            const size_t before = s.ranked();
            s.round();
            std::printf("X %zu\n", s.ranked() - before);
        }
        std::printf("end\n");
        std::fflush(stdout);
    }
    return 0;
}
