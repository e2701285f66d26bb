// The schedule of symgpu_mpa_index_dev (symphonia_b200/csrc/mpa_index_kernel.cu) run on the CPU through the same functions of
// include/symgpu/packetizer.hpp the kernels call, over many files in one buffer: the candidates in virtual byte order, their node
// words, successors S and hunt steps G, H jumping rounds of G, each file's first frame and track, K doubling rounds of the chains,
// the packets' samples, the exclusive scans over candidate order, the per-file records and the packets.  Input on stdin, one request
// per line:
//   index <path> <seekable> <h> <k> <n> (offset len)*n  -> "R H K" (the rounds mpa_hunt_rounds / mpa_chain_rounds give for these
//                                                       ranges), then per file "P <symgpu_mpa_packet fields>" per packet and
//                                                       "T status <symgpu_mpa_track fields>"; h / k < 0 run H / K rounds
//   extra <path> <n> (offset len)*n                   -> "X g r": the hunt entries and ranks a further round of each would change
//                                                       after H and K rounds (0 0: the rounds suffice)
//   minframe                                          -> "M m": the smallest frame any header word gives, header included
//   extrapolate                                       -> "E checked differ": mpa_extrapolate against double arithmetic
#include <algorithm>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "../../symphonia_b200/csrc/mpa_records.h"

using namespace symgpu::packet;

namespace {

struct File {
    uint64_t offset, len, vbase;
};

struct Schedule {
    const std::vector<uint8_t>& d;
    bool seekable;
    std::vector<File> files;
    std::vector<uint64_t> vpos;
    std::vector<uint32_t> node, rank, jump[2], hunt[2];
    uint32_t hunt_run = 0, chain_run = 0;

    size_t file_of(uint64_t v) const {  // the last file whose vbase <= v
        size_t lo = 0, hi = files.size();
        while (hi - lo > 1) {
            const size_t mid = (lo + hi) / 2;
            if (files[mid].vbase <= v) lo = mid;
            else hi = mid;
        }
        return lo;
    }
    const uint8_t* bytes(size_t i) const { return d.data() + files[i].offset; }

    Schedule(const std::vector<uint8_t>& data, const std::vector<std::pair<uint64_t, uint64_t>>& ranges, bool seek) : d(data), seekable(seek) {
        uint64_t total = 0;
        for (const auto& r : ranges) files.push_back(File{r.first, r.second, total}), total += r.second;
        size_t f = 0;
        for (uint64_t v = 0; v < total; ++v) {
            while (v >= files[f].vbase + files[f].len) ++f;
            const size_t q = size_t(v - files[f].vbase);
            if (mpa_is_candidate(bytes(f), size_t(files[f].len), q)) vpos.push_back(v), node.push_back(mpa_node(bytes(f), size_t(files[f].len), q));
        }
        const uint32_t n = uint32_t(vpos.size());
        rank.assign(n, kAdtsUnranked), jump[0].resize(n), jump[1].resize(n), hunt[0].resize(n), hunt[1].resize(n);
        for (uint32_t c = 0; c < n; ++c) {
            const size_t i = file_of(vpos[c]);
            const uint64_t end = files[i].vbase + files[i].len, q = vpos[c] - files[i].vbase;
            jump[0][c] = mpa_successor(vpos.data(), n, c, node[c], end);
            hunt[0][c] = mpa_hunt(vpos.data(), n, c, node[c], mpa_first_rejected(bytes(i), size_t(files[i].len), size_t(q), node[c]), jump[0][c], end);
        }
    }

    void hunt_round() {
        const uint32_t k = hunt_run++;
        for (uint32_t c = 0; c < vpos.size(); ++c) mpa_hunt_jump(hunt[k & 1].data(), hunt[(k + 1) & 1].data(), c);
    }
    const std::vector<uint32_t>& hunted() const { return hunt[hunt_run & 1]; }

    // the track step: each file's first candidate, its root, its track; the first frame ranked 0
    std::vector<uint32_t> fcand;
    std::vector<MpaTrack> tracks;
    std::vector<uint8_t> no_frame;
    void open() {
        const uint32_t n = uint32_t(vpos.size());
        fcand.assign(files.size() + 1, n), tracks.assign(files.size(), MpaTrack{}), no_frame.assign(files.size(), 0);
        for (size_t i = 0; i < files.size(); ++i) {
            const uint32_t c0 = detail::first_at_or_after(vpos.data(), 0, n, files[i].vbase);
            fcand[i] = c0;
            const uint32_t root = c0 < n && vpos[c0] < files[i].vbase + files[i].len ? hunted()[c0] : kMpaEnd;
            if (root == kMpaEnd || mpa_node_kind(node[root]) != kMpaFrame) {
                no_frame[i] = 1;
                continue;
            }
            mpa_open_track(crc16_ansi_le_table(), bytes(i), size_t(files[i].len), size_t(vpos[root] - files[i].vbase), seekable, tracks[i]);
            rank[root] = 0;
        }
    }

    void chain_round() {
        const uint32_t k = chain_run++;
        for (uint32_t c = 0; c < vpos.size(); ++c) adts_double(rank.data(), jump[k & 1].data(), jump[(k + 1) & 1].data(), c, k);
    }

    uint64_t max_len() const {
        uint64_t m = 0;
        for (const File& f : files) m = std::max(m, f.len);
        return m;
    }

    void print() const {
        const uint32_t n = uint32_t(vpos.size());
        std::vector<uint32_t> dur(n), pidx(n + 1);
        std::vector<uint64_t> before(n + 1);
        for (uint32_t c = 0; c < n; ++c) {
            const size_t i = file_of(vpos[c]);
            dur[c] = rank[c] == kAdtsUnranked ? 0 : mpa_packet_dur(crc16_ansi_le_table(), bytes(i), size_t(vpos[c] - files[i].vbase), node[c], rank[c], uint8_t(tracks[i].tag));
        }
        for (uint32_t c = 0; c < n; ++c) pidx[c + 1] = pidx[c] + (dur[c] != 0), before[c + 1] = before[c] + dur[c];
        std::vector<symgpu_mpa_packet> packets(pidx[n]);
        for (uint32_t c = 0; c < n; ++c) {
            if (!dur[c]) continue;
            const size_t i = file_of(vpos[c]);
            const uint64_t q = vpos[c] - files[i].vbase;
            const int64_t ts = int64_t(before[c] - before[fcand[i]]) - int64_t(tracks[i].delay);
            packets[pidx[c]] = symgpu_detail::mpa_packet_record(mpa_frame_packet(detail::be32(bytes(i) + q), q, ts, tracks[i]), bytes(i) + q);
        }
        for (size_t i = 0; i < files.size(); ++i) {
            for (uint32_t k = pidx[fcand[i]]; k < pidx[fcand[i + 1]]; ++k) {
                const symgpu_mpa_packet& p = packets[k];
                std::printf("P %llu %u %08x %lld %u %u %llu %d\n", (unsigned long long)p.offset, p.size, p.header, (long long)p.pts, p.dur, p.trim_start,
                            (unsigned long long)p.trim_end, p.main_data_begin);
            }
            const symgpu_mpa_track t = no_frame[i] ? symgpu_mpa_track{} : symgpu_detail::mpa_track_record(tracks[i]);
            std::printf("T %u %08x %u %u %u %u %u %u %u %u %u %llu %llu\n", no_frame[i], t.first_header, t.sample_rate, t.version, t.layer, t.channels,
                        t.tag, t.has_delay, t.has_num_frames, t.delay, t.padding, (unsigned long long)t.num_frames, (unsigned long long)t.first_packet_pos);
        }
    }
};

std::vector<uint8_t> read_file(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

}  // namespace

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string mode, path;
        in >> mode;
        if (mode == "extrapolate") {  // mpa_extrapolate against the double arithmetic it restates
            uint64_t checked = 0, differ = 0, rng = 0x9e3779b97f4a7c15u;
            auto next = [&] { return rng ^= rng << 13, rng ^= rng >> 7, rng ^= rng << 17; };
            for (uint64_t count = 1; count <= 17; ++count)
                for (uint64_t len = count; len <= 17 * 2881 + 4; ++len)
                    for (int k = 0; k < 6; ++k) {
                        uint64_t total = k == 0 ? len : k == 1 ? (next() % 4096) * len : k == 2 ? (next() % 1000) * len / count : next() % (uint64_t(1) << (k == 3 ? 32 : 20));
                        if (k == 4) total = next() % 100;
                        const uint64_t want = uint64_t(double(total) / (double(len) / double(count)));
                        differ += want != mpa_extrapolate(total, len, count), ++checked;
                    }
            std::printf("E %llu %llu\nend\n", (unsigned long long)checked, (unsigned long long)differ);
            std::fflush(stdout);
            continue;
        }
        if (mode == "minframe") {
            uint32_t m = ~0u;
            for (uint32_t low = 0; low < (1u << 21); ++low) {
                MpaHeader h;
                if (mpa_parse_header(0xffe00000u | low, h) == Status::Ok) m = std::min(m, 4 + h.frame_size);
            }
            std::printf("M %u\nend\n", m);
            std::fflush(stdout);
            continue;
        }
        in >> path;
        long seekable = 1, h = -1, k = -1;
        if (mode == "index") in >> seekable >> h >> k;
        size_t n;
        in >> n;
        std::vector<std::pair<uint64_t, uint64_t>> ranges(n);
        for (auto& r : ranges) in >> r.first >> r.second;
        const std::vector<uint8_t> d = read_file(path);
        Schedule s(d, ranges, seekable != 0);
        const uint32_t H = mpa_hunt_rounds(s.max_len()), K = mpa_chain_rounds(s.max_len());
        for (long r = 0; r < (h < 0 ? long(H) : h); ++r) s.hunt_round();
        if (mode == "index") {
            std::printf("R %u %u\n", H, K);
            s.open();
            for (long r = 0; r < (k < 0 ? long(K) : k); ++r) s.chain_round();
            s.print();
        } else if (mode == "extra") {
            const std::vector<uint32_t> g = s.hunted();
            s.hunt_round();
            size_t g_changed = 0;
            for (size_t c = 0; c < g.size(); ++c) g_changed += g[c] != s.hunted()[c];
            s.hunt_run--;  // the track step reads the H-round hunt
            s.open();
            for (uint32_t r = 0; r < K; ++r) s.chain_round();
            auto ranked = [&] { return size_t(std::count_if(s.rank.begin(), s.rank.end(), [](uint32_t x) { return x != kAdtsUnranked; })); };
            const size_t before = ranked();
            s.chain_round();
            std::printf("X %zu %zu\n", g_changed, ranked() - before);
        }
        std::printf("end\n");
        std::fflush(stdout);
    }
    return 0;
}
