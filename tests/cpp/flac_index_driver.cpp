// The schedule of symgpu_flac_index_dev (symphonia_b200/csrc/flac_index_kernel.cu) run on the CPU through the same functions of
// include/symgpu/packetizer.hpp the kernels call, over many files in one buffer: each file's open(), the tiles of 4096 bytes in
// spans of 16 bytes, their CRC key shares and the xor-scan over them, the nodes with their keys, each node's header, the stable
// radix sort by key in 4-bit passes, the two max trees, the end search, the successors, K doubling rounds, the scans over node
// order and the packets.  Input on stdin, one request per line:
//   index <path> <k> <n> (offset len)*n  -> "R T K" (the tree levels flac_tree_levels and the rounds flac_chain_rounds give for these
//                                          ranges), then per file "P offset ts size dur" per packet and "I open <info fields>";
//                                          k < 0 runs K rounds
//   extra <path> <n> (offset len)*n      -> "X r": the ranks a further doubling round would add after K rounds (0: K suffice)
//   crc <seed> <count>                   -> "C checked differ": crc16_combine and flac_key_part against crc16_ansi_update on random
//                                          spans
#include <algorithm>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "../../symphonia_b200/csrc/flac_records.h"

using namespace symgpu::packet;

namespace {

constexpr uint64_t kTile = 4096, kSpan = 16, kNodeTile = 4096;

struct File {
    uint64_t offset, len, vbase;
};
struct Opened {
    FlacStreamInfo info{};
    uint64_t first_frame = 0;
    Status status = Status::Ok;
};

struct Schedule {
    const std::vector<uint8_t>& d;
    std::vector<File> files;
    std::vector<Opened> opened;
    uint64_t total = 0;
    std::vector<uint64_t> vpos;
    std::vector<uint32_t> node, key, fx0, fnode, skey, sid, ends, rank, jump[2];
    std::vector<FlacHead> head;
    std::vector<uint64_t> ev, sv, gv;
    std::vector<std::vector<uint64_t>> ends_levels, good_levels;
    uint32_t top = 0, chain_run = 0;

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

    // the CRC key share of virtual bytes [v0, v1), one part per file they touch (thread_key_share)
    uint16_t share(uint64_t v0, uint64_t v1) const {
        uint16_t x = 0;
        for (uint64_t v = v0; v < v1;) {
            const size_t f = file_of(v);
            const File& fd = files[f];
            const uint64_t e = std::min(fd.vbase + fd.len, v1);
            x ^= flac_key_part(crc16_ansi_table(), bytes(f), size_t(fd.len), size_t(v - fd.vbase), size_t(e - fd.vbase));
            v = e;
        }
        return x;
    }

    static FlacTree tree(const std::vector<uint64_t>& level0, std::vector<std::vector<uint64_t>>& levels, uint32_t top) {
        levels.assign(top, {});
        FlacTree t{};
        t.n = uint32_t(level0.size()), t.top = top, t.level[0] = level0.data();
        const std::vector<uint64_t>* below = &level0;
        for (uint32_t k = 1; k <= top; ++k) {
            levels[k - 1].resize((below->size() + 1) / 2);
            for (size_t j = 0; j < levels[k - 1].size(); ++j) levels[k - 1][j] = flac_tree_max(below->data(), below->size(), j);
            below = &levels[k - 1];
            t.level[k] = below->data();
        }
        return t;
    }

    Schedule(const std::vector<uint8_t>& data, const std::vector<std::pair<uint64_t, uint64_t>>& ranges) : d(data) {
        uint64_t longest = 0;
        for (const auto& r : ranges) files.push_back(File{r.first, r.second, total}), total += r.second, longest = std::max(longest, r.second);
        top = flac_tree_levels(longest);
        // open(), one file at a time
        for (size_t i = 0; i < files.size(); ++i) {
            Opened o;
            size_t first = 0;
            o.status = flac_open(bytes(i), size_t(files[i].len), o.info, &first);
            o.first_frame = first;
            opened.push_back(o);
        }
        // the tiles' key shares, their exclusive xor-scan, and the walk that gives every node its key prefix
        const uint64_t n_tiles = (total + kTile - 1) / kTile;
        std::vector<uint16_t> tile_x(n_tiles + 1, 0);
        for (uint64_t t = 0; t < n_tiles; ++t)
            for (uint64_t v0 = t * kTile; v0 < std::min(total, (t + 1) * kTile); v0 += kSpan) tile_x[t] ^= share(v0, std::min(total, v0 + kSpan));
        uint16_t carry = 0;
        for (auto& x : tile_x) {
            const uint16_t here = x;
            x = carry, carry ^= here;
        }
        fx0.assign(files.size(), 0);
        for (uint64_t t = 0; t < n_tiles; ++t) {
            uint16_t pre = tile_x[t];
            for (uint64_t v0 = t * kTile; v0 < std::min(total, (t + 1) * kTile); v0 += kSpan) {
                const uint64_t v1 = std::min(total, v0 + kSpan);
                for (uint64_t v = v0; v < v1;) {
                    const size_t f = file_of(v);
                    const File& fd = files[f];
                    const uint8_t* b = bytes(f);
                    const size_t n = size_t(fd.len);
                    const uint64_t e = std::min(fd.vbase + fd.len, v1);
                    uint16_t s = 0;
                    for (uint64_t u = v; u < e; ++u) {
                        const size_t q = size_t(u - fd.vbase);
                        if (q == 0) fx0[f] = pre;
                        if (flac_is_node(b, n, q)) {
                            const bool end = flac_node(n, q) & kFlacEndNode;
                            const uint16_t s_at = end ? crc16_ansi_update(s, b + q, 1) : s;
                            vpos.push_back(u), node.push_back(flac_node(n, q)), key.push_back(pre ^ flac_key_inside(s_at, n, end ? n : q));
                        }
                        s = crc16_ansi_update(s, b + q, 1);
                    }
                    pre ^= flac_key_inside(s, n, size_t(e - fd.vbase));
                    v = e;
                }
            }
        }
        const uint32_t nn = uint32_t(vpos.size());
        // each file's first node; each node's header, sort key and end-search value
        fnode.resize(files.size() + 1);
        for (size_t i = 0; i < files.size(); ++i) fnode[i] = detail::first_at_or_after(vpos.data(), 0, nn, files[i].vbase);
        fnode[files.size()] = nn;
        head.resize(nn), skey.resize(nn), sid.resize(nn), ev.resize(nn);
        for (uint32_t c = 0; c < nn; ++c) {
            const size_t i = file_of(vpos[c]);
            const Opened& o = opened[i];
            head[c] = flac_head(bytes(i), size_t(files[i].len), size_t(vpos[c] - files[i].vbase), node[c], o.status == Status::Ok, size_t(o.first_frame), o.info);
            skey[c] = (key[c] ^ fx0[i]) & 0xffff, sid[c] = c;
            ev[c] = flac_end_value(head[c], node[c]);
        }
        // the radix sort, 4 bits a pass, stable: counts per digit, then each node to its digit's next slot in node order
        for (uint32_t p = 0; p < 4; ++p) {
            uint64_t at[16] = {}, base = 0;
            for (uint32_t c = 0; c < nn; ++c) ++at[(skey[c] >> (4 * p)) & 15];
            for (auto& a : at) {
                const uint64_t here = a;
                a = base, base += here;
            }
            std::vector<uint32_t> k2(nn), i2(nn);
            for (uint32_t c = 0; c < nn; ++c) {
                const uint64_t slot = at[(skey[c] >> (4 * p)) & 15]++;
                k2[slot] = skey[c], i2[slot] = sid[c];
            }
            skey.swap(k2), sid.swap(i2);
        }
        sv.resize(nn);
        for (uint32_t i = 0; i < nn; ++i) sv[i] = ev[sid[i]];
        const FlacTree ends_tree = tree(sv, ends_levels, top);
        // the ends
        ends.assign(nn, kFlacNone), gv.assign(nn, 0), rank.assign(nn, kAdtsUnranked);
        for (uint32_t c = 0; c < nn; ++c) {
            if (!head[c].plausible) continue;
            const size_t i = file_of(vpos[c]);
            ends[c] = flac_end(vpos.data(), node.data(), c, fnode[i + 1], files[i].vbase, head[c], (key[c] ^ fx0[i]) & 0xffff, skey.data(), sid.data(), ends_tree);
            gv[c] = ends[c] == kFlacNone ? 0 : flac_value(head[c].seq);
        }
        const FlacTree good_tree = tree(gv, good_levels, top);
        // successors and first frames
        jump[0].resize(nn), jump[1].resize(nn);
        for (size_t i = 0; i < files.size(); ++i) {
            if (opened[i].status != Status::Ok) continue;
            const uint32_t a = flac_first_frame(vpos.data(), node.data(), fnode[i], fnode[i + 1], files[i].vbase, size_t(opened[i].first_frame), good_tree);
            if (a != kFlacNone) rank[a] = 0;
        }
        for (uint32_t c = 0; c < nn; ++c) jump[0][c] = flac_successor(node.data(), ends[c], fnode[file_of(vpos[c]) + 1], head[c].seq, good_tree);
    }

    void chain_round() {
        const uint32_t k = chain_run++;
        for (uint32_t c = 0; c < vpos.size(); ++c) adts_double(rank.data(), jump[k & 1].data(), jump[(k + 1) & 1].data(), c, k);
    }

    void print() const {
        const uint32_t nn = uint32_t(vpos.size());
        std::vector<uint32_t> dur(nn), pidx(nn + 1);
        for (uint32_t c = 0; c < nn; ++c) dur[c] = rank[c] == kAdtsUnranked ? 0 : head[c].block;
        for (uint32_t c = 0; c < nn; ++c) pidx[c + 1] = pidx[c] + (dur[c] != 0);
        std::vector<symgpu_flac_packet> packets(pidx[nn]);
        for (uint32_t c = 0; c < nn; ++c) {
            if (!dur[c]) continue;
            const size_t i = file_of(vpos[c]);
            packets[pidx[c]] = symgpu_detail::flac_packet_record(
                flac_chain_packet(vpos[c] - files[i].vbase, flac_npos(vpos.data(), node.data(), ends[c], files[i].vbase), head[c], opened[i].info));
        }
        for (size_t i = 0; i < files.size(); ++i) {
            for (uint32_t k = pidx[fnode[i]]; k < pidx[fnode[i + 1]]; ++k) {
                const symgpu_flac_packet& p = packets[k];
                std::printf("P %llu %llu %u %u\n", (unsigned long long)p.offset, (unsigned long long)p.ts, p.size, p.dur);
            }
            const Opened& o = opened[i];
            const int open = o.status == Status::Ok ? 0 : o.status == Status::Unsupported ? 2 : 1;
            const symgpu_flac_stream_info r = open ? symgpu_flac_stream_info{} : symgpu_detail::flac_info_record(o.info, o.first_frame);
            std::printf("I %d %llu %llu %u %u %u %u %u %u %u %u", open, (unsigned long long)r.n_samples, (unsigned long long)r.first_frame_pos,
                        r.sample_rate, r.frame_min, r.frame_max, r.block_min, r.block_max, r.channels, r.bits_per_sample, r.has_md5);
            for (int k = 0; k < 16; ++k) std::printf(" %u", r.md5[k]);
            std::printf("\n");
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
        if (mode == "crc") {  // (a, la) o (b, lb) and the key parts against the plain CRC over the joined bytes
            uint64_t seed, count, checked = 0, differ = 0;
            in >> seed >> count;
            uint64_t rng = seed * 0x9e3779b97f4a7c15u + 1;
            auto next = [&] { return rng ^= rng << 13, rng ^= rng >> 7, rng ^= rng << 17; };
            std::vector<uint8_t> buf;
            for (uint64_t k = 0; k < count; ++k) {
                const size_t n = size_t(next() % (k % 7 == 0 ? 70000 : 300)) + 1;
                buf.resize(n);
                for (auto& b : buf) b = uint8_t(next());
                const size_t a = size_t(next() % (n + 1)), b = a + size_t(next() % (n - a + 1));
                const uint16_t whole = crc16_ansi_update(0, buf.data(), b), left = crc16_ansi_update(0, buf.data(), a);
                const uint16_t right = crc16_ansi_update(0, buf.data() + a, b - a);
                differ += crc16_combine(left, right, b - a) != whole;
                // key parts: the xor of the parts of [0, a) and [a, b), over a file of n bytes, is the state of [0, b) times x^(8 (n - b))
                const uint16_t parts = flac_key_part(crc16_ansi_table(), buf.data(), n, 0, a) ^ flac_key_part(crc16_ansi_table(), buf.data(), n, a, b);
                differ += parts != crc16_mulmod(whole, crc16_xpow8(n - b));
                // and equal keys are exactly a matching CRC-16 in front of the later position
                if (b >= a + 2) {
                    const uint16_t ka = flac_key_inside(left, n, a), kb = flac_key_inside(whole, n, b);
                    differ += (ka == kb) != (crc16_ansi_update(0, buf.data() + a, b - a - 2) == detail::be16(buf.data() + b - 2));
                }
                checked += 1;
            }
            std::printf("C %llu %llu\nend\n", (unsigned long long)checked, (unsigned long long)differ);
            std::fflush(stdout);
            continue;
        }
        in >> path;
        long k = -1;
        if (mode == "index") in >> k;
        size_t n;
        in >> n;
        std::vector<std::pair<uint64_t, uint64_t>> ranges(n);
        uint64_t longest = 0;
        for (auto& r : ranges) in >> r.first >> r.second, longest = std::max(longest, r.second);
        const std::vector<uint8_t> d = read_file(path);
        Schedule s(d, ranges);
        const uint32_t K = flac_chain_rounds(longest);
        if (mode == "index") {
            std::printf("R %u %u\n", s.top, K);
            for (long r = 0; r < (k < 0 ? long(K) : k); ++r) s.chain_round();
            s.print();
        } else if (mode == "extra") {
            for (uint32_t r = 0; r < K; ++r) s.chain_round();
            auto ranked = [&] { return size_t(std::count_if(s.rank.begin(), s.rank.end(), [](uint32_t x) { return x != kAdtsUnranked; })); };
            const size_t before = ranked();
            s.chain_round();
            std::printf("X %zu\n", ranked() - before);
        }
        std::printf("end\n");
        std::fflush(stdout);
    }
    return 0;
}
