// Host driver of the shared Layer III packet rules (symphonia_b200/csrc/mp3_entropy.h), for tests/test_mp3_entropy_shared.py.
// Built with -DSYMGPU_MP3E_DEVICE_WINDOW (the bit window the device composes from byte loads) and, in a second build, with
// AddressSanitizer + UndefinedBehaviorSanitizer.
//
//   mp3_entropy_driver IN OUT
// IN:  u32 n_files; per file u32 n_packets, per packet u32 len, len bytes.
// OUT: 1. per file, what symgpu_mp3_fe_decode_packets returns: u64 status, u64 n_good, frame_of [n_good] u32, units [n_good][4],
//         quant [n_good][4][576] i16;
//      2. the device schedule, on the CPU: the prologue of every packet of every file first (the first one of a file that
//         passes fixes its specification), then the side read of every packet; then rounds: the reservoir walk per file
//         (only the files that failed in the previous round, with their first failed frame marked), the main-data gather,
//         and every granule-channel job of those files decoded on its own in a shuffled order.  Per file: u32 rounds, u8
//         status per packet (0 decoded, 1 refused, 2 failed, 3 left out), units and quant of the decoded frames in stream
//         order.  Each packet lives in a buffer of exactly its length, each file's main data in a buffer of 2048 bytes per
//         packet.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../symphonia_b200/csrc/mp3_entropy.h"

namespace {

namespace me = symgpu::mp3e;

template <class T>
void put(std::vector<uint8_t>& out, const T* p, size_t n) {
    const uint8_t* b = reinterpret_cast<const uint8_t*>(p);
    out.insert(out.end(), b, b + n * sizeof(T));
}

uint32_t u32_at(const std::vector<uint8_t>& in, size_t at) {
    uint32_t v;
    std::memcpy(&v, in.data() + at, 4);
    return v;
}

struct File {
    std::vector<std::vector<uint8_t>> own;  // every packet in a buffer of its own size
    std::vector<uint8_t> data;
    std::vector<symgpu_mpa_packet> packets;
};

}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    std::vector<uint8_t> in;
    if (FILE* f = std::fopen(argv[1], "rb")) {
        uint8_t buf[65536];
        size_t got;
        while ((got = std::fread(buf, 1, sizeof buf, f)) > 0) in.insert(in.end(), buf, buf + got);
        std::fclose(f);
    } else {
        return 2;
    }
    if (in.size() < 4) return 2;
    const uint32_t n_files = u32_at(in, 0);
    std::vector<File> files(n_files);
    size_t at = 4;
    for (File& F : files) {
        if (at + 4 > in.size()) return 2;
        const uint32_t n_packets = u32_at(in, at);
        at += 4;
        for (uint32_t i = 0; i < n_packets; ++i) {
            if (at + 4 > in.size()) return 2;
            const uint32_t len = u32_at(in, at);
            at += 4;
            if (at + len > in.size()) return 2;
            symgpu_mpa_packet p{};
            p.offset = F.data.size(), p.size = len;
            F.packets.push_back(p);
            F.data.insert(F.data.end(), in.begin() + long(at), in.begin() + long(at + len));
            F.own.emplace_back(in.begin() + long(at), in.begin() + long(at + len));
            at += len;
        }
    }
    std::vector<uint8_t> out;
    // 1. the front-end loop
    for (File& F : files) {
        const size_t n = F.packets.size();
        std::vector<symgpu_mp3_gc> units(std::max<size_t>(n, 1) * 4);
        std::vector<int16_t> quant(std::max<size_t>(n, 1) * 4 * 576);
        std::vector<uint32_t> frame_of(std::max<size_t>(n, 1));
        symgpu_mp3_fe* fe = nullptr;
        if (symgpu_mp3_fe_create(&fe) != SYMGPU_OK) return 2;
        size_t good = 0;
        const symgpu_status st = symgpu_mp3_fe_decode_packets(fe, F.data.data(), F.data.size(), F.packets.data(), n, units.data(), quant.data(),
                                                              frame_of.data(), &good, nullptr);
        symgpu_mp3_fe_destroy(fe);
        const uint64_t head[2] = {uint64_t(st), good};
        put(out, head, 2);
        put(out, frame_of.data(), good);
        put(out, units.data(), good * 4);
        put(out, quant.data(), good * 4 * 576);
    }
    // 2. the device schedule
    struct Head {
        bool ok;
        size_t q;
        symgpu::packet::MpaHeader h;
    };
    std::vector<std::vector<Head>> heads(n_files);
    for (uint32_t f = 0; f < n_files; ++f)  // prologue pass
        for (const auto& p : files[f].own) {
            Head hd{};
            hd.ok = me::read_header(p.data(), p.size(), hd.h, hd.q) == me::kDecoded;
            heads[f].push_back(hd);
        }
    const me::LongEdges& E = symgpu::mp3_long_edges_host();
    std::vector<std::vector<me::FrameSide>> sides(n_files);
    for (uint32_t f = 0; f < n_files; ++f) {  // side pass
        const Head* first = nullptr;
        for (const Head& hd : heads[f])
            if (hd.ok) {
                first = &hd;
                break;
            }
        for (size_t i = 0; i < files[f].own.size(); ++i) {
            me::FrameSide s{};
            s.state = me::kSideRefused;
            const Head& hd = heads[f][i];
            uint32_t a, b;
            if (hd.ok && hd.h.sample_rate == first->h.sample_rate && hd.h.n_channels() == first->h.n_channels() &&
                me::body_of(hd.h, 3, files[f].own[i].size(), hd.q, a, b))
                me::read_frame_side(files[f].own[i].data() + a, a, b, hd.h, E, s);
            sides[f].push_back(s);
        }
    }
    const me::HuffSet& hs = symgpu::mp3_huffset_host(nullptr);
    std::vector<std::vector<uint8_t>> bad(n_files), status(n_files), md(n_files);
    std::vector<std::vector<me::GcJob>> gc(n_files);
    std::vector<std::vector<uint32_t>> slot_job(n_files);
    std::vector<std::vector<symgpu_mp3_gc>> units(n_files);
    std::vector<std::vector<int16_t>> quant(n_files);
    std::vector<uint32_t> rounds(n_files, 0), fail(n_files, ~0u);
    std::vector<uint8_t> redo(n_files, 1);
    for (uint32_t f = 0; f < n_files; ++f) {
        const size_t n = files[f].own.size();
        bad[f].assign(n, 0), status[f].assign(n, 1), md[f].assign(n * 2048, 0xA5);
        gc[f].resize(n * 4), slot_job[f].assign(n, ~0u), units[f].resize(n * 4), quant[f].resize(n * 4 * 576);
    }
    std::mt19937 rng(12345);
    for (;;) {
        for (uint32_t f = 0; f < n_files; ++f) {  // walk + gather of the files this round is for
            if (!redo[f]) continue;
            ++rounds[f];
            const size_t n = files[f].own.size();
            me::Reservoir r{0, 0, 0};
            uint32_t good = 0, back = 0;
            for (size_t i = 0; i < n; ++i) {
                const me::FrameSide& s = sides[f][i];
                me::GcJob four[4];
                me::StepOut o{};
                const int step = me::reservoir_step(r, s, bad[f][i] ? bad[f][i] : (s.mismatch ? 2 : 0), 0, four, o);
                const bool real = step == me::kStepDecoded || step == me::kStepLeftOut;
                const uint32_t slot = step == me::kStepDecoded ? good++ : uint32_t(n - 1 - back++);
                for (int q = 0; q < 4; ++q) {
                    if (!real) four[q] = me::GcJob{}, four[q].kind = me::kJobMute;
                    four[q].out_index = slot * 4 + uint32_t(q);
                    gc[f][slot * 4 + q] = four[q];
                }
                slot_job[f][slot] = real ? uint32_t(i) : ~0u;
                if (real) {
                    if (o.copy_at + o.slot > md[f].size()) {
                        std::printf("main data outside the file's region: file %u packet %zu\n", f, i);
                        return 1;
                    }
                    std::memcpy(md[f].data() + o.copy_at, files[f].own[i].data() + s.body_at + s.side_len, o.slot);
                }
                status[f][i] = uint8_t(step == me::kStepDecoded ? 0 : step == me::kStepFailed ? 2 : step == me::kStepLeftOut ? 3 : 1);
            }
        }
        struct Item {
            uint32_t file, t;
        };
        std::vector<Item> items;
        for (uint32_t f = 0; f < n_files; ++f)
            if (redo[f])
                for (uint32_t t = 0; t < gc[f].size(); ++t) items.push_back(Item{f, t});
        std::shuffle(items.begin(), items.end(), rng);
        for (const Item& it : items) {  // every granule-channel on its own
            const me::GcJob& j = gc[it.file][it.t];
            if (me::decode_gc_job(j, md[it.file].data(), hs, &units[it.file][it.t], &quant[it.file][size_t(it.t) * 576]))
                fail[it.file] = std::min(fail[it.file], slot_job[it.file][it.t >> 2]);
        }
        bool again = false;
        for (uint32_t f = 0; f < n_files; ++f) {
            redo[f] = fail[f] != ~0u;
            if (redo[f]) bad[f][fail[f]] = 1, fail[f] = ~0u, again = true;
        }
        if (!again) break;
    }
    uint32_t n_dec = 0;
    for (uint32_t f = 0; f < n_files; ++f) {
        put(out, &rounds[f], 1);
        put(out, status[f].data(), status[f].size());
        const size_t good = size_t(std::count(status[f].begin(), status[f].end(), uint8_t(0)));
        put(out, units[f].data(), good * 4);
        put(out, quant[f].data(), good * 4 * 576);
        n_dec += uint32_t(good);
    }
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 2;
    std::fwrite(out.data(), 1, out.size(), f);
    std::fclose(f);
    std::printf("%u files, %u frames decoded\n", n_files, n_dec);
    return 0;
}
