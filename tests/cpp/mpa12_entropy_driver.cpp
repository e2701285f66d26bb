// Host driver of the shared Layer I / II packet rules (symphonia_b200/csrc/mpa12_entropy.h), for tests/test_mpa12_entropy_shared.py.
// Built with -DSYMGPU_MP3E_DEVICE_WINDOW (the bit window the device composes from byte loads) and, in a second build, with
// AddressSanitizer + UndefinedBehaviorSanitizer.
//
//   mpa12_entropy_driver IN OUT
// IN:  u32 layer, n_packets; per packet u32 len, len bytes.
// OUT: 1. what symgpu_mpa12_fe_decode_packets returns over all packets: u64 status, u64 n_good, frame_of [n_good] u32, subbands
//         [n_good][2][32][n_slots] f32;
//      2. the device schedule, on the CPU: the prologue of every packet first (the first one that passes fixes the signal
//         specification), then the side read and the fit rule of every packet, then every sample codeword of every accepted
//         frame decoded on its own at its closed-form bit position, in a shuffled order: u8 accepted per packet, then the
//         accepted frames' subbands in stream order.  Each packet lives in a buffer of exactly its length.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../symphonia_b200/csrc/mpa12_entropy.h"

namespace {

namespace me = symgpu::mpa12e;

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
    if (in.size() < 8) return 2;
    const int layer = int(u32_at(in, 0));
    const uint32_t n_packets = u32_at(in, 4);
    const size_t n_slots = layer == 1 ? 12 : 36, per_frame = 64 * n_slots;
    std::vector<uint8_t> data;
    std::vector<symgpu_mpa_packet> packets(n_packets);
    std::vector<std::vector<uint8_t>> own(n_packets);  // every packet in a buffer of its own size
    size_t at = 8;
    for (uint32_t i = 0; i < n_packets; ++i) {
        if (at + 4 > in.size()) return 2;
        const uint32_t len = u32_at(in, at);
        at += 4;
        if (at + len > in.size()) return 2;
        packets[i] = symgpu_mpa_packet{};
        packets[i].offset = data.size(), packets[i].size = len;
        data.insert(data.end(), in.begin() + long(at), in.begin() + long(at + len));
        own[i].assign(in.begin() + long(at), in.begin() + long(at + len));
        at += len;
    }
    std::vector<uint8_t> out;
    // 1. the front-end loop
    {
        std::vector<float> sub(std::max<size_t>(n_packets, 1) * per_frame);
        std::vector<uint32_t> frame_of(std::max<uint32_t>(n_packets, 1));
        size_t good = 0;
        const symgpu_status st = symgpu_mpa12_fe_decode_packets(data.data(), data.size(), packets.data(), n_packets, layer, sub.data(), frame_of.data(),
                                                                &good, nullptr);
        const uint64_t head[2] = {uint64_t(st), good};
        put(out, head, 2);
        put(out, frame_of.data(), good);
        put(out, sub.data(), good * per_frame);
    }
    // 2. the device schedule
    const me::Constants& K = me::host_constants();
    std::vector<me::MpaHeader> heads(n_packets);
    std::vector<size_t> qs(n_packets);
    std::vector<uint8_t> head_ok(n_packets, 0);
    uint32_t first = n_packets;
    for (uint32_t i = 0; i < n_packets; ++i) {  // prologue pass
        head_ok[i] = me::read_header(own[i].data(), own[i].size(), heads[i], qs[i]) == me::kDecoded;
        if (head_ok[i] && first == n_packets) first = i;
    }
    std::vector<me::Side> sides(n_packets);
    std::vector<uint8_t> accepted(n_packets, 0);
    std::vector<uint32_t> place(n_packets, 0);
    uint32_t n_acc = 0;
    for (uint32_t i = 0; i < n_packets; ++i) {  // side pass
        if (!head_ok[i]) continue;
        const me::MpaHeader& h = heads[i];
        if (h.sample_rate != heads[first].sample_rate || h.n_channels() != heads[first].n_channels()) continue;
        me::Side& s = sides[i];
        if (!me::body_of(h, layer, own[i].size(), qs[i], s.body_at, s.body_bytes)) continue;
        if (!me::read_side(K, own[i].data() + s.body_at, h, s) || !me::fits(s)) continue;
        accepted[i] = 1, place[i] = n_acc++;
    }
    put(out, accepted.data(), n_packets);
    // sample pass: every (frame, granule, sub-band, channel) codeword on its own, shuffled; NaN marks what nobody wrote
    std::vector<float> sub(size_t(n_acc) * per_frame, __builtin_nanf(""));
    struct Item {
        uint32_t packet;
        uint8_t gr, sb, c;
    };
    std::vector<Item> items;
    for (uint32_t i = 0; i < n_packets; ++i)
        if (accepted[i])
            for (int gr = 0; gr < 12; ++gr)
                for (int sb = 0; sb < 32; ++sb)
                    for (int c = 0; c < 2; ++c) items.push_back(Item{i, uint8_t(gr), uint8_t(sb), uint8_t(c)});
    std::mt19937 rng(12345);
    std::shuffle(items.begin(), items.end(), rng);
    const int per = layer == 1 ? 1 : 3;
    for (const Item& it : items) {
        const me::Side& s = sides[it.packet];
        float* o = sub.data() + size_t(place[it.packet]) * per_frame + (size_t(it.c) * 32 + it.sb) * n_slots + size_t(it.gr) * per;
        if (it.c >= s.n_ch) {
            for (int k = 0; k < per; ++k) o[k] = 0.0f;
        } else if (!me::decode_codeword(K, s, own[it.packet].data() + s.body_at, it.gr, it.sb, it.c, o)) {
            std::printf("codeword read past the body after fits(): packet %u\n", it.packet);
            return 1;
        }
    }
    put(out, sub.data(), sub.size());
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 2;
    std::fwrite(out.data(), 1, out.size(), f);
    std::fclose(f);
    std::printf("%u packets, %u accepted\n", n_packets, n_acc);
    return 0;
}
