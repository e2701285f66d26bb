// Host driver of the shared ALAC packet decoder (symphonia_b200/csrc/alac_entropy.h), for tests/test_alac_entropy_shared.py and
// tests/test_alac_fuzz_sanitized.py.  Built plainly, with -DSYMGPU_MP3E_DEVICE_WINDOW (the bit window the device composes from
// byte loads), and with AddressSanitizer + UndefinedBehaviorSanitizer; linked with oracle/oracle_alac.cpp.
//
//   alac_entropy_driver IN
// IN: per packet u32 frame_length, bit_depth, pb, mb, kb, channels, len, then len bytes.
// Each packet is decoded three ways: by symgpu_alac_fe_decode_packets, by the three shared functions called as the device kernels
// call them (each buffer exactly as large as the packet's job: 8 channel records, channels x frame_length samples and tail bits),
// and by oracle_alac_packet.  Prints "packets decoded refused mismatches"; exit status 1 on any mismatch.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../symphonia_b200/csrc/alac_entropy.h"

extern "C" int oracle_alac_packet(const uint8_t* data, size_t len, uint32_t frame_length, uint32_t bit_depth, uint32_t pb, uint32_t mb, uint32_t kb,
                                  uint32_t channels, int32_t* planes, uint32_t* frames);

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::vector<uint8_t> in;
    if (FILE* f = std::fopen(argv[1], "rb")) {
        uint8_t buf[65536];
        size_t got;
        while ((got = std::fread(buf, 1, sizeof buf, f)) > 0) in.insert(in.end(), buf, buf + got);
        std::fclose(f);
    } else {
        return 2;
    }
    using namespace symgpu::alac;
    size_t at = 0, n = 0, decoded = 0, refused = 0, bad = 0;
    while (at + 28 <= in.size()) {
        uint32_t h[7];
        std::memcpy(h, in.data() + at, 28);
        at += 28;
        if (h[6] > in.size() - at) return 2;
        // the packet in its own allocation, so that a read past its end is the sanitizer's to see
        std::vector<uint8_t> pkt(in.begin() + at, in.begin() + at + h[6]);
        at += h[6];
        ++n;
        symgpu_alac_group g{};
        g.frame_length = h[0], g.bit_depth = uint8_t(h[1]), g.pb = uint8_t(h[2]), g.mb = uint8_t(h[3]), g.kb = uint8_t(h[4]), g.channels = uint8_t(h[5]);
        const uint32_t ch = g.channels, fl = g.frame_length;
        // 1. the front-end
        symgpu_piece piece{0, h[6], 0};
        uint8_t st = 9;
        uint32_t fe_frames = 0;
        std::vector<int32_t> fe(size_t(ch) * fl + 1);
        size_t n_fe = 0;
        const symgpu_status rc = symgpu_alac_fe_decode_packets(pkt.data(), pkt.size(), &piece, 1, &g, &st, &fe_frames, fe.data(), fe.size(), &n_fe);
        if (rc != SYMGPU_OK) return 3;
        // 2. as the kernels call the shared functions
        const Config cfg{fl, g.bit_depth, g.pb, g.mb, g.kb, ch};
        std::vector<Channel> recs(8);
        std::vector<int32_t> planes(size_t(ch) * fl);
        std::vector<uint16_t> tails(size_t(ch) * fl);
        uint32_t k_frames = 0;
        const int r = decode_packet(pkt.data(), pkt.size(), cfg, recs.data(), planes.data(), tails.data(), fl, &k_frames);
        std::vector<int32_t> dev;
        if (r == kDecoded) {
            for (uint32_t c = 0; c < ch; ++c) predict_channel(recs[c], planes.data() + size_t(c) * fl);
            for (uint32_t t = 0; t < k_frames; ++t)
                for (uint32_t c = 0; c < ch; ++c)
                    dev.push_back(finish_sample(recs[c], planes.data() + size_t(c) * fl, planes.data() + size_t(recs[c].partner) * fl,
                                                tails.data() + size_t(c) * fl, t, cfg.bit_depth));
        }
        // 3. the oracle
        std::vector<int32_t> o(size_t(ch) * (fl ? fl : 1));
        uint32_t o_frames = 0;
        const int orc = oracle_alac_packet(pkt.data(), pkt.size(), fl, g.bit_depth, g.pb, g.mb, g.kb, ch, o.data(), &o_frames);
        bool same = (orc == 0) == (st == kDecoded) && (r == kDecoded) == (st == kDecoded);
        if (same && orc == 0) {
            same = fe_frames == o_frames && k_frames == o_frames && n_fe == size_t(o_frames) * ch && dev.size() == n_fe;
            for (uint32_t t = 0; same && t < o_frames; ++t)
                for (uint32_t c = 0; c < ch; ++c)
                    if (fe[size_t(t) * ch + c] != o[size_t(c) * fl + t] || dev[size_t(t) * ch + c] != fe[size_t(t) * ch + c]) same = false;
        }
        decoded += orc == 0, refused += orc != 0, bad += !same;
    }
    std::printf("%zu %zu %zu %zu\n", n, decoded, refused, bad);
    return bad ? 1 : 0;
}
