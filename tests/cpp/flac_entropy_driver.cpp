// Host driver of the shared FLAC frame decoder (symphonia_b200/csrc/flac_entropy.h), for tests/test_flac_entropy_shared.py.
// Built with -DSYMGPU_MP3E_DEVICE_WINDOW (the bit window the device composes from byte loads) and, in a second build, with
// AddressSanitizer + UndefinedBehaviorSanitizer.
//
//   flac_entropy_driver IN OUT
// IN:  u32 stream_bps, stream_channels, max_block, n_packets; per packet u32 slot, u32 len, len bytes.
// OUT: 1. what symgpu_flac_fe_decode_packets returns over all packets (status, n_good, n_subs, n_samples as u64, then frames,
//         infos, frame_of, subs, samples), its sample capacity grown from 64 samples on SYMGPU_ERR_LIMIT as a caller does;
//      2. per packet, decode_packet called as the device kernel calls it -- exactly channels sub-frame records and
//         channels x slot samples of room, each in a buffer of exactly that size -- : u8 status, then on kDecoded the frame,
//         info, its sub-frame records and its channels x block samples.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../symphonia_b200/csrc/flac_entropy.h"

namespace {

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
    if (in.size() < 16) return 2;
    const uint32_t bps = u32_at(in, 0), channels = u32_at(in, 4), max_block = u32_at(in, 8), n_packets = u32_at(in, 12);
    std::vector<uint8_t> data;
    std::vector<symgpu_piece> pieces(n_packets);
    std::vector<uint32_t> slots(n_packets);
    size_t at = 16;
    for (uint32_t i = 0; i < n_packets; ++i) {
        if (at + 8 > in.size()) return 2;
        slots[i] = u32_at(in, at);
        const uint32_t len = u32_at(in, at + 4);
        at += 8;
        if (at + len > in.size()) return 2;
        pieces[i] = symgpu_piece{data.size(), len, 0};
        data.insert(data.end(), in.begin() + long(at), in.begin() + long(at + len));
        at += len;
    }
    std::vector<uint8_t> out;
    // 1. the front-end loop
    {
        std::vector<symgpu_flac_frame> frames(n_packets);
        std::vector<symgpu_flac_frame_info> infos(n_packets);
        std::vector<uint32_t> frame_of(n_packets);
        std::vector<symgpu_flac_subframe> subs(size_t(n_packets) * 8);
        size_t cap = 64, good = 0, n_subs = 0, n_samples = 0;
        symgpu_status st;
        for (;;) {
            std::vector<int32_t> samples(cap);
            st = symgpu_flac_fe_decode_packets(data.data(), data.size(), pieces.data(), n_packets, bps, channels, max_block, frames.data(), infos.data(),
                                               frame_of.data(), subs.data(), subs.size(), samples.data(), cap, &good, &n_subs, &n_samples);
            if (st == SYMGPU_ERR_LIMIT) {
                cap *= 4;
                continue;
            }
            const uint64_t head[4] = {uint64_t(st), good, n_subs, n_samples};
            put(out, head, 4);
            put(out, frames.data(), good);
            put(out, infos.data(), good);
            put(out, frame_of.data(), good);
            put(out, subs.data(), n_subs);
            put(out, samples.data(), n_samples);
            break;
        }
    }
    // 2. one packet at a time, as the device kernel decodes it
    const uint32_t ch = channels ? channels : 8;
    for (uint32_t i = 0; i < n_packets; ++i) {
        std::vector<symgpu_flac_subframe> subs(ch);
        std::vector<int32_t> samples(size_t(ch) * slots[i]);
        symgpu_flac_frame frame{};
        symgpu_flac_frame_info info{};
        const int r = symgpu::flace::decode_packet(data.data() + pieces[i].offset, pieces[i].len, bps, channels, max_block, 0, subs.data(), ch, samples.data(), 0,
                                                   samples.size(), slots[i], &frame, &info);
        const uint8_t s = uint8_t(r);
        put(out, &s, 1);
        if (r == symgpu::flace::kDecoded) {
            put(out, &frame, 1);
            put(out, &info, 1);
            put(out, subs.data(), frame.channels);
            put(out, samples.data(), size_t(frame.channels) * info.block_size);
        }
    }
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 2;
    std::fwrite(out.data(), 1, out.size(), f);
    std::fclose(f);
    std::printf("%u packets\n", n_packets);
    return 0;
}
