// symgpu packetisers (SURVEY §8f N2): cut MPEG audio, ADTS and Ogg byte streams into codec packets the way
// the reference's format readers do, but as INDEX BUILDERS over one resident byte buffer.
//
// The reference pulls packets one at a time out of a consuming reader and copies each into its own allocation
// (symphonia-bundle-mp3/src/demuxer.rs:598-604, symphonia-codec-aac/src/adts.rs:303-308,
// symphonia-format-ogg/src/logical.rs:577-597).  A batched device decoder wants the opposite: the whole file
// goes to HBM in ONE copy and the front-end kernels are handed a table of (offset, length) references into it.
// So nothing here copies payload bytes: an MPEG / ADTS packet is a byte range of the source, an Ogg packet --
// which may straddle pages -- is a short gather list of ranges.  The byte RULES (what counts as sync, what is
// skipped as junk, which frames are tags, how packets continue across pages, where the time stamps and trims come
// from) are the reference's, cited at each function, and are checked bit for bit against oracle/packetizer_oracle.py.
//
// Header-only C++17, no dependencies.  The MPEG, ADTS and FLAC rules are also device functions when the header is compiled by nvcc
// (SYMGPU_PACKET_HD), so the Layer I / II device decoder and the device MPEG, ADTS and FLAC indexes parse headers and tags with
// this very code; C++ compilers see plain inline functions.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <map>
#include <utility>
#include <vector>

#if defined(__CUDACC__)
#define SYMGPU_PACKET_HD __host__ __device__
#else
#define SYMGPU_PACKET_HD
#endif

namespace symgpu {
namespace packet {

enum class Status : uint8_t {
    Ok = 0,
    EndOfStream,  // the bytes ran out (the reference: IoError UnexpectedEof)
    DecodeError,  // malformed stream (Error::DecodeError)
    Unsupported,  // well-formed but not handled by the reference either (Error::Unsupported)
};

// A byte range of the source buffer.
struct Piece {
    uint64_t offset;
    uint32_t len;
};

namespace detail {
SYMGPU_PACKET_HD inline uint32_t be32(const uint8_t* p) { return uint32_t(p[0]) << 24 | uint32_t(p[1]) << 16 | uint32_t(p[2]) << 8 | p[3]; }
SYMGPU_PACKET_HD inline uint32_t be24(const uint8_t* p) { return uint32_t(p[0]) << 16 | uint32_t(p[1]) << 8 | p[2]; }
SYMGPU_PACKET_HD inline uint32_t be16(const uint8_t* p) { return uint32_t(p[0]) << 8 | p[1]; }
SYMGPU_PACKET_HD inline uint32_t le32(const uint8_t* p) { return uint32_t(p[3]) << 24 | uint32_t(p[2]) << 16 | uint32_t(p[1]) << 8 | p[0]; }
SYMGPU_PACKET_HD inline uint64_t le64(const uint8_t* p) { return uint64_t(le32(p + 4)) << 32 | le32(p); }

struct Crc32Table {  // slicing-by-8: t[k][b] = contribution of byte b seen k bytes before the end of an 8-byte block
    uint32_t t[8][256];
    constexpr Crc32Table() : t() {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i << 24;
            for (int k = 0; k < 8; ++k) c = (c & 0x80000000u) ? (c << 1) ^ 0x04c11db7u : c << 1;
            t[0][i] = c;
        }
        for (int k = 1; k < 8; ++k)
            for (uint32_t i = 0; i < 256; ++i) t[k][i] = (t[k - 1][i] << 8) ^ t[0][t[k - 1][i] >> 24];
    }
};
struct Crc16Table {
    uint16_t t[256];
    constexpr Crc16Table() : t() {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xa001u : c >> 1;
            t[i] = uint16_t(c);
        }
    }
};
// Four-character codes as the big-endian words be32 reads.
constexpr uint32_t tag4(const char (&s)[5]) { return uint32_t(uint8_t(s[0])) << 24 | uint32_t(uint8_t(s[1])) << 16 | uint32_t(uint8_t(s[2])) << 8 | uint8_t(s[3]); }
constexpr uint32_t kXing = tag4("Xing"), kInfo = tag4("Info"), kVbri = tag4("VBRI"), kLame = tag4("LAME"), kLavf = tag4("Lavf"), kLavc = tag4("Lavc");
// The first candidate of vpos[lo .. n) (ascending) at or after target; n when there is none.
SYMGPU_PACKET_HD inline uint32_t first_at_or_after(const uint64_t* vpos, uint32_t lo, uint32_t n, uint64_t target) {
    uint32_t hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (vpos[mid] < target) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
}  // namespace detail

// CRC-32, polynomial 0x04c11db7, most-significant bit first, no final xor; the caller supplies the initial state
// (Ogg pages: 0).  symphonia-core/src/checksum/crc32.rs:543-570.
// `t` is a slicing-by-8 table (detail::Crc32Table::t): the device keeps its copy in shared memory.
SYMGPU_PACKET_HD inline uint32_t crc32_update_with(const uint32_t (*t)[256], uint32_t state, const uint8_t* p, size_t n) {
    for (; n >= 8; p += 8, n -= 8) {
        const uint32_t hi = state ^ detail::be32(p), lo = detail::be32(p + 4);
        state = t[7][hi >> 24] ^ t[6][(hi >> 16) & 0xff] ^ t[5][(hi >> 8) & 0xff] ^ t[4][hi & 0xff] ^
                t[3][lo >> 24] ^ t[2][(lo >> 16) & 0xff] ^ t[1][(lo >> 8) & 0xff] ^ t[0][lo & 0xff];
    }
    for (size_t i = 0; i < n; ++i) state = (state << 8) ^ t[0][(state >> 24) ^ p[i]];
    return state;
}
inline uint32_t crc32_update(uint32_t state, const uint8_t* p, size_t n) {
    static constexpr detail::Crc32Table tab{};
    return crc32_update_with(tab.t, state, p, n);
}

// CRC-16, polynomial 0x8005, least-significant bit first, no final xor (the LAME tag's checksum).
// symphonia-core/src/checksum/crc16.rs:377-404.  `t` is detail::Crc16Table::t: the device keeps its copy in constant memory.
SYMGPU_PACKET_HD inline uint16_t crc16_ansi_le_update_with(const uint16_t* t, uint16_t state, const uint8_t* p, size_t n) {
    for (size_t i = 0; i < n; ++i) state = uint16_t((state >> 8) ^ t[(state ^ p[i]) & 0xff]);
    return state;
}
inline const uint16_t* crc16_ansi_le_table() {
    static constexpr detail::Crc16Table tab{};
    return tab.t;
}
inline uint16_t crc16_ansi_le_update(uint16_t state, const uint8_t* p, size_t n) { return crc16_ansi_le_update_with(crc16_ansi_le_table(), state, p, n); }

// =====================================================================================================================
// MPEG audio (Layers I-III)
// =====================================================================================================================

enum class MpaVersion : uint8_t { Mpeg1 = 0, Mpeg2 = 1, Mpeg2p5 = 2 };
enum class MpaMode : uint8_t { Stereo = 0, JointStereo = 1, DualMono = 2, Mono = 3 };

// The 32-bit frame header, decoded.  symphonia-bundle-mp3/src/header.rs:107-233, common.rs:155-212.
struct MpaHeader {
    MpaVersion version;
    uint8_t layer;            // 1, 2 or 3
    MpaMode mode;
    uint8_t sample_rate_idx;  // 0..8: 44.1 / 48 / 32 kHz, then the halved and quartered rates (the reference's table index)
    bool mid_side;            // Layer III joint stereo
    bool intensity;           // Layer III joint stereo
    uint8_t bound;            // Layers I / II joint stereo: first sub-band coded in intensity stereo, else 32
    uint8_t emphasis;         // 0 none, 1 50/15 us, 3 CCITT J.17
    bool copyrighted, original, padding, crc;
    uint32_t bitrate;         // bit/s
    uint32_t sample_rate;     // Hz
    uint32_t frame_size;      // bytes AFTER the 4-byte header word

    SYMGPU_PACKET_HD int n_channels() const { return mode == MpaMode::Mono ? 1 : 2; }
    SYMGPU_PACKET_HD int n_granules() const { return version == MpaVersion::Mpeg1 ? 2 : 1; }
    SYMGPU_PACKET_HD uint32_t samples_per_frame() const { return layer == 1 ? 384u : layer == 2 ? 1152u : 576u * uint32_t(n_granules()); }
    SYMGPU_PACKET_HD uint32_t header_size() const { return 4u + (crc ? 2u : 0u); }
    SYMGPU_PACKET_HD uint32_t side_info_len() const {
        const bool mono = mode == MpaMode::Mono;
        return version == MpaVersion::Mpeg1 ? (mono ? 17u : 32u) : (mono ? 9u : 17u);
    }
};

// header.rs:71-75: eleven set bits.
SYMGPU_PACKET_HD inline bool mpa_is_synced(uint32_t w) { return (w & 0xffe00000u) == 0xffe00000u; }

// header.rs:49-69: the cheap plausibility test applied while hunting for sync.
SYMGPU_PACKET_HD inline bool mpa_check_header(uint32_t w) {
    return ((w >> 19) & 3) != 1 && ((w >> 17) & 3) != 0 && ((w >> 12) & 15) != 15 && ((w >> 10) & 3) != 3;
}

SYMGPU_PACKET_HD inline Status mpa_parse_header(uint32_t w, MpaHeader& h) {
    static constexpr uint16_t kbps[5][15] = {
        {0, 32, 64, 96, 128, 160, 192, 224, 256, 288, 320, 352, 384, 416, 448},  // MPEG-1 Layer I
        {0, 32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384},     // MPEG-1 Layer II
        {0, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320},      // MPEG-1 Layer III
        {0, 32, 48, 56, 64, 80, 96, 112, 128, 144, 160, 176, 192, 224, 256},     // MPEG-2 / 2.5 Layer I
        {0, 8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160},          // MPEG-2 / 2.5 Layers II, III
    };
    static constexpr uint32_t rates[3] = {44100, 48000, 32000};
    const uint32_t v = (w >> 19) & 3, l = (w >> 17) & 3, bi = (w >> 12) & 15, ri = (w >> 10) & 3, m = (w >> 6) & 3;
    if (v == 1 || l == 0) return Status::DecodeError;
    h.version = v == 3 ? MpaVersion::Mpeg1 : v == 2 ? MpaVersion::Mpeg2 : MpaVersion::Mpeg2p5;
    h.layer = uint8_t(4 - l);
    if (bi == 0) return Status::Unsupported;  // free format
    if (bi == 15) return Status::DecodeError;
    const int row = h.version == MpaVersion::Mpeg1 ? h.layer - 1 : (h.layer == 1 ? 3 : 4);
    h.bitrate = uint32_t(kbps[row][bi]) * 1000u;
    if (ri == 3) return Status::DecodeError;
    const int shift = int(h.version);  // 0, 1, 2: full, half, quarter rate
    h.sample_rate = rates[ri] >> shift;
    h.sample_rate_idx = uint8_t(ri + 3 * shift);
    h.mode = MpaMode(m == 0 ? 0 : m == 1 ? 1 : m == 2 ? 2 : 3);
    h.mid_side = h.intensity = false;
    h.bound = 32;
    if (h.mode == MpaMode::JointStereo) {
        if (h.layer == 3) {
            h.mid_side = (w & 0x20) != 0;
            h.intensity = (w & 0x10) != 0;
        } else {
            h.bound = uint8_t((1 + ((w >> 4) & 3)) << 2);
        }
    }
    if (h.layer == 2) {  // header.rs:176-187: combinations Layer II forbids
        const uint32_t k = h.bitrate / 1000;
        if (h.mode == MpaMode::Mono ? (k == 224 || k == 256 || k == 320 || k == 384) : (k == 32 || k == 48 || k == 56 || k == 80))
            return Status::DecodeError;
    }
    const uint32_t e = w & 3;
    h.emphasis = uint8_t(e == 1 ? 1 : e == 3 ? 3 : 0);
    h.copyrighted = (w & 8) != 0;
    h.original = (w & 4) != 0;
    h.padding = (w & 0x200) != 0;
    h.crc = (w & 0x10000) == 0;
    const uint32_t factor = h.layer == 1 ? 12u : (h.layer == 3 && h.version != MpaVersion::Mpeg1) ? 72u : 144u;
    const uint32_t slots = factor * h.bitrate / h.sample_rate + (h.padding ? 1u : 0u);
    h.frame_size = slots * (h.layer == 1 ? 4u : 1u) - 4u;
    return Status::Ok;
}

// Longest frame the format can express, header included (header.rs:17).
constexpr uint32_t kMpaMaxFrameSize = 2881;

struct MpaLameInfo {
    char encoder[9];
    uint32_t delay, padding;  // samples the decoder output starts / ends with that are not audio
    uint32_t peak;            // raw 9.23 fixed-point replay-gain peak, 0 = absent
};

// Xing / Info tag of a Layer III frame (demuxer.rs:761-925).
struct MpaInfoTag {
    bool has_num_frames, has_num_bytes, has_toc, has_quality, is_cbr, has_lame;
    uint32_t num_frames, num_bytes, quality;
    MpaLameInfo lame;
};
struct MpaVbriTag {
    uint32_t num_bytes, num_mpeg_frames;
};

// demuxer.rs:942-968.  `f` = the whole frame, header word first.
SYMGPU_PACKET_HD inline bool mpa_is_maybe_info_tag(const uint8_t* f, size_t n, const MpaHeader& h) {
    if (h.layer != 3) return false;
    const size_t at = 4 + h.side_info_len();
    if (n < at + 8) return false;
    const uint32_t id = detail::be32(f + at);
    if (id != detail::kXing && id != detail::kInfo) return false;
    for (size_t i = h.header_size(); i < at; ++i)
        if (f[i]) return false;
    return true;
}

// True when the frame is a tag the reference would act on; false for everything else, INCLUDING a tag whose
// flagged fields do not fit the frame (the reference flattens that read error to "no tag").  crc16: crc16_ansi_le_table().
SYMGPU_PACKET_HD inline bool mpa_read_info_tag_with(const uint16_t* crc16, const uint8_t* f, size_t n, const MpaHeader& h, MpaInfoTag& t) {
    if (!mpa_is_maybe_info_tag(f, n, h)) return false;
    const size_t base = 4 + h.side_info_len();
    size_t at = base;
    t = MpaInfoTag{};
    t.is_cbr = detail::be32(f + at) == detail::kInfo;
    const uint32_t flags = detail::be32(f + at + 4);
    at += 8;
    if (flags & 1) {
        if (at + 4 > n) return false;
        t.has_num_frames = true, t.num_frames = detail::be32(f + at), at += 4;
    }
    if (flags & 2) {
        if (at + 4 > n) return false;
        t.has_num_bytes = true, t.num_bytes = detail::be32(f + at), at += 4;
    }
    if (flags & 4) {
        if (at + 100 > n) return false;
        t.has_toc = true, at += 100;
    }
    if (flags & 8) {
        if (at + 4 > n) return false;
        t.has_quality = true, t.quality = detail::be32(f + at), at += 4;
    }
    // LAME extension: 24 bytes up to the delay / padding field, 12 more up to its CRC-16 (over everything before it).
    if (n - at >= 24) {
        const uint8_t* e = f + at;
        MpaLameInfo li{};
        for (int i = 0; i < 9; ++i) li.encoder[i] = char(e[i]);
        li.peak = detail::be32(e + 11);
        const uint32_t trim = detail::be24(e + 21);
        const uint32_t id = detail::be32(e);
        const bool lame = id == detail::kLame, known = lame || id == detail::kLavf || id == detail::kLavc;
        if (known) {
            li.delay = 528 + 1 + (trim >> 12);
            const uint32_t pad = trim & 0xfff;
            li.padding = pad > 529 ? pad - 529 : 0;
        }
        at += 24;
        bool ok = true;
        if (n - at >= 12) {
            at += 10;
            if (h.crc || lame) {
                const uint32_t written = detail::be16(f + at);
                ok = written == 0 || written == crc16_ansi_le_update_with(crc16, 0, f, at);
            }
        }
        if (ok) t.has_lame = true, t.lame = li;
    }
    return true;
}
inline bool mpa_read_info_tag(const uint8_t* f, size_t n, const MpaHeader& h, MpaInfoTag& t) {
    return mpa_read_info_tag_with(crc16_ansi_le_table(), f, n, h, t);
}

// demuxer.rs:1023-1047, 980-1019.
SYMGPU_PACKET_HD inline bool mpa_is_maybe_vbri_tag(const uint8_t* f, size_t n, const MpaHeader& h) {
    if (h.layer != 3 || n < 36 + 26 || detail::be32(f + 36) != detail::kVbri) return false;
    for (size_t i = h.header_size(); i < 36; ++i)
        if (f[i]) return false;
    return true;
}
SYMGPU_PACKET_HD inline bool mpa_read_vbri_tag(const uint8_t* f, size_t n, const MpaHeader& h, MpaVbriTag& t) {
    if (!mpa_is_maybe_vbri_tag(f, n, h) || detail::be16(f + 40) != 1) return false;
    t.num_bytes = detail::be32(f + 46);
    t.num_mpeg_frames = detail::be32(f + 50);
    return true;
}

// main_data_begin of a Layer III frame: how many bytes of THIS frame's main data live in earlier frames
// (demuxer.rs:664-680).  The bit-reservoir front end needs it per frame; -1 when the frame is too short.
SYMGPU_PACKET_HD inline int mpa_main_data_begin(const uint8_t* f, size_t n, const MpaHeader& h) {
    const size_t at = h.header_size();
    if (h.version == MpaVersion::Mpeg1) return at + 2 <= n ? int(detail::be16(f + at) >> 7) : -1;
    return at + 1 <= n ? int(f[at]) : -1;
}

// demuxer.rs:186-200: a frame next() drops wherever it turns up -- a Xing / Info tag when it looks like one and reads as one,
// else a VBRI tag that reads as one.
SYMGPU_PACKET_HD inline bool mpa_drops_tag(const uint16_t* crc16, const uint8_t* f, size_t n, const MpaHeader& h) {
    MpaInfoTag info;
    MpaVbriTag vbri;
    return mpa_is_maybe_info_tag(f, n, h) ? mpa_read_info_tag_with(crc16, f, n, h, info) : mpa_read_vbri_tag(f, n, h, vbri);
}

// demuxer.rs:620-627: the word behind a first-frame candidate h looks like the same kind of stream.
SYMGPU_PACKET_HD inline bool mpa_similar(uint32_t next, const MpaHeader& h) {
    MpaHeader c;
    return mpa_is_synced(next) && mpa_parse_header(next, c) == Status::Ok && c.version == h.version && c.layer == h.layer &&
           c.sample_rate == h.sample_rate && c.n_channels() == h.n_channels();
}

namespace detail {
// m x 2^e = n / d rounded to nearest, ties to even, with 2^52 <= m < 2^53: an IEEE double division of positive values, in integers.
SYMGPU_PACKET_HD inline uint64_t div_rn53(unsigned __int128 n, unsigned __int128 d, int& e) {
    auto bits = [](unsigned __int128 v) {
        int b = 0;
        for (; v; v >>= 1) ++b;
        return b;
    };
    for (int sh = 52 - (bits(n) - bits(d));; ++sh) {
        const unsigned __int128 num = sh >= 0 ? n << sh : n, den = sh >= 0 ? d : d << -sh;
        uint64_t m = uint64_t(num / den);
        if (m < (uint64_t(1) << 52)) continue;
        const unsigned __int128 r2 = (num % den) * 2;
        if (r2 > den || (r2 == den && (m & 1))) ++m;
        e = -sh;
        if (m == uint64_t(1) << 53) m >>= 1, ++e;
        return m;
    }
}
}  // namespace detail

// uint64_t(double(total) / (double(len) / double(count))) for 0 < count <= len < 2^32 and total < 2^33, computed in integers: both
// divisions correctly rounded as IEEE doubles, the quotient truncated.  The device gets the same bits without double arithmetic.
SYMGPU_PACKET_HD inline uint64_t mpa_extrapolate(uint64_t total, uint64_t len, uint64_t count) {
    if (total == 0) return 0;
    int ex, ey;
    const uint64_t mx = detail::div_rn53(len, count, ex);                                   // len / count = mx x 2^ex
    const uint64_t my = ex <= 0 ? detail::div_rn53((unsigned __int128)(total) << -ex, mx, ey)  // total / (mx x 2^ex)
                                : detail::div_rn53(total, (unsigned __int128)(mx) << ex, ey);
    return ey >= 0 ? my << ey : ey <= -64 ? 0 : my >> -ey;
}

// demuxer.rs:683-733: average the first frames of d[from ..][.. n) (more than 16 of them or more than 16 KiB) and extrapolate.
// At most 17 frames are read.
SYMGPU_PACKET_HD inline bool mpa_estimate_frames(const uint8_t* d, size_t n, size_t from, uint64_t& frames) {
    size_t q = from, len = 0;
    unsigned count = 0;
    for (;;) {
        MpaHeader h;
        if (q + 4 > n || mpa_parse_header(detail::be32(d + q), h) != Status::Ok) return false;
        len += 4 + h.frame_size, ++count;
        if (q + 4 + h.frame_size > n) return false;
        q += 4 + h.frame_size;
        if (count > 16 || len > 16 * 1024) break;
    }
    frames = mpa_extrapolate(n - from, len, count);
    return true;
}

// One packet = one frame, a byte range of the source.
struct MpaPacket {
    uint64_t offset;      // of the header word
    uint32_t size;        // header word included
    uint32_t header;      // the header word
    int64_t pts;          // in samples; starts at -delay
    uint32_t dur;         // samples the frame decodes to
    uint32_t trim_start;  // leading samples to drop (encoder delay)
    uint64_t trim_end;    // trailing samples to drop; NOT capped to dur, as in the reference (packet.rs:334-338)
};

struct MpaTrack {
    MpaHeader first;           // codec parameters come from the first frame
    uint32_t first_word;
    bool has_delay, has_num_frames;
    uint32_t delay, padding;
    uint64_t num_frames;       // samples of audio, delay and padding removed (exact, from a tag) or estimated
    enum Tag : uint8_t { None, Xing, Info, Vbri } tag;
    uint64_t first_packet_pos;
};

// demuxer.rs:445-487: what open() learns from the accepted first frame at d[at ..] of a buffer of n bytes.  A frame that reads
// as a Xing / Info or VBRI tag is no packet (first_packet_pos lies behind it); for any other, a seekable stream gets the estimate.
SYMGPU_PACKET_HD inline void mpa_open_track(const uint16_t* crc16, const uint8_t* d, size_t n, size_t at, bool seekable, MpaTrack& t) {
    const uint32_t w = detail::be32(d + at);
    MpaHeader h{};
    mpa_parse_header(w, h);
    const size_t size = 4 + size_t(h.frame_size);
    t = MpaTrack{};
    t.first = h;
    t.first_word = w;
    t.tag = MpaTrack::None;
    t.first_packet_pos = at + size;
    MpaInfoTag info;
    MpaVbriTag vbri;
    if (mpa_read_info_tag_with(crc16, d + at, size, h, info)) {
        t.tag = info.is_cbr ? MpaTrack::Info : MpaTrack::Xing;
        if (info.has_lame) t.has_delay = true, t.delay = info.lame.delay, t.padding = info.lame.padding;
        if (info.has_num_frames) {
            const uint64_t total = uint64_t(info.num_frames) * h.samples_per_frame();
            const uint64_t cut = uint64_t(t.delay) + t.padding;
            t.has_num_frames = true, t.num_frames = total > cut ? total - cut : 0;
        }
    } else if (mpa_read_vbri_tag(d + at, size, h, vbri)) {
        t.tag = MpaTrack::Vbri;
        t.has_num_frames = true, t.num_frames = uint64_t(vbri.num_mpeg_frames) * h.samples_per_frame();
    } else {
        t.first_packet_pos = at;  // an ordinary frame: it is the first packet
        uint64_t frames;
        if (seekable && mpa_estimate_frames(d, n, at, frames)) t.has_num_frames = true, t.num_frames = frames * h.samples_per_frame();
    }
}

// demuxer.rs:201-218: the packet of a kept frame with header word w at `at`, ts = the samples of the packets before it - delay.
SYMGPU_PACKET_HD inline MpaPacket mpa_frame_packet(uint32_t w, uint64_t at, int64_t ts, const MpaTrack& t) {
    MpaHeader h{};
    mpa_parse_header(w, h);
    const uint32_t dur = h.samples_per_frame();
    MpaPacket p;
    p.offset = at, p.size = 4 + h.frame_size, p.header = w, p.pts = ts, p.dur = dur;
    p.trim_start = ts < 0 ? uint32_t(-ts < int64_t(dur) ? -ts : int64_t(dur)) : 0u;
    p.trim_end = 0;
    if (t.has_num_frames) {
        const int64_t over = ts + int64_t(dur) - int64_t(t.num_frames);
        if (over > 0) p.trim_end = uint64_t(over);
    }
    return p;
}

// ---- the frame search, step by step: shared by MpaIndexer and the device index (symgpu_mpa_index_dev) ------------------------
// 1. A candidate: where the frame search stops to look at a word -- the sync bits and the plausibility test (header.rs:77-103).
//    Candidates may be adjacent (FF FF E...), so a buffer of n bytes holds at most n - 3.
SYMGPU_PACKET_HD inline bool mpa_is_candidate(const uint8_t* d, size_t n, size_t q) {
    if (q + 4 > n || d[q] != 0xff) return false;
    const uint32_t w = detail::be32(d + q);
    return mpa_is_synced(w) && mpa_check_header(w);
}

// 2. A candidate's node word, what the search does there.  Bits 0-1, the kind: a Skip (the full parse fails: the search goes on
//    4 bytes later), a Stop (the frame runs past the buffer: the search ends) or a Frame.  Bits 3 on: a Frame's size, header
//    word included.
enum : uint32_t { kMpaSkip = 0, kMpaStop = 1, kMpaFrame = 2 };
constexpr uint32_t kMpaEnd = 0xffffffffu;  // no such candidate
SYMGPU_PACKET_HD inline uint32_t mpa_node(const uint8_t* d, size_t n, size_t q) {
    MpaHeader h;
    if (mpa_parse_header(detail::be32(d + q), h) != Status::Ok) return kMpaSkip;
    const size_t size = 4 + size_t(h.frame_size);
    return q + size > n ? kMpaStop : uint32_t(size) << 3 | kMpaFrame;
}
SYMGPU_PACKET_HD inline uint32_t mpa_node_kind(uint32_t node) { return node & 3; }
SYMGPU_PACKET_HD inline uint32_t mpa_node_size(uint32_t node) { return node >> 3; }

// The smallest frame a header can express, header word included (MPEG-2 Layer III, 8 kbit/s, 24 kHz: 72 x 8000 / 24000).  A
// file's frames do not overlap, so a buffer of n bytes holds at most n / kMpaMinFrameSize packets.
constexpr uint32_t kMpaMinFrameSize = 24;

// 3. open() rejects a Frame as the first frame when the word behind it exists but does not look like the same stream
//    (demuxer.rs:610-640); the hunt then restarts one byte on.
SYMGPU_PACKET_HD inline bool mpa_first_rejected(const uint8_t* d, size_t n, size_t q, uint32_t node) {
    if (mpa_node_kind(node) != kMpaFrame) return false;
    const size_t size = mpa_node_size(node);
    MpaHeader h;
    mpa_parse_header(detail::be32(d + q), h);
    return q + size + 4 <= n && !mpa_similar(detail::be32(d + q + size), h);
}

// The candidates of the files of a device call lie in one virtual byte space, named by their index in ascending virtual position
// (vpos); file_end is the virtual end of candidate c's file.
// 4. S(c), the packet successor: the candidate the search visits after c -- for a Frame the first at or after its end, for a
//    Skip the first at or after c + 4; none (kMpaEnd) for a Stop or when that lies past the file.
SYMGPU_PACKET_HD inline uint32_t mpa_successor(const uint64_t* vpos, uint32_t n_cand, uint32_t c, uint32_t node, uint64_t file_end) {
    const uint32_t kind = mpa_node_kind(node);
    if (kind == kMpaStop) return kMpaEnd;
    const uint32_t s = detail::first_at_or_after(vpos, c + 1, n_cand, vpos[c] + (kind == kMpaFrame ? mpa_node_size(node) : 4));
    return s < n_cand && vpos[s] < file_end ? s : kMpaEnd;
}

// 5. G(c), the first-frame hunt: S(c) for a Skip, c + 1 (when in the file) for a rejected Frame, and c itself for a root -- a
//    Stop or an accepted Frame.  The file's first frame is the root G leads to from its first candidate, when that is a Frame.
SYMGPU_PACKET_HD inline uint32_t mpa_hunt(const uint64_t* vpos, uint32_t n_cand, uint32_t c, uint32_t node, bool rejected, uint32_t succ,
                                          uint64_t file_end) {
    if (mpa_node_kind(node) == kMpaSkip) return succ;
    if (!rejected) return c;
    return c + 1 < n_cand && vpos[c + 1] < file_end ? c + 1 : kMpaEnd;
}

// 6. Jumping round at c: next = G o G.  After k rounds hunt[c] = G^(2^k)(c); roots are fixed points, kMpaEnd absorbs.
SYMGPU_PACKET_HD inline void mpa_hunt_jump(const uint32_t* hunt, uint32_t* next, uint32_t c) {
    const uint32_t g = hunt[c];
    next[c] = g == kMpaEnd ? kMpaEnd : hunt[g];
}

// The jumping rounds that bring every hunt of files of at most max_len bytes to its end: G rises by at least one candidate a step.
SYMGPU_PACKET_HD inline uint32_t mpa_hunt_rounds(uint64_t max_len) {
    uint32_t k = 0;
    for (uint64_t m = max_len; m; m >>= 1) ++k;
    return k;
}

// 7. The packets are the Frames on the S-chain from the first frame, ranked from it by adts_double over S; S moves at least 4
//    bytes, so a chain has at most max_len / 4 nodes and these rounds rank them all.
SYMGPU_PACKET_HD inline uint32_t mpa_chain_rounds(uint64_t max_len) { return mpa_hunt_rounds(max_len / 4); }

// 8. The samples of the packet candidate c at d[q ..] of a file of n bytes gives, 0 when it gives none: c must be a chain Frame
//    (rank: its rank on the chain, kAdtsUnranked off it) that next() keeps; the first frame (rank 0) is left out when open() read
//    it as a tag (first_tag).
SYMGPU_PACKET_HD inline uint32_t mpa_packet_dur(const uint16_t* crc16, const uint8_t* d, size_t q, uint32_t node, uint32_t rank, uint8_t first_tag) {
    if (rank == 0xffffffffu /* kAdtsUnranked */ || mpa_node_kind(node) != kMpaFrame) return 0;
    MpaHeader h;
    mpa_parse_header(detail::be32(d + q), h);
    if (rank == 0 ? first_tag != MpaTrack::None : mpa_drops_tag(crc16, d + q, mpa_node_size(node), h)) return 0;
    return h.samples_per_frame();
}

// The reference's MpaReader over a resident buffer: open() = try_new, next() = next_packet.
class MpaIndexer {
  public:
    MpaIndexer(const uint8_t* data, size_t n) : d_(data), n_(n) {}

    // demuxer.rs:414-487.  EndOfStream: the buffer holds no frame.  `seekable` = the reference's is_seekable():
    // without it no duration is estimated for an untagged stream and nothing is trimmed from its end.
    Status open(bool seekable = true) {
        size_t at = 0;
        uint32_t node;
        // demuxer.rs:610-640: accept a first frame only when the next word looks like the same kind of stream;
        // rejected candidates restart the hunt one byte further.
        for (size_t from = 0;;) {
            if (!find_frame(from, at, node)) return Status::EndOfStream;
            if (!mpa_first_rejected(d_, n_, at, node)) break;
            from = at + 1;
        }
        mpa_open_track(crc16_ansi_le_table(), d_, n_, at, seekable, track_);
        pos_ = track_.first_packet_pos;
        ts_ = -int64_t(track_.delay);
        open_ = true;
        return Status::Ok;
    }

    const MpaTrack& track() const { return track_; }

    // demuxer.rs:160-218.  Frames that are Xing / Info / VBRI tags are dropped wherever they turn up.
    Status next(MpaPacket& p) {
        if (!open_) return Status::DecodeError;
        for (;;) {
            size_t at;
            uint32_t node;
            if (!find_frame(pos_, at, node)) return Status::EndOfStream;
            const size_t size = mpa_node_size(node);
            pos_ = at + size;
            const uint32_t w = detail::be32(d_ + at);
            MpaHeader h;
            mpa_parse_header(w, h);
            if (mpa_drops_tag(crc16_ansi_le_table(), d_ + at, size, h)) continue;
            p = mpa_frame_packet(w, at, ts_, track_);
            ts_ += p.dur;
            return Status::Ok;
        }
    }

    // Everything at once.
    static Status index(const uint8_t* data, size_t n, MpaTrack& track, std::vector<MpaPacket>& out, bool seekable = true) {
        MpaIndexer ix(data, n);
        const Status s = ix.open(seekable);
        if (s != Status::Ok) return s;
        track = ix.track();
        MpaPacket p;
        while (ix.next(p) == Status::Ok) out.push_back(p);
        return Status::Ok;
    }

  private:
    // header.rs:77-103 + demuxer.rs:585-607 as a window search: the first candidate at or after `from`; a Skip costs its 4
    // bytes, a Stop ends the stream, a Frame is returned with its node word.
    bool find_frame(size_t from, size_t& at, uint32_t& node) const {
        for (size_t q = from; q + 4 <= n_;) {
            // cheap reject on the first byte keeps the scan at memchr speed through payload bytes
            if (d_[q] != 0xff) {
                const void* hit = std::memchr(d_ + q, 0xff, n_ - q);
                if (!hit) return false;
                q = size_t(static_cast<const uint8_t*>(hit) - d_);
                if (q + 4 > n_) return false;
            }
            if (!mpa_is_candidate(d_, n_, q)) {
                ++q;
                continue;
            }
            node = mpa_node(d_, n_, q);
            if (mpa_node_kind(node) == kMpaSkip) {
                q += 4;
                continue;
            }
            if (mpa_node_kind(node) == kMpaStop) return false;
            at = q;
            return true;
        }
        return false;
    }

    const uint8_t* d_;
    size_t n_;
    size_t pos_ = 0;
    int64_t ts_ = 0;
    bool open_ = false;
    MpaTrack track_{};
};

// =====================================================================================================================
// ADTS (AAC)
// =====================================================================================================================

struct AdtsHeader {
    uint8_t profile;       // MPEG-4 audio object type: 1 Main, 2 LC, 3 SSR, 4 LTP
    uint8_t channels;      // 0: configured in-band (program config element)
    uint8_t header_len;    // 7, or 9 with a CRC
    bool has_crc;
    uint16_t crc;
    uint16_t frame_len;    // sync word, header and payload
    uint32_t sample_rate;
    SYMGPU_PACKET_HD uint32_t payload_len() const { return uint32_t(frame_len) - header_len; }
};

// adts.rs:202-204: 0xfff, layer bits zero; the MPEG-2/4 bit and the protection bit are free.
SYMGPU_PACKET_HD inline bool adts_is_sync(uint32_t w16) { return (w16 & 0xfff6u) == 0xfff0u; }

// adts.rs:137-198.  `p` points at the sync word; `n` bytes are readable.  EndOfStream: fewer than header_len bytes.
SYMGPU_PACKET_HD inline Status adts_parse_header(const uint8_t* p, size_t n, AdtsHeader& h) {
    static constexpr uint32_t rates[13] = {96000, 88200, 64000, 48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025, 8000, 7350};
    static constexpr uint8_t chans[8] = {0, 1, 2, 3, 4, 5, 6, 8};
    if (n < 2) return Status::EndOfStream;
    h.has_crc = (p[1] & 1) == 0;
    h.header_len = h.has_crc ? 9 : 7;
    if (n < h.header_len) return Status::EndOfStream;
    h.profile = uint8_t((p[2] >> 6) + 1);
    const uint32_t ri = (p[2] >> 2) & 15;
    if (ri > 12) return Status::DecodeError;  // 15 is the escape ADTS forbids, 13 / 14 are reserved
    h.sample_rate = rates[ri];
    h.channels = chans[((p[2] & 1) << 2) | (p[3] >> 6)];
    h.frame_len = uint16_t(((p[3] & 3) << 11) | (p[4] << 3) | (p[5] >> 5));
    if (h.frame_len < h.header_len) return Status::DecodeError;
    if ((p[6] & 3) != 0) return Status::Unsupported;  // more than one raw data block per frame
    h.crc = h.has_crc ? uint16_t(detail::be16(p + 7)) : 0;
    return Status::Ok;
}

struct AdtsPacket {
    uint64_t offset;  // of the PAYLOAD (the raw data block), as the reference's packets carry no ADTS header
    uint32_t size;
    int64_t pts;      // 1024 samples per packet
    uint32_t sample_rate;
    uint8_t channels, profile;
};

// adts.rs:278-309 over a resident buffer.
class AdtsIndexer {
  public:
    AdtsIndexer(const uint8_t* data, size_t n) : d_(data), n_(n) {}

    // EndOfStream at the end of the bytes (truncated() tells a clean end from a cut payload); DecodeError /
    // Unsupported leave the cursor behind the offending header, as the reference's reader does, so that a caller
    // that chooses to carry on resynchronises from there.
    Status next(AdtsPacket& p) {
        size_t q = pos_;
        for (;; ++q) {
            if (q + 2 > n_) return pos_ = n_, Status::EndOfStream;
            if (d_[q] != 0xff) {
                const void* hit = std::memchr(d_ + q, 0xff, n_ - q);
                if (!hit) return pos_ = n_, Status::EndOfStream;
                q = size_t(static_cast<const uint8_t*>(hit) - d_);
                if (q + 2 > n_) return pos_ = n_, Status::EndOfStream;
            }
            if (adts_is_sync(detail::be16(d_ + q))) break;
        }
        AdtsHeader h;
        const Status s = adts_parse_header(d_ + q, n_ - q, h);
        if (s == Status::EndOfStream) return pos_ = n_, s;
        pos_ = q + h.header_len;
        if (s != Status::Ok) return s;
        if (pos_ + h.payload_len() > n_) return truncated_ = true, pos_ = n_, Status::EndOfStream;
        p.offset = pos_, p.size = h.payload_len(), p.pts = ts_, p.sample_rate = h.sample_rate, p.channels = h.channels, p.profile = h.profile;
        pos_ += h.payload_len();
        ts_ += 1024;
        return Status::Ok;
    }
    bool truncated() const { return truncated_; }

    // Up to the first non-Ok status, which is returned.
    static Status index(const uint8_t* data, size_t n, std::vector<AdtsPacket>& out, bool* truncated = nullptr) {
        AdtsIndexer ix(data, n);
        AdtsPacket p;
        Status s;
        while ((s = ix.next(p)) == Status::Ok) out.push_back(p);
        if (truncated) *truncated = ix.truncated();
        return s;
    }

  private:
    const uint8_t* d_;
    size_t n_;
    size_t pos_ = 0;
    int64_t ts_ = 0;
    bool truncated_ = false;
};

// ---- the schedule of the device index (symgpu_adts_index_dev), step by step over the files of a call ----------------------------
// The files lie back to back, in call order, in one virtual byte space, so the candidates of every file sorted by virtual
// position are each file's candidates in turn.  A candidate is named by its 32-bit index in that order.
//
// 1. A candidate: a place where AdtsIndexer::next ends its search for sync.  Its second byte is never 0xff, so two candidates are
//    never adjacent and a file of n bytes holds at most n / 2.
SYMGPU_PACKET_HD inline bool adts_is_candidate(const uint8_t* d, size_t n, size_t q) {
    return q + 2 <= n && d[q] == 0xff && adts_is_sync(detail::be16(d + q));
}

// 2. A candidate's node word, what AdtsIndexer::next does there.  Bits 0-2, the kind: a Frame, whose payload lies in the file, or a
//    Stop, numbered as the stop symgpu_adts_index reports (0 a cut header, a clean end; 1 / 2 a bad header, decode error /
//    unsupported; 3 a payload past the file's end).  Bit 3 (kAdtsLast): set in step 3 when the node has no successor.  Bits 4-16:
//    a Frame's frame length.
enum : uint32_t { kAdtsStopOk = 0, kAdtsStopDecode = 1, kAdtsStopUnsupported = 2, kAdtsStopLimit = 3, kAdtsFrame = 4, kAdtsLast = 8 };
constexpr uint32_t kAdtsEnd = 0xffffffffu;       // no successor
constexpr uint32_t kAdtsUnranked = 0xffffffffu;  // not (yet) known to be on its file's chain

SYMGPU_PACKET_HD inline uint32_t adts_node(const uint8_t* d, size_t n, size_t q) {
    AdtsHeader h;
    const Status s = adts_parse_header(d + q, n - q, h);
    if (s == Status::EndOfStream) return kAdtsStopOk;
    if (s != Status::Ok) return s == Status::DecodeError ? kAdtsStopDecode : kAdtsStopUnsupported;
    if (q + h.frame_len > n) return kAdtsStopLimit;
    return uint32_t(h.frame_len) << 4 | kAdtsFrame;
}

// 3. A node's successor: for candidate c, a Frame, the first candidate at or after the frame's end when it lies before file_end
//    (the virtual end of c's file); else, and for a Stop, kAdtsEnd.  vpos: the n_cand candidates' virtual positions, ascending.
SYMGPU_PACKET_HD inline uint32_t adts_successor(const uint64_t* vpos, uint32_t n_cand, uint32_t c, uint32_t node, uint64_t file_end) {
    if ((node & 7) != kAdtsFrame) return kAdtsEnd;
    const uint32_t lo = detail::first_at_or_after(vpos, c + 1, n_cand, vpos[c] + (node >> 4));
    return lo < n_cand && vpos[lo] < file_end ? lo : kAdtsEnd;
}

// 4. The chain of a file starts at its first candidate, rank 0: candidate c is one when the one before it lies before file_begin
//    (the virtual start of c's file).  Every other candidate starts unranked.
SYMGPU_PACKET_HD inline uint32_t adts_initial_rank(const uint64_t* vpos, uint32_t c, uint64_t file_begin) {
    return c == 0 || vpos[c - 1] < file_begin ? 0 : kAdtsUnranked;
}

// 5. Doubling round k at candidate c: jump = J_k (J_0: the successors), next = J_(k+1) = J_k o J_k, and a chain node ranked below
//    2^k ranks the node J_k leads to as its rank + 2^k.  After round k exactly the chain nodes of rank below 2^(k+1) are ranked.
//    The candidates may run in any order: J_k is injective on the chain, so no two writes meet, and a node ranked in round k had no
//    rank before it and gets one of at least 2^k, so its own test fails whether it reads the old rank or the new one.
SYMGPU_PACKET_HD inline void adts_double(uint32_t* rank, const uint32_t* jump, uint32_t* next, uint32_t c, uint32_t k) {
    const uint32_t j = jump[c], r = rank[c];
    next[c] = j == kAdtsEnd ? kAdtsEnd : jump[j];
    if (j != kAdtsEnd && r < (1u << k)) rank[j] = r + (1u << k);
}

// The rounds that rank every chain of files of at most max_len bytes: a chain has at most max_len / 2 nodes.
SYMGPU_PACKET_HD inline uint32_t adts_rounds(uint64_t max_len) {
    uint32_t k = 0;
    for (uint64_t m = max_len / 2; m; m >>= 1) ++k;
    return k;
}

// 6. The file's record from its chain's last node (ranked, kAdtsLast): its packets are the chain's Frames, and the stop is the
//    last node's kind, or a clean end after a Frame.
SYMGPU_PACKET_HD inline void adts_file_end(uint32_t node, uint32_t rank, uint32_t* n_packets, uint32_t* stop) {
    const bool frame = (node & 7) == kAdtsFrame;
    *n_packets = rank + (frame ? 1u : 0u), *stop = frame ? kAdtsStopOk : node & 7;
}

// 7. The packet of the chain's Frame of rank `rank` at q of a file of n bytes, as AdtsIndexer::next gives it.
SYMGPU_PACKET_HD inline AdtsPacket adts_frame_packet(const uint8_t* d, size_t n, size_t q, uint32_t rank) {
    AdtsHeader h{};
    adts_parse_header(d + q, n - q, h);
    AdtsPacket p{};
    p.offset = q + h.header_len, p.size = h.payload_len(), p.pts = int64_t(rank) * 1024;
    p.sample_rate = h.sample_rate, p.channels = h.channels, p.profile = h.profile;
    return p;
}

// =====================================================================================================================
// Ogg
// =====================================================================================================================

constexpr size_t kOggHeaderSize = 27;
constexpr size_t kOggMaxPageSize = kOggHeaderSize + 255 + 255 * 255;  // page.rs:17
constexpr uint64_t kOggMaxPacketLen = 16u * 1024 * 1024;              // logical.rs:61

struct OggPage {
    uint64_t offset;       // of the capture pattern
    uint64_t absgp;        // granule position
    uint32_t serial, sequence, crc;
    uint8_t n_segments;
    bool continuation, first, last;
    uint64_t body_offset;  // first body byte
    uint32_t body_len;
    const uint8_t* lacing; // the n_segments lacing values, in the source buffer
    uint16_t n_packets;    // packets that END on this page
    uint16_t packet_len[255];
    uint32_t partial_len() const {  // body bytes after the last packet end: a packet continued on a later page
        uint32_t used = 0;
        for (unsigned i = 0; i < n_packets; ++i) used += packet_len[i];
        return body_len - used;
    }
};

// The fields of a page header, read where a capture pattern was found.
struct OggPageHead {
    uint64_t offset;       // of the capture pattern
    uint64_t absgp;        // granule position
    uint64_t body_offset;  // first body byte
    uint32_t serial, sequence, crc, body_len;
    uint8_t n_segments;    // lacing values, at offset + kOggHeaderSize
    bool continuation, first, last;
};

// The header fields of the page at q, its lacing values included (the caller knows they lie inside the buffer).
SYMGPU_PACKET_HD inline void ogg_page_fields(const uint8_t* d, size_t q, OggPageHead& pg) {
    const uint8_t* h = d + q;
    pg.offset = q;
    pg.continuation = h[5] & 1, pg.first = (h[5] & 2) != 0, pg.last = (h[5] & 4) != 0;
    pg.absgp = detail::le64(h + 6);
    pg.serial = detail::le32(h + 14), pg.sequence = detail::le32(h + 18), pg.crc = detail::le32(h + 22);
    pg.n_segments = h[26];
    uint32_t body = 0;
    for (unsigned i = 0; i < pg.n_segments; ++i) body += h[kOggHeaderSize + i];
    pg.body_offset = q + kOggHeaderSize + pg.n_segments, pg.body_len = body;
}

// One attempt of page.rs:166-271 at a capture pattern: d[0..n) is the file, "OggS" starts at q (q + 4 <= n).  Ok: a page
// that verifies, *next = its end.  DecodeError: a bad version / flag byte (*next = q + 27, the search resumes after that
// header) or a checksum mismatch (*next = q + 4, right after the capture pattern).  EndOfStream: the header, the lacing or the
// body is cut by the end of the file, which ends the search.  Nothing outside d[0..n) is read.  `crc` is a slicing-by-8 table.
SYMGPU_PACKET_HD inline Status ogg_check_page(const uint8_t* d, size_t n, size_t q, const uint32_t (*crc)[256], OggPageHead& pg, size_t* next) {
    *next = n;
    if (q + kOggHeaderSize > n) return Status::EndOfStream;
    const uint8_t* h = d + q;
    if (h[4] != 0 || (h[5] & 0xf8)) return *next = q + kOggHeaderSize, Status::DecodeError;
    if (q + kOggHeaderSize + h[26] > n) return Status::EndOfStream;
    ogg_page_fields(d, q, pg);
    const uint32_t body = pg.body_len;
    if (pg.body_offset + body > n) return Status::EndOfStream;
    // checksum over the page with its own checksum field read as zero
    const uint8_t zero[4] = {0, 0, 0, 0};
    uint32_t c = crc32_update_with(crc, 0, h, 22);
    c = crc32_update_with(crc, c, zero, 4);
    c = crc32_update_with(crc, c, h + 26, 1 + size_t(pg.n_segments) + body);
    if (c != pg.crc) return *next = q + 4, Status::DecodeError;
    *next = pg.body_offset + body;
    return Status::Ok;
}

// page.rs:166-271 over a resident buffer.
class OggPageReader {
  public:
    OggPageReader(const uint8_t* data, size_t n) : d_(data), n_(n) {}

    // One attempt (try_next_page): DecodeError for a bad version / flag byte (the search resumes after that header)
    // or a checksum mismatch (the search resumes right after the capture pattern that led here).
    Status try_next(OggPage& pg) {
        size_t q = pos_;
        for (;; ++q) {
            if (q + 4 > n_) return pos_ = n_, Status::EndOfStream;
            if (d_[q] != 'O') {
                const void* hit = std::memchr(d_ + q, 'O', n_ - q);
                if (!hit) return pos_ = n_, Status::EndOfStream;
                q = size_t(static_cast<const uint8_t*>(hit) - d_);
                if (q + 4 > n_) return pos_ = n_, Status::EndOfStream;
            }
            if (std::memcmp(d_ + q, "OggS", 4) == 0) break;
        }
        static constexpr detail::Crc32Table tab{};
        OggPageHead h;
        const Status s = ogg_check_page(d_, n_, q, tab.t, h, &pos_);
        if (s != Status::Ok) return s;
        pg.offset = h.offset, pg.absgp = h.absgp, pg.serial = h.serial, pg.sequence = h.sequence, pg.crc = h.crc;
        pg.n_segments = h.n_segments, pg.continuation = h.continuation, pg.first = h.first, pg.last = h.last;
        pg.body_offset = h.body_offset, pg.body_len = h.body_len;
        pg.lacing = d_ + q + kOggHeaderSize;
        uint32_t run = 0;
        pg.n_packets = 0;
        for (unsigned i = 0; i < pg.n_segments; ++i) {
            run += pg.lacing[i];
            if (pg.lacing[i] < 255) pg.packet_len[pg.n_packets++] = uint16_t(run), run = 0;  // a short segment closes a packet
        }
        return Status::Ok;
    }

    // next_page: skip whatever does not verify.
    Status next(OggPage& pg) {
        for (;;) {
            const Status s = try_next(pg);
            if (s == Status::Ok || s == Status::EndOfStream) return s;
            ++n_rejected_;
        }
    }
    size_t position() const { return pos_; }
    size_t rejected() const { return n_rejected_; }

  private:
    const uint8_t* d_;
    size_t n_;
    size_t pos_ = 0;
    size_t n_rejected_ = 0;
};

// A packet of a logical stream: pieces [first_piece, first_piece + n_pieces) of the stream's piece list.
struct OggPacket {
    uint32_t first_piece;
    uint32_t n_pieces;
    uint64_t len;
    uint32_t page_sequence;  // of the page it ended on
    uint64_t page_absgp;     // granule position of that page: the end time of its LAST completed packet
    bool last_on_page;
};

// What a logical stream carries from one page to the next.  The stream's pieces are numbered from 0; the open packet owns
// pieces [part_first, n_pieces).
struct OggStreamState {
    uint64_t part_len = 0;  // bytes of the packet still waiting for its continuation
    uint32_t part_first = 0, n_pieces = 0, prev_seq = 0;
    bool have_prev = false;
};

// logical.rs:104-205, 577-620 without the codec mapper: one page of a logical stream.  `lacing` holds the page's
// n_segments lacing values.  The sink is told sink.piece(index, offset, len) for every piece (an index below an earlier
// one replaces what was dropped), sink.packet(first_piece, n_pieces, len, page) for every completed packet and
// sink.last_on_page() after the page's last completed packet.  DecodeError when an open packet would pass the reference's
// 16 MiB cap; the page's completed packets are kept.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable  // a host sink makes a host-only instantiation
#endif
template <class Sink>
SYMGPU_PACKET_HD inline Status ogg_stream_page(OggStreamState& st, const OggPageHead& pg, const uint8_t* lacing, Sink& sink) {
    if (st.have_prev && (pg.sequence < st.prev_seq || pg.sequence - st.prev_seq > 1)) st.n_pieces = st.part_first, st.part_len = 0;  // lost or re-ordered pages
    st.have_prev = true, st.prev_seq = pg.sequence;
    if (!pg.continuation && st.part_len > 0) st.n_pieces = st.part_first, st.part_len = 0;  // the continuation never came
    unsigned seg = 0;
    // the next packet that ends on this page (false: none left)
    auto next_len = [&](uint32_t& len) {
        uint32_t run = 0;
        while (seg < pg.n_segments) {
            const uint8_t v = lacing[seg++];
            run += v;
            if (v < 255) return len = run, true;
        }
        return false;
    };
    uint64_t at = pg.body_offset;
    uint32_t n;
    bool more = next_len(n);
    if (pg.continuation && st.part_len == 0) {
        // the head of this packet was never seen: drop its tail, or the whole page when nothing else ends here
        if (!more) return Status::Ok;
        at += n;
        more = next_len(n);
    }
    bool any = false;
    for (; more; more = next_len(n)) {
        sink.piece(st.n_pieces++, at, n);
        sink.packet(st.part_first, st.n_pieces - st.part_first, st.part_len + n, pg);
        st.part_first = st.n_pieces, st.part_len = 0;
        at += n;
        any = true;
    }
    if (any) sink.last_on_page();
    const uint64_t rest = pg.body_offset + pg.body_len - at;
    if (rest > 0) {
        if (st.part_len + rest > kOggMaxPacketLen) return Status::DecodeError;
        sink.piece(st.n_pieces++, at, uint32_t(rest));
        st.part_len += rest;
    }
    return Status::Ok;
}

class OggLogicalStream {
  public:
    // DecodeError when an open packet would pass the reference's 16 MiB cap; the page's completed packets are kept.
    Status read_page(const OggPage& pg) {
        OggPageHead h;
        h.offset = pg.offset, h.absgp = pg.absgp, h.body_offset = pg.body_offset, h.serial = pg.serial, h.sequence = pg.sequence;
        h.crc = pg.crc, h.body_len = pg.body_len, h.n_segments = pg.n_segments;
        h.continuation = pg.continuation, h.first = pg.first, h.last = pg.last;
        Sink sink{this};
        const Status s = ogg_stream_page(st_, h, pg.lacing, sink);
        pieces_.resize(st_.n_pieces);
        return s;
    }

    const std::vector<OggPacket>& packets() const { return packets_; }
    const std::vector<Piece>& pieces() const { return pieces_; }
    uint64_t open_len() const { return st_.part_len; }  // bytes of a packet still waiting for its continuation

    // Copy a packet out of the source buffer (tests, host-side header parsing); the device path gathers instead.
    void gather(const uint8_t* src, const OggPacket& p, uint8_t* dst) const {
        for (uint32_t k = 0; k < p.n_pieces; ++k) {
            const Piece& pc = pieces_[p.first_piece + k];
            std::memcpy(dst, src + pc.offset, pc.len);
            dst += pc.len;
        }
    }

  private:
    struct Sink {
        OggLogicalStream* ls;
        void piece(uint32_t i, uint64_t offset, uint32_t len) {
            ls->pieces_.resize(i);
            ls->pieces_.push_back(Piece{offset, len});
        }
        void packet(uint32_t first, uint32_t count, uint64_t len, const OggPageHead& pg) {
            ls->packets_.push_back(OggPacket{first, count, len, pg.sequence, pg.absgp, false});
        }
        void last_on_page() { ls->packets_.back().last_on_page = true; }
    };
    std::vector<OggPacket> packets_;
    std::vector<Piece> pieces_;
    OggStreamState st_;
};

// ---- the schedule of the device index (symgpu_ogg_index_dev), step by step over one file d[0..n) --------------------------
// 1. A successor word per 4-byte group, each found on its own: two capture patterns cannot start within 4 bytes of each other, so
//    a group holds at most one.  0 = none; else bits 0-1 its place in the group, bits 2-3 the kind, bits 5.. the distance from
//    it to where the reader goes next (< 2^17: at most a page).
enum : uint32_t { kOggWordPage = 1, kOggWordSkip = 2, kOggWordEnd = 3 };

SYMGPU_PACKET_HD inline uint32_t ogg_successor_word(const uint8_t* d, size_t n, size_t w, const uint32_t (*crc)[256]) {
    for (uint32_t k = 0; k < 4 && w * 4 + k + 4 <= n; ++k) {
        const size_t q = w * 4 + k;
        if (d[q] != 'O' || d[q + 1] != 'g' || d[q + 2] != 'g' || d[q + 3] != 'S') continue;
        OggPageHead pg;
        size_t next;
        const Status s = ogg_check_page(d, n, q, crc, pg, &next);
        const uint32_t kind = s == Status::Ok ? kOggWordPage : s == Status::DecodeError ? kOggWordSkip : kOggWordEnd;
        return uint32_t(kind == kOggWordEnd ? 0 : next - q) << 5 | kind << 2 | k;
    }
    return 0;
}

// 2. The chain: the next page that verifies at or after *pos (false: the file ends); *pos moves past it as the reader's does.
//    Over a whole file, *pos only grows, so the chain costs one look per word at most.
SYMGPU_PACKET_HD inline bool ogg_next_page(const uint32_t* succ, uint64_t n, uint64_t* pos, uint64_t* page) {
    const uint64_t n_words = (n + 3) / 4;
    for (uint64_t w = *pos / 4; w < n_words; ++w) {
        const uint32_t v = succ[w];
        if (!v) continue;
        const uint64_t q = w * 4 + (v & 3);
        if (q < *pos) continue;
        const uint32_t kind = (v >> 2) & 3;
        if (kind == kOggWordEnd) break;
        *pos = q + (v >> 5);
        if (kind == kOggWordPage) return *page = q, true;
        w = *pos / 4 - 1;
    }
    *pos = n;
    return false;
}

// 3. The chain's pages ordered by serial, chain order kept within a serial: a stable least-significant-digit radix sort, four
//    passes of 8 bits, so linear in the pages whatever the serials.  keys[i] = the serial of page i, vals[i] = its offset;
//    tmp_keys / tmp_vals hold n items each; the result is back in keys / vals.
SYMGPU_PACKET_HD inline void ogg_sort_by_serial(uint32_t* keys, uint32_t* vals, uint32_t* tmp_keys, uint32_t* tmp_vals, size_t n) {
    uint32_t *ik = keys, *iv = vals, *ok = tmp_keys, *ov = tmp_vals;
    for (int shift = 0; shift < 32; shift += 8) {
        uint32_t count[256];
        for (int b = 0; b < 256; ++b) count[b] = 0;
        for (size_t i = 0; i < n; ++i) ++count[(ik[i] >> shift) & 0xff];
        uint32_t at = 0;
        for (int b = 0; b < 256; ++b) {
            const uint32_t c = count[b];
            count[b] = at, at += c;
        }
        for (size_t i = 0; i < n; ++i) {
            const uint32_t j = count[(ik[i] >> shift) & 0xff]++;
            ok[j] = ik[i], ov[j] = iv[i];
        }
        uint32_t* t = ik;
        ik = ok, ok = t, t = iv, iv = ov, ov = t;
    }
}

// 4. The logical streams (OggIndex::build's routing) from the chain sorted by serial: in ascending serial order, a serial's pages
//    before its first first-page are orphans, the rest go through ogg_stream_page.  sink.begin_stream(serial) / end_stream()
//    bracket every stream.  Linear in the pages.  Returns true when a page hit the 16 MiB cap.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable  // a host sink makes a host-only instantiation
#endif
template <class Sink>
SYMGPU_PACKET_HD inline bool ogg_walk_streams(const uint8_t* d, const uint32_t* serials, const uint32_t* offsets, size_t n_pages, Sink& sink) {
    bool cap_hit = false;
    for (size_t k = 0; k < n_pages;) {
        const uint32_t serial = serials[k];
        size_t j = k;
        while (j < n_pages && serials[j] == serial && !(d[offsets[j] + 5] & 2)) ++j;
        if (j < n_pages && serials[j] == serial) {
            OggStreamState st;
            sink.begin_stream(serial);
            for (; j < n_pages && serials[j] == serial; ++j) {
                OggPageHead pg;
                ogg_page_fields(d, offsets[j], pg);
                if (ogg_stream_page(st, pg, d + offsets[j] + kOggHeaderSize, sink) != Status::Ok) cap_hit = true;
            }
            sink.end_stream();
        }
        k = j;
    }
    return cap_hit;
}

// A physical stream: every page that verifies, routed by serial number.  A logical stream exists from its
// beginning-of-stream page on (demuxer.rs:320-345); pages of serials never announced are counted and skipped.
struct OggIndex {
    std::vector<OggPage> pages;
    std::map<uint32_t, OggLogicalStream> streams;
    size_t rejected = 0;  // capture patterns that did not lead to a valid page
    size_t orphans = 0;   // valid pages of unannounced serials

    static Status build(const uint8_t* data, size_t n, OggIndex& ix, bool keep_pages = true) {
        OggPageReader rd(data, n);
        OggPage pg;
        Status worst = Status::Ok;
        while (rd.next(pg) == Status::Ok) {
            if (keep_pages) ix.pages.push_back(pg);
            auto it = ix.streams.find(pg.serial);
            if (it == ix.streams.end()) {
                if (!pg.first) {
                    ++ix.orphans;
                    continue;
                }
                it = ix.streams.emplace(pg.serial, OggLogicalStream{}).first;
            }
            if (it->second.read_page(pg) != Status::Ok) worst = Status::DecodeError;
        }
        ix.rejected = rd.rejected();
        return worst;
    }
};

// =====================================================================================================================
// Vorbis in Ogg: what the container layer has to know about the codec
// =====================================================================================================================
// The mapper (symphonia-format-ogg/src/mappings/vorbis.rs) sorts a logical stream's packets into identification /
// comment / setup headers and audio, hands the decoder its `extra_data` (identification packet followed by the
// setup packet, consumed at symphonia-codec-vorbis/src/lib.rs:75-89) and derives every audio packet's duration
// from its first bits: the mode number selects a short or long block, and a packet yields a quarter of the
// previous block plus a quarter of its own.  For that it must walk the WHOLE setup header -- codebooks, floors,
// residues, mappings -- just to reach the mode list at its end.

// Bits least-significant first, as Vorbis packs them (symphonia-core/src/io/bit.rs:941-1027).
class BitReaderRtl {
  public:
    SYMGPU_PACKET_HD BitReaderRtl(const uint8_t* p, size_t n) : p_(p), n_bits_(uint64_t(n) * 8) {}
    SYMGPU_PACKET_HD bool ok() const { return ok_; }
    SYMGPU_PACKET_HD uint64_t bits_left() const { return n_bits_ - at_; }
    // Past the end: returns 0 and latches !ok() (every caller checks once per structure, not per field).
    SYMGPU_PACKET_HD uint32_t read(unsigned width) {
        if (width > bits_left()) return ok_ = false, at_ = n_bits_, 0u;
        uint64_t v = 0;
        const uint64_t byte = at_ >> 3;
        const unsigned shift = unsigned(at_ & 7), need = (shift + width + 7) >> 3;
        for (unsigned k = 0; k < need; ++k) v |= uint64_t(p_[byte + k]) << (8 * k);
        at_ += width;
        return uint32_t((v >> shift) & ((uint64_t(1) << width) - 1));
    }
    SYMGPU_PACKET_HD bool read_bool() { return read(1) != 0; }
    SYMGPU_PACKET_HD void ignore(uint64_t width) {
        if (width > bits_left()) ok_ = false, at_ = n_bits_;
        else at_ += width;
    }

  private:
    const uint8_t* p_;
    uint64_t n_bits_, at_ = 0;
    bool ok_ = true;
};

SYMGPU_PACKET_HD inline uint32_t vorbis_ilog(uint32_t x) {
    uint32_t n = 0;
    for (; x; x >>= 1) ++n;
    return n;
}

struct VorbisIdent {
    uint8_t n_channels;
    uint32_t sample_rate;
    uint8_t bs0_exp, bs1_exp;  // block sizes as powers of two, 6..13, short <= long
};

// mappings/vorbis.rs:293-360.  The Ogg mapper only accepts an identification packet of exactly 30 bytes (:113-117).
inline Status vorbis_read_ident(const uint8_t* p, size_t n, VorbisIdent& id) {
    if (n < 30) return Status::EndOfStream;
    if (p[0] != 1 || std::memcmp(p + 1, "vorbis", 6) != 0) return Status::DecodeError;
    if (detail::le32(p + 7) != 0) return Status::Unsupported;
    id.n_channels = p[11];
    id.sample_rate = detail::le32(p + 12);
    if (id.n_channels == 0 || id.sample_rate == 0) return Status::DecodeError;
    id.bs0_exp = p[28] & 15, id.bs1_exp = p[28] >> 4;
    if (id.bs0_exp < 6 || id.bs0_exp > 13 || id.bs1_exp < 6 || id.bs1_exp > 13 || id.bs0_exp > id.bs1_exp) return Status::DecodeError;
    if (p[29] != 1) return Status::DecodeError;  // framing
    return Status::Ok;
}

namespace detail {
// The largest v with v^dims <= entries (the reference computes it in f32 and asserts exactly this, :717-730).
inline uint32_t vorbis_lookup1_values(uint32_t entries, uint32_t dims) {
    if (dims == 1) return entries;  // (untrusted input: keep the search short -- for dims >= 2 the root of 2^24 is <= 4096)
    uint32_t v = 0;
    for (;;) {
        uint64_t pw = 1;
        bool over = false;
        for (uint32_t k = 0; k < dims && !over; ++k) pw *= uint64_t(v) + 1, over = pw > entries;
        if (over) return v;
        ++v;
    }
}

// mappings/vorbis.rs:426-500.
inline bool vorbis_skip_codebook(BitReaderRtl& bs) {
    if (bs.read(24) != 0x564342 || !bs.ok()) return false;
    const uint32_t dims = bs.read(16), entries = bs.read(24);
    if (!bs.read_bool()) {        // lengths in entry order
        if (bs.read_bool()) {     // sparse: a used flag in front of every length
            for (uint32_t i = 0; i < entries && bs.ok(); ++i)
                if (bs.read_bool()) bs.read(5);
        } else {
            bs.ignore(uint64_t(entries) * 5);
        }
    } else {                      // lengths as run lengths of ascending code length
        bs.read(5);
        for (uint32_t cur = 0;;) {
            cur += bs.read(entries > cur ? vorbis_ilog(entries - cur) : 0);
            if (!bs.ok() || cur > entries) return false;
            if (cur == entries) break;
        }
    }
    const uint32_t lookup = bs.read(4);
    if (!bs.ok()) return false;
    if (lookup == 0) return true;
    if (lookup > 2) return false;
    bs.ignore(64);
    const uint32_t value_bits = bs.read(4) + 1;
    bs.read_bool();
    if (!bs.ok()) return false;
    if (lookup == 1 && dims == 0) return false;  // the reference's float root is meaningless here (it asserts)
    const uint64_t values = lookup == 1 ? vorbis_lookup1_values(entries, dims) : uint64_t(entries) * dims;
    bs.ignore(values * value_bits);
    return bs.ok();
}

// :528-590
inline bool vorbis_skip_floor(BitReaderRtl& bs) {
    const uint32_t type = bs.read(16);
    if (!bs.ok() || type > 1) return false;
    if (type == 0) {
        bs.ignore(8 + 16 + 16 + 6 + 8);
        bs.ignore((uint64_t(bs.read(4)) + 1) * 8);
        return bs.ok();
    }
    const uint32_t partitions = bs.read(5);
    uint8_t cls[32] = {0}, dims[16] = {0};
    if (partitions > 0) {
        uint32_t max_class = 0;
        for (uint32_t i = 0; i < partitions; ++i) {
            cls[i] = uint8_t(bs.read(4));
            if (cls[i] > max_class) max_class = cls[i];
        }
        for (uint32_t c = 0; c <= max_class; ++c) {
            dims[c] = uint8_t(bs.read(3) + 1);
            const uint32_t sub = bs.read(2);
            if (sub) bs.read(8);
            bs.ignore((uint64_t(1) << sub) * 8);
        }
    }
    bs.read(2);
    const uint32_t rangebits = bs.read(4);
    for (uint32_t i = 0; i < partitions; ++i) bs.ignore(uint64_t(dims[cls[i]]) * rangebits);
    return bs.ok();
}

// :592-620
inline bool vorbis_skip_residue(BitReaderRtl& bs) {
    bs.read(16);
    bs.ignore(24 + 24 + 24);
    const uint32_t classes = bs.read(6) + 1;
    bs.ignore(8);
    uint32_t books = 0;
    for (uint32_t i = 0; i < classes && bs.ok(); ++i) {
        uint32_t used = bs.read(3);
        if (bs.read_bool()) used |= bs.read(5) << 3;
        for (; used; used &= used - 1) ++books;
    }
    bs.ignore(uint64_t(books) * 8);
    return bs.ok();
}

// :622-673
inline bool vorbis_skip_mapping(BitReaderRtl& bs, uint8_t channels) {
    if (bs.read(16) != 0 || !bs.ok()) return false;
    const uint32_t submaps = bs.read_bool() ? bs.read(4) + 1 : 1;
    if (bs.read_bool()) {
        const uint32_t steps = bs.read(8) + 1, width = vorbis_ilog(uint32_t(channels) - 1);
        bs.ignore(uint64_t(steps) * 2 * width);
    }
    if (bs.read(2) != 0 || !bs.ok()) return false;
    if (submaps > 1) bs.ignore(uint64_t(channels) * 4);
    bs.ignore(uint64_t(submaps) * 24);
    return bs.ok();
}
}  // namespace detail

// mappings/vorbis.rs:362-405, 675-708: the mode list of a setup packet, as a bit mask of "long block" flags.
inline Status vorbis_read_setup_modes(const uint8_t* p, size_t n, const VorbisIdent& id, uint8_t& num_modes, uint64_t& long_block_mask) {
    if (n < 7) return Status::EndOfStream;
    if (p[0] != 5 || std::memcmp(p + 1, "vorbis", 6) != 0) return Status::DecodeError;
    BitReaderRtl bs(p + 7, n - 7);
    for (uint32_t i = 0, count = bs.read(8) + 1; i < count; ++i)
        if (!detail::vorbis_skip_codebook(bs)) return Status::DecodeError;
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i)
        if (bs.read(16) != 0 || !bs.ok()) return Status::DecodeError;  // time-domain transforms: placeholders
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i)
        if (!detail::vorbis_skip_floor(bs)) return Status::DecodeError;
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i)
        if (!detail::vorbis_skip_residue(bs)) return Status::DecodeError;
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i)
        if (!detail::vorbis_skip_mapping(bs, id.n_channels)) return Status::DecodeError;
    const uint32_t count = bs.read(6) + 1;
    uint64_t mask = 0;
    for (uint32_t i = 0; i < count; ++i) {
        if (bs.read_bool()) mask |= uint64_t(1) << i;
        const uint32_t window = bs.read(16), transform = bs.read(16);
        bs.read(8);
        if (!bs.ok() || window != 0 || transform != 0) return Status::DecodeError;
    }
    if (!bs.read_bool() || !bs.ok()) return Status::DecodeError;  // framing
    num_modes = uint8_t(count), long_block_mask = mask;
    return Status::Ok;
}

// ---- the decoder's view of the setup header ---------------------------------------------------------------------------
// symphonia-codec-vorbis/src/lib.rs:490-770 (read_setup: floors, residues, mappings, modes with their cross checks),
// floor.rs:160-201 (floor 0), :455-560 (floor 1: classes, X list, neighbours, sort order), residue.rs:73-140.
// Everything the synthesis configuration needs EXCEPT the codebooks' contents, which are walked over with the same
// syntax checks as above but not built (their Huffman trees and VQ tables belong to the packet decoder).
struct VorbisFloor1Setup {
    uint8_t multiplier;  // 1..4
    uint8_t n_posts;     // 2..65
    uint16_t x_list[65];
    uint8_t low[65], high[65];   // neighbours among the earlier posts (0, 0 for the first two, as find_neighbors leaves them)
    uint8_t sort_order[65];      // posts by ascending x (stable)
    uint8_t partitions;
    uint8_t partition_class[32];
    struct Class {
        uint8_t dimensions, subclass_bits, mainbook, subbook_used;
        uint8_t subbooks[8];
    } classes[16];
};
struct VorbisResidueSetup {
    uint16_t type;
    uint32_t begin, end, partition_size;
    uint8_t classifications, classbook, max_pass;
    uint8_t used[64];
    uint8_t books[64][8];
};
struct VorbisMappingSetup {
    uint8_t n_submaps;
    std::vector<std::pair<uint8_t, uint8_t>> couplings;  // (magnitude channel, angle channel)
    std::vector<uint8_t> multiplex;                      // sub-map of each channel
    uint8_t submap_floor[16], submap_residue[16];
};
struct VorbisSetup {
    uint32_t n_codebooks = 0;
    std::vector<uint8_t> floor_type;          // 0 or 1 per floor
    std::vector<VorbisFloor1Setup> floor1;    // per floor; zeroed for type-0 floors
    std::vector<VorbisResidueSetup> residues;
    std::vector<VorbisMappingSetup> mappings;
    std::vector<std::pair<bool, uint8_t>> modes;  // (long block, mapping)
};

inline Status vorbis_read_setup(const uint8_t* p, size_t n, const VorbisIdent& id, VorbisSetup& out) {
    if (n < 7) return Status::EndOfStream;
    if (p[0] != 5 || std::memcmp(p + 1, "vorbis", 6) != 0) return Status::DecodeError;
    BitReaderRtl bs(p + 7, n - 7);
    out = VorbisSetup{};
    out.n_codebooks = bs.read(8) + 1;
    for (uint32_t i = 0; i < out.n_codebooks; ++i)
        if (!detail::vorbis_skip_codebook(bs)) return Status::DecodeError;
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i)
        if (bs.read(16) != 0 || !bs.ok()) return Status::DecodeError;
    const uint8_t max_book = uint8_t(out.n_codebooks);  // `codebooks.len() as u8` (lib.rs:517): 256 codebooks wrap to 0
    // ---- floors
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i) {
        const uint32_t type = bs.read(16);
        if (!bs.ok() || type > 1) return Status::DecodeError;
        VorbisFloor1Setup f{};
        if (type == 0) {
            bs.ignore(8 + 16 + 16 + 6 + 8);
            for (uint32_t k = 0, books = bs.read(4) + 1; k < books; ++k)
                if (bs.read(8) >= max_book || !bs.ok()) return Status::DecodeError;
        } else {
            f.partitions = uint8_t(bs.read(5));
            if (f.partitions) {
                uint8_t max_class = 0;
                for (int k = 0; k < f.partitions; ++k) f.partition_class[k] = uint8_t(bs.read(4)), max_class = std::max(max_class, f.partition_class[k]);
                for (int c = 0; c <= max_class; ++c) {
                    auto& cl = f.classes[c];
                    cl.dimensions = uint8_t(bs.read(3) + 1), cl.subclass_bits = uint8_t(bs.read(2));
                    if (cl.subclass_bits) {
                        cl.mainbook = uint8_t(bs.read(8));
                        if (cl.mainbook >= max_book) return Status::DecodeError;
                    }
                    for (int k = 0; k < (1 << cl.subclass_bits); ++k) {
                        uint8_t book = uint8_t(bs.read(8));
                        if (book > 0) {  // 0 = no codebook for this sub-class; otherwise the number minus one
                            if (--book >= max_book) return Status::DecodeError;
                            cl.subbook_used |= uint8_t(1 << k);
                        }
                        cl.subbooks[k] = book;
                    }
                }
            }
            f.multiplier = uint8_t(bs.read(2) + 1);
            const uint32_t rangebits = bs.read(4);
            if (!bs.ok()) return Status::DecodeError;
            int np = 0;
            f.x_list[np++] = 0, f.x_list[np++] = uint16_t(1u << rangebits);
            for (int k = 0; k < f.partitions; ++k) {
                const int dims = f.classes[f.partition_class[k]].dimensions;
                if (np + dims > 65) return Status::DecodeError;
                for (int d = 0; d < dims; ++d) {
                    const uint32_t x = bs.read(rangebits);
                    // every READ element must be new among the read ones; the two implied ends are not in that set
                    // (floor.rs:519-536 inserts only what it reads)
                    for (int e = 2; e < np; ++e)
                        if (f.x_list[e] == x) return Status::DecodeError;
                    f.x_list[np++] = uint16_t(x);
                }
            }
            if (!bs.ok()) return Status::DecodeError;
            f.n_posts = uint8_t(np);
            for (int i2 = 0; i2 < np; ++i2) {  // floor.rs:748-773
                uint32_t lo = 0, hi = 0xffffffffu;
                for (int e = 0; e < i2; ++e) {
                    const uint32_t xv = f.x_list[e];
                    if (xv > lo && xv < f.x_list[i2]) lo = xv, f.low[i2] = uint8_t(e);
                    if (xv < hi && xv > f.x_list[i2]) hi = xv, f.high[i2] = uint8_t(e);
                }
                f.sort_order[i2] = uint8_t(i2);
            }
            std::stable_sort(f.sort_order, f.sort_order + np, [&](uint8_t a, uint8_t b) { return f.x_list[a] < f.x_list[b]; });
        }
        out.floor_type.push_back(uint8_t(type)), out.floor1.push_back(f);
    }
    // ---- residues
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i) {
        VorbisResidueSetup r{};
        r.type = uint16_t(bs.read(16));
        if (!bs.ok() || r.type > 2) return Status::DecodeError;
        r.begin = bs.read(24), r.end = bs.read(24), r.partition_size = bs.read(24) + 1;
        r.classifications = uint8_t(bs.read(6) + 1), r.classbook = uint8_t(bs.read(8));
        if (!bs.ok() || r.classbook >= max_book || r.end < r.begin) return Status::DecodeError;
        for (int c = 0; c < r.classifications; ++c) {
            const uint32_t low = bs.read(3);
            r.used[c] = uint8_t((bs.read_bool() ? bs.read(5) << 3 : 0) | low);
        }
        for (int c = 0; c < r.classifications; ++c)
            for (int j = 0; j < 8; ++j)
                if (r.used[c] & (1 << j)) {
                    r.books[c][j] = uint8_t(bs.read(8));
                    if (!bs.ok() || r.books[c][j] == 0 || r.books[c][j] >= max_book) return Status::DecodeError;
                    r.max_pass = std::max<uint8_t>(r.max_pass, uint8_t(j));
                }
        if (!bs.ok()) return Status::DecodeError;
        out.residues.push_back(r);
    }
    // ---- mappings
    const uint8_t max_floor = uint8_t(out.floor_type.size()), max_residue = uint8_t(out.residues.size());
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i) {
        if (bs.read(16) != 0 || !bs.ok()) return Status::DecodeError;
        VorbisMappingSetup m{};
        m.n_submaps = uint8_t(bs.read_bool() ? bs.read(4) + 1 : 1);
        if (bs.read_bool()) {
            const uint32_t steps = bs.read(8) + 1, width = vorbis_ilog(uint32_t(id.n_channels) - 1), max_ch = uint32_t(id.n_channels) - 1;
            for (uint32_t k = 0; k < steps; ++k) {
                const uint32_t mag = bs.read(width) & 0xff, ang = bs.read(width) & 0xff;
                if (!bs.ok() || mag == ang || mag > max_ch || ang > max_ch) return Status::DecodeError;
                m.couplings.emplace_back(uint8_t(mag), uint8_t(ang));
            }
        }
        if (bs.read(2) != 0 || !bs.ok()) return Status::DecodeError;
        m.multiplex.assign(id.n_channels, 0);
        if (m.n_submaps > 1)
            for (int c = 0; c < id.n_channels; ++c) {
                m.multiplex[c] = uint8_t(bs.read(4));
                if (!bs.ok() || m.multiplex[c] >= m.n_submaps) return Status::DecodeError;
            }
        for (int k = 0; k < m.n_submaps; ++k) {
            bs.read(8);
            m.submap_floor[k] = uint8_t(bs.read(8)), m.submap_residue[k] = uint8_t(bs.read(8));
            if (!bs.ok() || m.submap_floor[k] >= max_floor) return Status::DecodeError;
            if (m.submap_residue[k] >= max_residue) return Status::DecodeError;
        }
        out.mappings.push_back(std::move(m));
    }
    // ---- modes
    const uint8_t max_mapping = uint8_t(out.mappings.size());
    for (uint32_t i = 0, count = bs.read(6) + 1; i < count; ++i) {
        const bool flag = bs.read_bool();
        const uint32_t window = bs.read(16), transform = bs.read(16), mapping = bs.read(8);
        if (!bs.ok() || window != 0 || transform != 0 || mapping >= max_mapping) return Status::DecodeError;
        out.modes.emplace_back(flag, uint8_t(mapping));
    }
    if (!bs.read_bool() || !bs.ok()) return Status::DecodeError;
    return Status::Ok;
}

// mappings/vorbis.rs:62-106 for one packet: the block exponent its mode names, 0 when the packet is not audio (type bit set),
// is cut short or names no mode.  p / n: its first bytes (two always suffice: 1 type bit + at most 6 mode bits).
SYMGPU_PACKET_HD inline uint8_t vorbis_packet_exp(const uint8_t* p, size_t n, uint8_t num_modes, uint64_t long_block_mask, uint8_t bs0_exp,
                                                  uint8_t bs1_exp) {
    BitReaderRtl bs(p, n);
    if (bs.read_bool() || !bs.ok()) return 0;
    const uint32_t mode = bs.read(vorbis_ilog(uint32_t(num_modes) - 1)) & 0xff;
    if (!bs.ok() || mode >= num_modes) return 0;
    return (long_block_mask >> mode) & 1 ? bs1_exp : bs0_exp;
}

// (duration, leading samples to discard) of a packet of block exponent `exp` whose nearest earlier packet with a non-zero
// exponent had `prev_exp` (0: none): a packet without a block takes no time, and a first block has nothing to overlap with,
// so its lapped half is thrown away.
SYMGPU_PACKET_HD inline void vorbis_packet_time(uint8_t prev_exp, uint8_t exp, uint64_t& dur, uint64_t& discard) {
    const uint64_t cur = exp ? uint64_t(1) << exp : 0;
    dur = discard = 0;
    if (exp && prev_exp) dur = ((uint64_t(1) << prev_exp) >> 2) + (cur >> 2);
    else if (exp) dur = discard = cur >> 1;
}

// mappings/vorbis.rs:45-107: (duration, leading samples to discard) of each audio packet in turn.
class VorbisPacketTimer {
  public:
    VorbisPacketTimer() = default;
    SYMGPU_PACKET_HD VorbisPacketTimer(const VorbisIdent& id, uint8_t num_modes, uint64_t long_block_mask)
        : mask_(long_block_mask), num_modes_(num_modes), bs0_(id.bs0_exp), bs1_(id.bs1_exp) {}
    SYMGPU_PACKET_HD void reset() { prev_exp_ = 0; }
    // New headers, same overlap state (a chained stream restarts its modes but a caller batching one stream in
    // several calls carries the previous block across them).
    SYMGPU_PACKET_HD void rebind(const VorbisIdent& id, uint8_t num_modes, uint64_t long_block_mask) {
        mask_ = long_block_mask, num_modes_ = num_modes, bs0_ = id.bs0_exp, bs1_ = id.bs1_exp;
    }
    SYMGPU_PACKET_HD uint8_t prev_exp() const { return prev_exp_; }  // 0: no previous block
    // A packet that is not audio, names no valid mode or is cut short takes no time and leaves the state alone.
    SYMGPU_PACKET_HD void next(const uint8_t* p, size_t n, uint64_t& dur, uint64_t& discard) {
        const uint8_t exp = vorbis_packet_exp(p, n, num_modes_, mask_, bs0_, bs1_);
        vorbis_packet_time(prev_exp_, exp, dur, discard);
        if (exp) prev_exp_ = exp;
    }

  private:
    uint64_t mask_ = 0;
    uint8_t num_modes_ = 1, bs0_ = 6, bs1_ = 6, prev_exp_ = 0;
};

// symphonia-common/src/xiph/audio/vorbis/mod.rs:66-118: Matroska / WebM carry the three Vorbis headers in one
// Xiph-laced blob (count byte 2, two lacing-coded lengths, then identification, comment and setup back to back).
inline Status vorbis_unpack_xiph_laced(const uint8_t* p, size_t n, Piece& ident, Piece& setup) {
    if (n == 0 || p[0] != 2) return Status::DecodeError;
    size_t at = 1;
    uint64_t len[2] = {0, 0};
    for (int k = 0; k < 2; ++k) {
        for (;;) {
            if (at >= n) return Status::DecodeError;
            const uint8_t v = p[at++];
            len[k] += v;
            if (v < 255) break;
        }
    }
    const uint64_t rest = n - at;
    if (rest == 0 || len[0] + len[1] > rest) return Status::DecodeError;
    ident = Piece{at, uint32_t(len[0])};
    setup = Piece{at + len[0] + len[1], uint32_t(rest - len[0] - len[1])};
    return Status::Ok;
}

// symphonia-format-ogg/src/logical.rs:164-302: end trims of the stream packets of one logical stream, page by page.  A page's
// granule position is the time stamp one past the last valid sample of the last packet that ends on it; a packet whose end
// (the running sum of decoded durations from the page's start) lies beyond that loses the excess, never more than it has left
// after its leading discard.  A page starts where the previous page ended when that page also completed a stream packet (its
// sequence number is the previous one's + 1), otherwise at end - total duration; a stream whose packets all end on one page
// starts at -discard when that leaves padding at the end (the reference's single-page rule, applied here to "every stream
// packet ends on the same page").
SYMGPU_PACKET_HD inline void ogg_page_end_trims(const uint32_t* page_sequence, const uint64_t* page_absgp, const uint32_t* dur, const uint32_t* discard,
                               size_t n, uint32_t* trim_end) {
    bool single_page = true;
    for (size_t i = 1; i < n; ++i) single_page = single_page && page_sequence[i] == page_sequence[0];
    bool have_prev = false;
    uint32_t prev_seq = 0;
    int64_t prev_end = 0;
    for (size_t i = 0; i < n;) {
        size_t j = i;
        int64_t tot = 0, disc = 0;
        while (j < n && page_sequence[j] == page_sequence[i]) tot += dur[j], disc += discard[j], ++j;
        const int64_t page_end = int64_t(page_absgp[i]);
        int64_t start;
        if (have_prev && prev_seq + 1 == page_sequence[i]) start = prev_end;
        else if (single_page && tot >= disc + page_end) start = -disc;
        else start = page_end - tot;
        int64_t next = start;
        for (size_t k = i; k < j; ++k) {
            next += dur[k];
            const int64_t left = int64_t(dur[k]) - int64_t(discard[k]);
            const int64_t over = next - page_end, room = left < 0 ? 0 : left;
            trim_end[k] = next > page_end ? uint32_t(over < room ? over : room) : 0u;
        }
        have_prev = true, prev_seq = page_sequence[i], prev_end = page_end, i = j;
    }
}

// ogg_page_end_trims restated run by run, so that each packet's trim can be computed on its own from prefix sums.  A run is a
// stretch of consecutive packets with equal page_sequence; `end` is its first packet's page_absgp, tot / disc its packets' dur
// / discard summed.  The run's start: the previous run's end when that run's sequence number is one less (uint32, so a wrap
// counts), else -disc when the run is the stream's only run and that leaves padding at the end, else end - tot.
SYMGPU_PACKET_HD inline int64_t ogg_run_start(bool have_prev, uint32_t prev_seq, int64_t prev_end, uint32_t seq, bool only_run, int64_t tot,
                                              int64_t disc, int64_t end) {
    if (have_prev && uint32_t(prev_seq + 1) == seq) return prev_end;
    if (only_run && tot >= disc + end) return -disc;
    return end - tot;
}
// A packet's trim: `next` is its run's start plus the durations of the run's packets up to and including it.
SYMGPU_PACKET_HD inline uint32_t ogg_packet_end_trim(int64_t next, int64_t end, uint32_t dur, uint32_t discard) {
    const int64_t left = int64_t(dur) - int64_t(discard), room = left < 0 ? 0 : left, over = next - end;
    return next > end ? uint32_t(over < room ? over : room) : 0u;
}

// Up to n leading bytes of a packet whose pieces are pieces[0 .. n_pieces) (offsets into d) into out; returns how many exist.
template <class P>
SYMGPU_PACKET_HD inline uint32_t ogg_packet_head(const uint8_t* d, const P* pieces, uint32_t n_pieces, uint8_t* out, uint32_t n) {
    uint32_t got = 0;
    for (uint32_t k = 0; k < n_pieces && got < n; ++k)
        for (uint32_t b = 0; b < pieces[k].len && got < n; ++b) out[got++] = d[pieces[k].offset + b];
    return got;
}

// The Vorbis headers of a file's packet table (packets grouped by serial in ascending order, as symgpu_ogg_index gives them),
// chosen as decode.ogg_vorbis_index chooses them: the stream is the packets of the first packet's serial, [0, n_stream); its
// first packet is the identification header; the setup header is the first later packet of 7 bytes or more that starts with
// 0x05 "vorbis" (n_stream when there is none).  The stream's end is found by bisection and the walk stops at the setup.
struct VorbisStreamHeads {
    uint32_t n_stream, setup;
};
// The chosen stream's packets, [0, n): those of the first packet's serial, found by bisection (0 for an empty table).
template <class Pk>
SYMGPU_PACKET_HD inline uint32_t ogg_first_stream_len(const Pk* packets, uint32_t n_packets) {
    if (n_packets == 0) return 0;
    const uint32_t serial = packets[0].serial;
    uint32_t lo = 1, hi = n_packets;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (packets[mid].serial == serial) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
template <class Pk, class P>
SYMGPU_PACKET_HD inline VorbisStreamHeads vorbis_stream_heads(const uint8_t* d, const Pk* packets, uint32_t n_packets, const P* pieces) {
    VorbisStreamHeads h{0, 0};
    if (n_packets == 0) return h;
    const uint32_t lo = ogg_first_stream_len(packets, n_packets);
    h.n_stream = h.setup = lo;
    for (uint32_t k = 1; k < lo; ++k) {
        uint8_t b[7];
        if (packets[k].len < 7 || ogg_packet_head(d, pieces + packets[k].first_piece, packets[k].n_pieces, b, 7) < 7) continue;
        if (b[0] == 5 && b[1] == 'v' && b[2] == 'o' && b[3] == 'r' && b[4] == 'b' && b[5] == 'i' && b[6] == 's') {
            h.setup = k;
            break;
        }
    }
    return h;
}
// Packet k of the table is an audio packet of the stream: after the setup, inside the stream, not empty, first byte even.
template <class Pk, class P>
SYMGPU_PACKET_HD inline bool vorbis_is_audio(const uint8_t* d, const Pk* packets, const P* pieces, VorbisStreamHeads h, uint32_t k) {
    uint8_t b0 = 1;
    return k > h.setup && k < h.n_stream && packets[k].len > 0 &&
           ogg_packet_head(d, pieces + packets[k].first_piece, packets[k].n_pieces, &b0, 1) == 1 && (b0 & 1) == 0;
}

// mappings/vorbis.rs:109-285: the per-stream state machine.  detect() on the first packet of the first page,
// map() on every later packet.
class OggVorbisMapper {
  public:
    enum class Kind : uint8_t { Audio, Comment, Setup, Unknown, Error };
    struct Mapped {
        Kind kind;
        uint64_t dur, discard;  // Audio only
    };

    // False: not a Vorbis stream (the packet is not a well-formed 30-byte identification header).
    bool detect(const uint8_t* p, size_t n) {
        if (n != 30 || vorbis_read_ident(p, n, ident_) != Status::Ok) return false;
        extra_.assign(p, p + n);
        return true;
    }

    Mapped map(const uint8_t* p, size_t n) {
        Mapped m{Kind::Error, 0, 0};
        if (n == 0) return m;
        if ((p[0] & 1) == 0) {  // even packet types are audio; before the setup header they take no time
            m.kind = Kind::Audio;
            if (have_timer_) timer_.next(p, n, m.dur, m.discard);
            return m;
        }
        if (n < 7 || std::memcmp(p + 1, "vorbis", 6) != 0) return m;
        if (p[0] == 3) return m.kind = Kind::Comment, m;
        if (p[0] != 5) return m.kind = Kind::Unknown, m;
        extra_.insert(extra_.end(), p, p + n);  // appended whether or not it parses, as in the reference
        uint8_t modes;
        uint64_t mask;
        if (vorbis_read_setup_modes(p, n, ident_, modes, mask) == Status::Ok) timer_ = VorbisPacketTimer(ident_, modes, mask), have_timer_ = true;
        ready_ = true;
        return m.kind = Kind::Setup, m;
    }

    void reset() { timer_.reset(); }
    bool ready() const { return ready_; }  // a setup header was seen
    const VorbisIdent& ident() const { return ident_; }
    // Identification packet + setup packet(s): what the decoder is constructed from.
    const std::vector<uint8_t>& extra_data() const { return extra_; }
    // Largest gap between points a decoder can start from: half the long block (:156-164).
    uint64_t max_rap_period() const { return have_timer_ ? (uint64_t(1) << ident_.bs1_exp) >> 1 : 0; }

  private:
    VorbisIdent ident_{};
    VorbisPacketTimer timer_;
    std::vector<uint8_t> extra_;
    bool have_timer_ = false, ready_ = false;
};

// =====================================================================================================================
// FLAC (native container)
// =====================================================================================================================
// "fLaC", metadata blocks (STREAMINFO first), then frames back to back.  A frame carries no length: its end is where
// the next frame starts, and the only proof of that is the CRC-16 in front of it.  The reference finds packets with a
// fragment-merging parser driven by moving averages of the frame size (symphonia-bundle-flac/src/parser.rs:149-560);
// this is a plain CRC-validated splitter instead: a frame starts at a sync code whose header parses, checks out (CRC-8)
// and fits the stream (parser.rs:586-648: rate, bit depth, channel count, block size, blocking strategy, monotonic
// sequence number), and ends at the first later such header -- or the end of the data -- in front of which the CRC-16
// of everything since the start matches.  On a well-formed file both give the same packets, time stamps and durations;
// on a damaged one this splitter drops exactly the frames whose checksum fails, which is not promised to be what the
// reference's heuristics do (DESIGN §5b).

struct FlacStreamInfo {  // symphonia-common/src/xiph/audio/flac/mod.rs:78-186
    uint16_t block_min, block_max;
    uint32_t frame_min, frame_max;  // bytes, 0 = unknown
    uint32_t sample_rate;
    uint8_t channels, bits_per_sample;
    uint64_t n_samples;             // 0 = unknown
    uint8_t md5[16];
    bool has_md5;
};

// The FLAC rules below are host / device functions: FlacIndexer (symgpu_flac_index) and the device index (symgpu_flac_index_dev,
// flac_index_kernel.cu) run this very code.  No memcmp / memchr and no double arithmetic in them.
SYMGPU_PACKET_HD inline Status flac_read_stream_info(const uint8_t* p, size_t n, FlacStreamInfo& si) {
    if (n < 34) return Status::EndOfStream;
    si.block_min = uint16_t(detail::be16(p)), si.block_max = uint16_t(detail::be16(p + 2));
    if (si.block_min < 16 || si.block_max < 16 || si.block_max < si.block_min) return Status::DecodeError;
    si.frame_min = detail::be24(p + 4), si.frame_max = detail::be24(p + 7);
    if (si.frame_min && si.frame_max && si.frame_max < si.frame_min) return Status::DecodeError;
    const uint64_t bits = uint64_t(detail::be32(p + 10)) << 32 | detail::be32(p + 14);  // 20 + 3 + 5 + 36 bits
    si.sample_rate = uint32_t(bits >> 44);
    if (si.sample_rate < 1 || si.sample_rate > 655350) return Status::DecodeError;
    si.channels = uint8_t(((bits >> 41) & 7) + 1);
    si.bits_per_sample = uint8_t(((bits >> 36) & 31) + 1);
    if (si.bits_per_sample < 4) return Status::DecodeError;
    si.n_samples = bits & 0xfffffffffull;
    si.has_md5 = false;
    for (int k = 0; k < 16; ++k) si.md5[k] = p[18 + k], si.has_md5 |= p[18 + k] != 0;
    return Status::Ok;
}

// demuxer.rs:60-170: the stream marker, then metadata blocks up to the one flagged last; the first must be STREAMINFO.  On Ok,
// *first_frame is where the frames begin.  A walk over the block headers, one thread per file on the device.
SYMGPU_PACKET_HD inline Status flac_open(const uint8_t* d, size_t n, FlacStreamInfo& info, size_t* first_frame) {
    if (n < 4 || d[0] != 'f' || d[1] != 'L' || d[2] != 'a' || d[3] != 'C') return Status::Unsupported;
    size_t at = 4;
    bool first = true;
    for (;;) {
        if (at + 4 > n) return Status::EndOfStream;
        const bool last = d[at] & 0x80;
        const unsigned type = d[at] & 0x7f;
        const size_t len = detail::be24(d + at + 1);
        at += 4;
        if (at + len > n) return Status::EndOfStream;
        if (first) {
            if (type != 0 || len != 34) return Status::DecodeError;
            const Status s = flac_read_stream_info(d + at, len, info);
            if (s != Status::Ok) return s;
            first = false;
        }
        at += len;
        if (last) break;
    }
    *first_frame = at;
    return Status::Ok;
}

SYMGPU_PACKET_HD inline uint8_t crc8_ccitt(const uint8_t* p, size_t n) {  // polynomial 0x07 (symphonia-core/src/checksum/crc8.rs:32-65)
    uint8_t c = 0;
    for (size_t i = 0; i < n; ++i) {
        c ^= p[i];
        for (int k = 0; k < 8; ++k) c = uint8_t(c & 0x80 ? (c << 1) ^ 0x07 : c << 1);
    }
    return c;
}
namespace detail {
struct Crc16Msb {
    uint16_t t[256];
    constexpr Crc16Msb() : t() {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i << 8;
            for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? (c << 1) ^ 0x8005 : c << 1;
            t[i] = uint16_t(c);
        }
    }
};
}  // namespace detail
// CRC-16, polynomial 0x8005, most-significant bit first, init 0, no final xor (the FLAC frame footer).  `t` is
// detail::Crc16Msb::t: the device keeps its copy in constant memory.
SYMGPU_PACKET_HD inline uint16_t crc16_ansi_update_with(const uint16_t* t, uint16_t state, const uint8_t* p, size_t n) {
    for (size_t i = 0; i < n; ++i) state = uint16_t((state << 8) ^ t[(state >> 8) ^ p[i]]);
    return state;
}
inline const uint16_t* crc16_ansi_table() {
    static constexpr detail::Crc16Msb tab{};
    return tab.t;
}
inline uint16_t crc16_ansi_update(uint16_t state, const uint8_t* p, size_t n) { return crc16_ansi_update_with(crc16_ansi_table(), state, p, n); }

// The CRC-16 state as an element of GF(2)[x] / (x^16 + x^15 + x^2 + 1): a zero byte multiplies it by x^8, so the state of A || B is
// crc(A) x^(8 |B|) + crc(B).  a x b in that ring:
SYMGPU_PACKET_HD inline uint16_t crc16_mulmod(uint16_t a, uint16_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 16; ++i)
        if ((b >> i) & 1) p ^= uint32_t(a) << i;
    for (int i = 30; i >= 16; --i)
        if ((p >> i) & 1) p ^= 0x18005u << (i - 16);
    return uint16_t(p);
}
// x^(8 k): what k zero bytes multiply a state by.
SYMGPU_PACKET_HD inline uint16_t crc16_xpow8(uint64_t k) {
    uint16_t r = 1, base = 0x100;
    for (; k; k >>= 1, base = crc16_mulmod(base, base))
        if (k & 1) r = crc16_mulmod(r, base);
    return r;
}
// (a, la) o (b, lb) = (x^(8 lb) a + b, la + lb): the state of two spans one after the other, from their states alone.
SYMGPU_PACKET_HD inline uint16_t crc16_combine(uint16_t a, uint16_t b, uint64_t lb) { return uint16_t(crc16_mulmod(a, crc16_xpow8(lb)) ^ b); }

struct FlacFrameHeader {
    uint64_t sequence;
    bool by_sample;
    uint32_t block, sample_rate, bits_per_sample;  // rate / depth 0: not in the header
    uint8_t channels;
    uint8_t size;  // bytes, sync code to CRC-8
};

namespace detail {
SYMGPU_PACKET_HD inline uint32_t flac_rate_code(unsigned sr) {  // codes 0-11
    switch (sr) {
        case 1: return 88200;
        case 2: return 176400;
        case 3: return 192000;
        case 4: return 8000;
        case 5: return 16000;
        case 6: return 22050;
        case 7: return 24000;
        case 8: return 32000;
        case 9: return 44100;
        case 10: return 48000;
        case 11: return 96000;
        default: return 0;
    }
}
SYMGPU_PACKET_HD inline uint32_t flac_depth_code(unsigned bd) {  // 255: reserved
    switch (bd) {
        case 1: return 8;
        case 2: return 12;
        case 3: return 255;
        case 4: return 16;
        case 5: return 20;
        case 6: return 24;
        case 7: return 32;
        default: return 0;
    }
}
}  // namespace detail

// frame.rs:81-233 at p[0..n): false unless a complete header with a matching CRC-8 starts here.
SYMGPU_PACKET_HD inline bool flac_parse_frame_header(const uint8_t* p, size_t n, FlacFrameHeader& h) {
    if (n < 6 || p[0] != 0xff || (p[1] & 0xfc) != 0xf8 || (p[3] & 1)) return false;
    size_t at = 4;
    h.by_sample = p[1] & 1;
    const unsigned bs = p[2] >> 4, sr = p[2] & 15, ch = p[3] >> 4, bd = (p[3] >> 1) & 7;
    uint64_t v = p[at++];
    int more;
    if (v < 0x80) more = 0;
    else if (v >= 0xc0 && v <= 0xdf) more = 1, v &= 0x1f;
    else if (v >= 0xe0 && v <= 0xef) more = 2, v &= 0x0f;
    else if (v >= 0xf0 && v <= 0xf7) more = 3, v &= 0x07;
    else if (v >= 0xf8 && v <= 0xfb) more = 4, v &= 0x03;
    else if (v >= 0xfc && v <= 0xfd) more = 5, v &= 0x01;
    else if (v == 0xfe) more = 6, v = 0;
    else return false;
    for (int k = 0; k < more; ++k) {
        if (at >= n) return false;
        v = v << 6 | (p[at++] & 0x3f);
    }
    if (v > (h.by_sample ? 0xfffffffffull : 0x7fffffffull)) return false;
    h.sequence = v;
    if (bs == 0) return false;
    if (bs == 1) h.block = 192;
    else if (bs <= 5) h.block = 576u << (bs - 2);
    else if (bs == 6) {
        if (at + 1 > n) return false;
        h.block = uint32_t(p[at++]) + 1;
    } else if (bs == 7) {
        if (at + 2 > n) return false;
        const uint32_t x = detail::be16(p + at);
        at += 2;
        if (x == 0xffff) return false;
        h.block = x + 1;
    } else h.block = 256u << (bs - 8);
    if (sr < 12) h.sample_rate = detail::flac_rate_code(sr);
    else if (sr == 12) {
        if (at + 1 > n) return false;
        h.sample_rate = uint32_t(p[at++]) * 1000;
    } else if (sr == 15) return false;
    else {
        if (at + 2 > n) return false;
        h.sample_rate = detail::be16(p + at) * (sr == 14 ? 10u : 1u);
        at += 2;
    }
    if (sr != 0 && (h.sample_rate < 1 || h.sample_rate > 655350)) return false;
    if (detail::flac_depth_code(bd) == 255) return false;
    h.bits_per_sample = detail::flac_depth_code(bd);
    if (ch <= 7) h.channels = uint8_t(ch + 1);
    else if (ch <= 10) h.channels = 2;
    else return false;
    if (at + 1 > n || p[at] != crc8_ccitt(p, at)) return false;
    h.size = uint8_t(at + 1);
    return true;
}

// parser.rs:586-648, the header against the stream: rate, depth, block size, channel count and blocking strategy.
SYMGPU_PACKET_HD inline bool flac_fits_stream(const FlacFrameHeader& h, const FlacStreamInfo& info) {
    if (h.sample_rate && h.sample_rate != info.sample_rate) return false;
    if (h.bits_per_sample && h.bits_per_sample != info.bits_per_sample) return false;
    if (h.block > info.block_max || h.channels != info.channels) return false;
    const bool fixed = info.block_min == info.block_max;
    return h.by_sample != fixed;
}
// A plausible frame start at d[q ..] of a file of n bytes: a header that parses, checks out and fits the stream.
SYMGPU_PACKET_HD inline bool flac_plausible(const uint8_t* d, size_t n, size_t q, const FlacStreamInfo& info, FlacFrameHeader& h) {
    return q + 6 <= n && flac_parse_frame_header(d + q, n - q, h) && flac_fits_stream(h, info);
}
// The sequence rule: a header follows a frame numbered last_seq when its number is larger, or 0.
SYMGPU_PACKET_HD inline bool flac_follows(uint64_t seq, uint64_t last_seq) { return seq > last_seq || seq == 0; }
// v(h): the number the sequence rule compares, with 0 (which follows everything) as the largest.
SYMGPU_PACKET_HD inline uint64_t flac_value(uint64_t seq) { return seq == 0 ? ~uint64_t(0) : seq; }

// parser.rs:566-584: the frame's first sample.
SYMGPU_PACKET_HD inline uint64_t flac_packet_ts(const FlacFrameHeader& h, const FlacStreamInfo& info) {
    const bool fixed = info.block_min == info.block_max;
    return h.by_sample ? h.sequence : h.sequence * (fixed ? info.block_min : h.block);
}

// ---- FLAC in Ogg (symphonia-format-ogg/src/mappings/flac.rs): the rules of the host index (decode.ogg_flac_index through
// symgpu_ogg_flac_packets) and of the device job build (ogg_flac_jobs_kernel.cu), on a stream chosen as the Vorbis rules choose it
// (ogg_first_stream_len).  The mapper's own frame-header parse only times packets; the decoder takes STREAMINFO as its extra data
// and decodes every audio packet with flac_entropy.h's rules, applying no Ogg trim.
constexpr uint32_t kOggFlacIdentLen = 51;
// flac.rs:43-125 on the stream's first packet: exactly 51 bytes of 0x7f "FLAC", major version 1 (minor version and header count
// ignored), "fLaC", a metadata block header of type STREAMINFO (the last-block flag ignored) and length 34, and the block.
// Unsupported: not Ogg FLAC (detect() gives no mapper).  Otherwise what flac_read_stream_info gives for the block: an Ogg FLAC
// stream whose STREAMINFO is refused is DecodeError, as detect() fails then.
SYMGPU_PACKET_HD inline Status ogg_flac_ident(const uint8_t* p, size_t n, FlacStreamInfo& si) {
    if (n != kOggFlacIdentLen || p[0] != 0x7f || p[1] != 'F' || p[2] != 'L' || p[3] != 'A' || p[4] != 'C' || p[5] != 1) return Status::Unsupported;
    if (p[9] != 'f' || p[10] != 'L' || p[11] != 'a' || p[12] != 'C') return Status::Unsupported;
    if ((p[13] & 0x7f) != 0 || detail::be24(p + 14) != 34) return Status::Unsupported;
    return flac_read_stream_info(p + 17, 34, si);
}
// flac.rs:299-345: a packet is audio when its first byte is 0xff; 0x00 / 0x80 and metadata blocks (any other first byte) are not.
SYMGPU_PACKET_HD inline bool ogg_flac_is_audio(uint32_t len, uint8_t first) { return len > 0 && first == 0xff; }
// The most bytes a frame header takes, sync code to CRC-8: 4 + a 7-byte sequence number + 2 (block) + 2 (rate) + 1.
constexpr uint32_t kFlacMaxHeader = 16;
// The block size of a packet as the decoder reads it (flac_entropy.h decode_packet: the first sync code of the packet, then
// read_frame_header, whose rules flac_parse_frame_header restates); 0 where there is no sync code or the decoder refuses the
// header.  The packet is pieces[0 .. n_pieces) of d.  This is the job's slot: a packet with slot 0 is refused.
template <class P>
SYMGPU_PACKET_HD inline uint32_t ogg_flac_packet_block(const uint8_t* d, const P* pieces, uint32_t n_pieces) {
    uint8_t h[kFlacMaxHeader];
    uint32_t got = 0;
    bool prev_ff = false;
    for (uint32_t k = 0; k < n_pieces && got < kFlacMaxHeader; ++k)
        for (uint64_t b = 0; b < pieces[k].len && got < kFlacMaxHeader; ++b) {
            const uint8_t x = d[pieces[k].offset + b];
            if (got) h[got++] = x;
            else if (prev_ff && (x & 0xfc) == 0xf8) h[0] = 0xff, h[1] = x, got = 2;
            else prev_ff = x == 0xff;
        }
    FlacFrameHeader fh;
    return got && flac_parse_frame_header(h, got, fh) ? fh.block : 0;
}

constexpr size_t kFlacMaxFrame = 16u * 1024 * 1024;  // frame.rs:17: how far past its start a frame's end is looked for
// The smallest frame: a 6-byte header and the 2-byte CRC-16, so a file of n bytes holds at most n / 8 packets.
constexpr uint32_t kFlacMinFrame = 8;

struct FlacPacket {
    uint64_t offset;
    uint32_t size;
    uint64_t ts;   // first sample (parser.rs:566-584)
    uint32_t dur;  // block size
};

// ---- the splitter as a chain: shared by FlacIndexer and the device index (symgpu_flac_index_dev) -------------------------------
// FlacIndexer::next is sequential, but what it returns is a function of each frame start alone (DESIGN §5b).  The files of a
// device call lie back to back in one virtual byte space; its nodes, in position order, are
//   * every sync position q of a file (q + 2 <= n, d[q] = 0xff, d[q + 1] & 0xfc = 0xf8), and
//   * one end node per non-empty file, stored at its last byte q = n - 1 (never a sync position) and standing for position n.
// A node is named by its 32-bit index in that order; npos is the file position it stands for.
SYMGPU_PACKET_HD inline bool flac_is_sync(const uint8_t* d, size_t n, size_t q) { return q + 2 <= n && d[q] == 0xff && (d[q + 1] & 0xfc) == 0xf8; }
constexpr uint32_t kFlacEndNode = 1;  // the node word of an end node (0: a sync position)
SYMGPU_PACKET_HD inline bool flac_is_node(const uint8_t* d, size_t n, size_t q) { return q + 1 == n || flac_is_sync(d, n, q); }
SYMGPU_PACKET_HD inline uint32_t flac_node(size_t n, size_t q) { return q + 1 == n ? kFlacEndNode : 0; }
SYMGPU_PACKET_HD inline uint64_t flac_npos(const uint64_t* vpos, const uint32_t* node, uint32_t c, uint64_t vbase) {
    return vpos[c] - vbase + (node[c] & kFlacEndNode);
}
constexpr uint32_t kFlacNone = 0xffffffffu;

// The first node of [lo, hi) (one file's, starting at vbase) whose npos is at least x >= 1; hi when there is none.
SYMGPU_PACKET_HD inline uint32_t flac_first_node_at(const uint64_t* vpos, const uint32_t* node, uint32_t lo, uint32_t hi, uint64_t vbase, uint64_t x) {
    uint32_t i = detail::first_at_or_after(vpos, lo, hi, vbase + x - 1);
    if (i < hi && !(node[i] & kFlacEndNode) && vpos[i] == vbase + x - 1) ++i;  // a sync position at x - 1 stands for itself
    return i;
}

// 1. The CRC key.  key(x) = the CRC-16 state of file bytes [0, x), continued over n - x zero bytes.  With init 0 and no final xor,
//    appending a frame's big-endian CRC-16 brings the state to 0, so crc16[s, q - 2) == be16(q - 2) exactly when
//    key(s) == key(q).  key(x) is the xor of x^(8 (n - 1 - p)) crc(byte p) over p < x: an exclusive xor-scan.  A span [a, b) of
//    the file contributes flac_key_part; a position q inside a span that began with prefix `pre` and has CRC state s over [a, q)
//    has key pre ^ flac_key_inside.
SYMGPU_PACKET_HD inline uint16_t flac_key_part(const uint16_t* t, const uint8_t* d, size_t n, size_t a, size_t b) {
    return crc16_mulmod(crc16_ansi_update_with(t, 0, d + a, b - a), crc16_xpow8(n - b));
}
SYMGPU_PACKET_HD inline uint16_t flac_key_inside(uint16_t s, size_t n, size_t q) { return crc16_mulmod(s, crc16_xpow8(n - q)); }

// 2. The search trees: a max tree over a table of values v[0 .. n) (level 0), level k holding the maxima of aligned runs of 2^k.
//    flac_tree_levels(L) levels above level 0 make every query over one file of at most L bytes logarithmic: a file has at most
//    L / 2 + 1 nodes.
struct FlacTree {
    const uint64_t* level[34];
    uint32_t n, top;
};
SYMGPU_PACKET_HD inline uint32_t flac_tree_levels(uint64_t max_len) {
    uint32_t k = 0;
    for (uint64_t m = max_len / 2; m; m >>= 1) ++k;
    return k;
}
SYMGPU_PACKET_HD inline uint64_t flac_tree_max(const uint64_t* below, uint64_t n_below, uint64_t j) {
    const uint64_t a = below[2 * j], b = 2 * j + 1 < n_below ? below[2 * j + 1] : 0;
    return a > b ? a : b;
}
// The first i of [a, b] with v[i] > thr, kFlacNone when there is none: up the tree past runs at most thr, then down into the first
// run above it.  b - a < 2^top.
SYMGPU_PACKET_HD inline uint32_t flac_first_above(const FlacTree& t, uint32_t a, uint32_t b, uint64_t thr) {
    uint64_t i = a;
    uint32_t k = 0;
    while (i <= b && i < t.n) {  // nothing of [a, i) is above thr, and 2^k divides i
        if (t.level[k][i >> k] > thr) {
            while (k > 0) {
                --k;
                if (t.level[k][i >> k] <= thr) i += uint64_t(1) << k;
            }
            return i <= b ? uint32_t(i) : kFlacNone;
        }
        i += uint64_t(1) << k;
        if (k < t.top && !((i >> k) & 1)) ++k;
    }
    return kFlacNone;
}

// 3. Each node's values.  A node is plausible when it is a sync position at or after the first frame of a file that opened, whose
//    header flac_plausible accepts; ev (the end search's table) is flac_value of a plausible node, ~0 for an end node and 0 for the
//    rest.
struct FlacHead {
    uint64_t seq;
    uint32_t block;
    uint8_t size, by_sample, plausible, reserved;
};
SYMGPU_PACKET_HD inline FlacHead flac_head(const uint8_t* d, size_t n, size_t q, uint32_t node, bool opened, size_t first_frame,
                                           const FlacStreamInfo& info) {
    FlacHead r{};
    FlacFrameHeader h;
    if (!(node & kFlacEndNode) && opened && q >= first_frame && flac_plausible(d, n, q, info, h))
        r.seq = h.sequence, r.block = h.block, r.size = h.size, r.by_sample = h.by_sample, r.plausible = 1;
    return r;
}
SYMGPU_PACKET_HD inline uint64_t flac_end_value(const FlacHead& h, uint32_t node) {
    return (node & kFlacEndNode) ? ~uint64_t(0) : h.plausible ? flac_value(h.seq) : 0;
}

// 4. end(s) of the plausible node c at file position q (its file's nodes [c, c1), the last its end node): the first node of the
//    window with c's key, at least size + 2 bytes on, that is the end node or follows c.  The window is FlacIndexer::next's
//    kMaxFrame rule: the sync positions up to and including the first one past q + kFlacMaxFrame, and the end node only when no
//    sync position lies past it.  The nodes with one key lie together in (skey, sid), sorted by key and, within a key, by node;
//    the tree is over their ev.  Returns the end node, kFlacNone when there is none.
SYMGPU_PACKET_HD inline uint32_t flac_key_lower(const uint32_t* skey, const uint32_t* sid, uint32_t n, uint32_t key, uint32_t id) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (skey[mid] < key || (skey[mid] == key && sid[mid] < id)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
SYMGPU_PACKET_HD inline uint32_t flac_end(const uint64_t* vpos, const uint32_t* node, uint32_t c, uint32_t c1, uint64_t vbase, const FlacHead& h,
                                          uint32_t key, const uint32_t* skey, const uint32_t* sid, const FlacTree& tree) {
    const uint64_t q = vpos[c] - vbase;
    const uint32_t lo = flac_first_node_at(vpos, node, c + 1, c1, vbase, q + h.size + 2);
    const uint32_t cut = flac_first_node_at(vpos, node, c + 1, c1, vbase, q + kFlacMaxFrame + 1);
    const uint32_t hi = cut < c1 ? cut : c1 - 1;
    if (lo > hi) return kFlacNone;
    const uint32_t a = flac_key_lower(skey, sid, tree.n, key, lo), e = flac_key_lower(skey, sid, tree.n, key, hi + 1);
    if (a >= e) return kFlacNone;
    const uint32_t i = flac_first_above(tree, a, e - 1, h.seq);
    return i == kFlacNone ? kFlacNone : sid[i];
}

// 5. good(c) = plausible with an end; the next frame's table gv is flac_value of a good node, 0 for the rest.  After the frame c
//    (ending at its end node e) the next frame is the first good node of [e, c1) that follows c -- none (kAdtsEnd) when e is the
//    end node.  A file's first frame is the first good node at or after its first frame position.  The successors form one chain
//    per file, ranked by adts_double.
SYMGPU_PACKET_HD inline uint32_t flac_successor(const uint32_t* node, uint32_t e, uint32_t c1, uint64_t seq, const FlacTree& good) {
    if (e == kFlacNone || (node[e] & kFlacEndNode)) return kFlacNone;
    return flac_first_above(good, e, c1 - 1, seq);
}
SYMGPU_PACKET_HD inline uint32_t flac_first_frame(const uint64_t* vpos, const uint32_t* node, uint32_t c0, uint32_t c1, uint64_t vbase,
                                                  size_t first_frame, const FlacTree& good) {
    const uint32_t a = flac_first_node_at(vpos, node, c0, c1, vbase, first_frame);
    return a < c1 ? flac_first_above(good, a, c1 - 1, 0) : kFlacNone;
}
// The rounds that rank every chain of files of at most max_len bytes: a frame is at least 8 bytes.
SYMGPU_PACKET_HD inline uint32_t flac_chain_rounds(uint64_t max_len) {
    uint32_t k = 0;
    for (uint64_t m = max_len / kFlacMinFrame; m; m >>= 1) ++k;
    return k;
}

// 6. The packet of the chain node c at q, ending at file position end.
SYMGPU_PACKET_HD inline FlacPacket flac_chain_packet(uint64_t q, uint64_t end, const FlacHead& h, const FlacStreamInfo& info) {
    FlacFrameHeader fh{};
    fh.sequence = h.seq, fh.by_sample = h.by_sample, fh.block = h.block;
    FlacPacket p;
    p.offset = q, p.size = uint32_t(end - q), p.dur = h.block, p.ts = flac_packet_ts(fh, info);
    return p;
}

class FlacIndexer {
  public:
    FlacIndexer(const uint8_t* data, size_t n) : d_(data), n_(n) {}

    Status open() {
        const Status s = flac_open(d_, n_, info_, &first_frame_);
        if (s != Status::Ok) return s;
        pos_ = first_frame_;
        have_last_ = false;
        return Status::Ok;
    }
    const FlacStreamInfo& info() const { return info_; }
    size_t first_frame_pos() const { return first_frame_; }
    size_t skipped_bytes() const { return skipped_; }  // bytes between packets that belonged to no valid frame

    Status next(FlacPacket& pk) {
        for (size_t start = pos_; start + 2 <= n_;) {
            FlacFrameHeader h;
            if (!candidate(start, h)) {
                const size_t q = next_sync(start + 1);
                skipped_ += q - start;
                start = pos_ = q;
                continue;
            }
            // the end: the next plausible header (or the end of the data) that the CRC-16 vouches for
            uint16_t crc = 0;
            size_t done = start;  // crc covers [start, done)
            for (size_t q = next_sync(start + h.size);; q = next_sync(q + 1)) {
                FlacFrameHeader nh;
                const bool at_end = q >= n_;
                if (at_end) q = n_;
                if (q - start >= 2 + size_t(h.size) && (at_end || candidate(q, nh, &h))) {
                    crc = crc16_ansi_update(crc, d_ + done, q - 2 - done), done = q - 2;
                    if (crc == detail::be16(d_ + q - 2)) {
                        pk.offset = start, pk.size = uint32_t(q - start), pk.dur = h.block;
                        pk.ts = flac_packet_ts(h, info_);
                        last_ = h, have_last_ = true, pos_ = q;
                        return Status::Ok;
                    }
                }
                if (at_end || q - start > kFlacMaxFrame) break;
            }
            const size_t q = next_sync(start + 1);  // no end vouched for: this was not a frame
            skipped_ += q - start;
            start = pos_ = q;
        }
        return Status::EndOfStream;
    }

    static Status index(const uint8_t* data, size_t n, FlacStreamInfo& info, std::vector<FlacPacket>& out) {
        FlacIndexer ix(data, n);
        const Status s = ix.open();
        if (s != Status::Ok) return s;
        info = ix.info();
        FlacPacket p;
        while (ix.next(p) == Status::Ok) out.push_back(p);
        return Status::Ok;
    }

  private:
    size_t next_sync(size_t from) const {
        for (size_t q = from; q + 2 <= n_;) {
            const void* hit = std::memchr(d_ + q, 0xff, n_ - q);  // (host only: the device visits every byte once in its tiles)
            if (!hit) break;
            q = size_t(static_cast<const uint8_t*>(hit) - d_);
            if (flac_is_sync(d_, n_, q)) return q;
            if (q + 2 > n_) break;
            ++q;
        }
        return n_;
    }
    // A header at `at` that fits the stream and follows `prev` (default: the last accepted frame).
    bool candidate(size_t at, FlacFrameHeader& h, const FlacFrameHeader* prev = nullptr) const {
        if (!flac_plausible(d_, n_, at, info_, h)) return false;
        const FlacFrameHeader* before = prev ? prev : (have_last_ ? &last_ : nullptr);
        return flac_follows(h.sequence, before ? before->sequence : 0);
    }

    const uint8_t* d_;
    size_t n_;
    size_t pos_ = 0, first_frame_ = 0, skipped_ = 0;
    FlacStreamInfo info_{};
    FlacFrameHeader last_{};
    bool have_last_ = false;
};

// ---- CAF holding ALAC (symphonia-format-caf/src/demuxer.rs:362-560, chunks.rs:82-614; the magic cookie of
// symphonia-common/src/apple/audio/alac.rs:34-171 and symphonia-codec-alac/src/lib.rs:295-300) -----------------------------
// caf_open walks the chunks as CafReader::read_chunks does and reads the magic cookie as AlacDecoder::try_new does; the
// packet table's integers are then read by caf_varint, serially (CafIndexer) or one integer per thread (the device index).
// The host and device indexes run these functions, so their records are equal by construction.

// Why a file does not open (SYMGPU_CAF_* in include/symgpu.h).
enum CafReason : uint8_t {
    kCafOk = 0,
    kCafTruncated = 1,   // a header, chunk or the packet table runs past the end of the file
    kCafNotCaf = 2,      // no "caff" marker
    kCafVersion = 3,     // file version other than 1
    kCafBadChunk = 4,    // a chunk size the reader refuses, or a second desc chunk
    kCafNoDesc = 5,      // the first chunk is not desc
    kCafBadDesc = 6,     // zero sample rate or channel count, or more channels than positions
    kCafNotAlac = 7,     // a format other than ALAC
    kCafLayout = 8,      // ALAC without variable bytes and constant frames per packet
    kCafBadTable = 9,    // negative counts, or an integer of more than 9 bytes
    kCafNoCookie = 10,   // no kuki chunk
    kCafBadCookie = 11,  // the magic cookie breaks a rule of MagicCookie::read, or its frame length exceeds 65 536
};

struct CafAlac {  // what a CAF file holding ALAC says once opened
    uint64_t data_start = 0;    // the first packet's byte: the audio of a sized data chunk, else the end of the file
    uint64_t table_at = 0;      // the last pakt chunk's first integer
    uint64_t table_packets = 0; // and its packet count
    uint64_t table_bytes = 0;   // and the bytes its integers take
    int64_t valid_frames = 0;
    int32_t priming_frames = 0, remainder_frames = 0;
    uint32_t frames_per_packet = 0;
    uint32_t frame_length = 0, max_frame_bytes = 0, avg_bit_rate = 0, sample_rate = 0;
    uint16_t max_run = 0;
    uint8_t compatible_version = 0, bit_depth = 0, pb = 0, mb = 0, kb = 0, channels = 0;
    uint8_t reason = kCafOk;
};

constexpr uint32_t kCaf_alac = detail::tag4("alac"), kCaf_caff = detail::tag4("caff"), kCaf_chan = detail::tag4("chan"), kCaf_data = detail::tag4("data"), kCaf_desc = detail::tag4("desc"), kCaf_frma = detail::tag4("frma"), kCaf_kuki = detail::tag4("kuki"), kCaf_pakt = detail::tag4("pakt");

namespace detail {
SYMGPU_PACKET_HD inline uint64_t be64(const uint8_t* p) { return uint64_t(be32(p)) << 32 | be32(p + 4); }
}  // namespace detail

// read_variable_length_integer (chunks.rs:599-615): 7 bits per byte, most significant first, a clear top bit ends it, at most 9
// bytes.  Status::EndOfStream when the bytes end first (the reference's read_byte fails), DecodeError when the ninth byte does
// not end it.
SYMGPU_PACKET_HD inline Status caf_varint(const uint8_t* d, size_t n, uint64_t& at, uint64_t& v) {
    v = 0;
    for (int k = 0; k < 9; ++k) {
        if (at >= n) return Status::EndOfStream;
        const uint8_t byte = d[at++];
        v |= byte & 0x7f;
        if (!(byte & 0x80)) return Status::Ok;
        v <<= 7;
    }
    return Status::DecodeError;
}

// The format ids AudioDescriptionFormatId::read knows (chunks.rs:282-311); any other fails the file.
SYMGPU_PACKET_HD inline bool caf_known_format(uint32_t f) {
    const uint32_t known[15] = {0x6c70636du /* lpcm */, 0x696d6134u /* ima4 */, 0x61616320u /* "aac " */, 0x4d414333u /* MAC3 */,
                                0x4d414336u /* MAC6 */, 0x756c6177u /* ulaw */, 0x616c6177u /* alaw */, 0x2e6d7031u /* .mp1 */,
                                0x2e6d7032u /* .mp2 */, 0x2e6d7033u /* .mp3 */, kCaf_alac, 0x666c6163u /* flac */, 0x6f707573u /* opus */, 0, 0};
    for (int k = 0; k < 13; ++k)
        if (f == known[k]) return true;
    return false;
}

// MagicCookie::read (alac.rs:34-171) and the frame-length limit of AlacDecoder::try_new (lib.rs:295-300).
SYMGPU_PACKET_HD inline Status caf_alac_cookie(const uint8_t* c, uint64_t len, CafAlac& a) {
    using detail::be16;
    using detail::be32;
    a.reason = kCafBadCookie;
    if (len < 24) return Status::Unsupported;
    if (be32(c + 4) == kCaf_frma) c += 12, len -= 12;
    if (be32(c + 4) == kCaf_alac) c += 12, len -= 12;
    if (len != 24 && len != 48) return Status::Unsupported;
    a.frame_length = be32(c), a.compatible_version = c[4], a.bit_depth = c[5], a.pb = c[6], a.mb = c[7], a.kb = c[8], a.channels = c[9];
    a.max_run = uint16_t(be16(c + 10)), a.max_frame_bytes = be32(c + 12), a.avg_bit_rate = be32(c + 16), a.sample_rate = be32(c + 20);
    if (a.compatible_version > 0) return Status::Unsupported;
    if (a.bit_depth > 32 || a.channels < 1 || a.channels > 8) return Status::DecodeError;
    if (len == 48) {
        const uint8_t* l = c + 24;
        if (be32(l) != 24 || be32(l + 4) != kCaf_chan || be32(l + 8) != 0) return Status::DecodeError;
        // the eight layout tags and their channel counts: (100..127, 142) << 16 | count
        const uint32_t tag = be32(l + 12), count = tag & 0xffff;
        const uint32_t tags[8] = {100, 101, 113, 116, 120, 124, 142, 127};
        if (count < 1 || count > 8 || (tag >> 16) != tags[count - 1]) return Status::DecodeError;
        if (count != a.channels) return Status::DecodeError;
        if (be32(l + 16) != 0 || be32(l + 20) != 0) return Status::DecodeError;
    }
    if (a.frame_length > 4096 * 16) return Status::Unsupported;
    a.reason = kCafOk;
    return Status::Ok;
}

// CafReader::check_file_header + read_chunks (demuxer.rs:362-560) with Chunk::read (chunks.rs:82-128) and each chunk's reader,
// then the cookie.  The walk ends only where a chunk ends exactly at the end of the file, as the reference's does; after a data
// chunk of size -1 the bytes that follow are read as chunks too.  The reader continues after a pakt chunk where its last
// integer ends and after a chan chunk where its last description ends, whatever their declared sizes say.  Only ALAC with
// variable bytes and constant frames per packet is taken, the layout every ALAC encoder writes.
SYMGPU_PACKET_HD inline Status caf_open(const uint8_t* d, uint64_t n, CafAlac& a) {
    using detail::be32;
    using detail::be64;
    a = CafAlac{};
    auto fail = [&](Status s, uint8_t why) {
        a.reason = why;
        return s;
    };
    if (n < 4) return fail(Status::EndOfStream, kCafTruncated);
    if (be32(d) != kCaf_caff) return fail(Status::Unsupported, kCafNotCaf);
    if (n < 8) return fail(Status::EndOfStream, kCafTruncated);
    if (detail::be16(d + 4) != 1) return fail(Status::Unsupported, kCafVersion);
    bool have_desc = false, have_cookie = false, sized_data = false;
    uint64_t cookie_at = 0, cookie_len = 0, at = 8;
    for (;;) {
        if (n - at < 12) return fail(Status::EndOfStream, kCafTruncated);
        const uint32_t type = be32(d + at);
        const int64_t size = int64_t(be64(d + at + 4));
        const uint64_t body = at + 12, left = n - body;
        if (type == kCaf_desc) {
            if (size != 32) return fail(Status::DecodeError, kCafBadChunk);
            if (left < 32) return fail(Status::EndOfStream, kCafTruncated);
            const uint8_t* p = d + body;
            if ((be64(p) & 0x7fffffffffffffffull) == 0) return fail(Status::DecodeError, kCafBadDesc);  // rate 0.0 or -0.0
            const uint32_t bytes_per_packet = be32(p + 16), frames_per_packet = be32(p + 20), channels = be32(p + 24);
            // AudioDescription::read: an unknown format id fails before the channel count is read; a known one that is not ALAC
            // is refused here only after the reader's own checks, where the reference would go on to another decoder
            const uint32_t fmt = be32(p + 8);
            if (!caf_known_format(fmt)) return fail(Status::Unsupported, kCafNotAlac);
            if (channels == 0) return fail(Status::DecodeError, kCafBadDesc);
            if (fmt != kCaf_alac) return fail(Status::Unsupported, kCafNotAlac);
            if (have_desc) return fail(Status::DecodeError, kCafBadChunk);
            if (channels > 26) return fail(Status::Unsupported, kCafBadDesc);  // Position::from_count has 26 positions
            if (bytes_per_packet != 0 || frames_per_packet == 0) return fail(Status::Unsupported, kCafLayout);
            have_desc = true, a.frames_per_packet = frames_per_packet;
            at = body + 32;
        } else if (type == kCaf_data) {
            if (size != -1 && size < 4) return fail(Status::DecodeError, kCafBadChunk);
            if (left < 4) return fail(Status::EndOfStream, kCafTruncated);
            a.data_start = body + 4;
            sized_data = size != -1;
            if (sized_data && uint64_t(size - 4) > n - a.data_start) return fail(Status::EndOfStream, kCafTruncated);
            at = a.data_start + (sized_data ? uint64_t(size - 4) : 0);
        } else if (type == kCaf_chan) {
            if (size < 12) return fail(Status::DecodeError, kCafBadChunk);
            if (left < 12 || uint64_t(be32(d + body + 8)) * 20 > left - 12) return fail(Status::EndOfStream, kCafTruncated);
            at = body + 12 + uint64_t(be32(d + body + 8)) * 20;
        } else if (type == kCaf_pakt) {
            if (size < 24) return fail(Status::DecodeError, kCafBadChunk);
            if (!have_desc) return fail(Status::DecodeError, kCafNoDesc);
            if (left < 24) return fail(Status::EndOfStream, kCafTruncated);
            const int64_t total = int64_t(be64(d + body)), valid = int64_t(be64(d + body + 8));
            if (total < 0 || valid < 0) return fail(Status::DecodeError, kCafBadTable);
            a.table_at = body + 24, a.table_packets = uint64_t(total), a.valid_frames = valid;
            a.priming_frames = int32_t(be32(d + body + 16)), a.remainder_frames = int32_t(be32(d + body + 20));
            at = a.table_at;
            for (uint64_t k = 0; k < a.table_packets; ++k) {
                uint64_t v;
                const Status vs = caf_varint(d, n, at, v);
                if (vs == Status::EndOfStream) return fail(vs, kCafTruncated);
                if (vs != Status::Ok) return fail(vs, kCafBadTable);
            }
            a.table_bytes = at - a.table_at;
        } else {  // kuki, free and every other chunk: skipped (a cookie is kept)
            if (size < 0) return fail(Status::DecodeError, kCafBadChunk);
            if (uint64_t(size) > left) return fail(Status::EndOfStream, kCafTruncated);
            if (type == kCaf_kuki) have_cookie = true, cookie_at = body, cookie_len = uint64_t(size);
            at = body + uint64_t(size);
        }
        if (!have_desc) return fail(Status::DecodeError, kCafNoDesc);
        if (at == n) break;
    }
    if (!sized_data) a.data_start = n;  // no seek back to the audio: the packets are read from where the walk stopped
    if (!have_cookie) return fail(Status::Unsupported, kCafNoCookie);
    const uint64_t data_start = a.data_start, table_at = a.table_at, table_packets = a.table_packets, table_bytes = a.table_bytes;
    const int64_t valid = a.valid_frames;
    const int32_t priming = a.priming_frames, remainder = a.remainder_frames;
    const uint32_t fpp = a.frames_per_packet;
    const Status s = caf_alac_cookie(d + cookie_at, cookie_len, a);
    a.data_start = data_start, a.table_at = table_at, a.table_packets = table_packets, a.table_bytes = table_bytes, a.valid_frames = valid;
    a.priming_frames = priming, a.remainder_frames = remainder, a.frames_per_packet = fpp;
    return s;
}

// Packets are read back to back from data_start (demuxer.rs:148-160); the first whose end passes the end of the file fails
// its read and ends the file's packets.  A packet of 2^32 bytes or more ends them too (it cannot fit a file the device index
// takes, and a decoder job's length is 32 bits).
SYMGPU_PACKET_HD inline bool caf_packet_fits(uint64_t data_start, uint64_t offset, uint64_t size, uint64_t n) {
    return size <= 0xffffffffull && data_start <= n && offset <= n - data_start && size <= n - data_start - offset;
}

struct CafPacket {
    uint64_t offset;  // in the file
    uint32_t size, frames;
};

// Host index: caf_open, then the packet table read integer by integer.
class CafIndexer {
public:
    CafIndexer(const uint8_t* d, size_t n) : d_(d), n_(n) {}
    Status open() { return caf_open(d_, n_, a_); }
    const CafAlac& alac() const { return a_; }
    // The packets in order, up to the first that does not fit.
    template <class Sink>
    void packets(Sink&& sink) const {
        uint64_t at = a_.table_at, offset = 0;
        for (uint64_t k = 0; k < a_.table_packets; ++k) {
            uint64_t size;
            caf_varint(d_, n_, at, size);  // caf_open read them all
            if (!caf_packet_fits(a_.data_start, offset, size, n_)) return;
            sink(CafPacket{a_.data_start + offset, uint32_t(size), a_.frames_per_packet});
            offset += size;
        }
    }

private:
    const uint8_t* d_;
    uint64_t n_;
    CafAlac a_{};
};

}  // namespace packet
}  // namespace symgpu
