// Vorbis packet rules of ONE audio packet, written once for host and device: the reference's bit reader, codeword reads (a
// 10-bit look-up, then the trie), floor-1 packet data, residue partitions of types 0 / 1 / 2 and the packet-level bookkeeping of
// VorbisDecoder::decode_inner up to -- not including -- inverse coupling (symphonia-codec-vorbis/src/{codebook,floor,residue,
// lib}.rs).  The CPU front-end (vorbis_frontend.cpp) calls decode_packet packet after packet with one class buffer per stream;
// the device decoder (vorbis_decode_kernel.cu) calls it once per packet with a fresh one.  Setup construction (codebooks, the
// canonical code assignment, VQ unpacking) is host only and lives in vorbis_frontend.cpp; it writes the flat form below.
//
// A packet depends on earlier packets only through the previous block flag, which decode_packet is handed (-1: none) and which
// is output, not input, of this stage.  The partition-class buffer's history never reaches an entry a packet reads before
// writing it, and what a class word writes does not depend on the buffer's size beyond the entries it has (the digits kept when
// it is cut are the same most significant ones); so a fresh buffer per packet gives the same output as the stream's buffer.
//
// Floating point: a residue element is the running f32 sum of the VQ values laid over it in pass order -- single IEEE
// additions; the VQ values themselves are computed on the host.  Host code is compiled with -ffp-contract=off, device code
// with -fmad=false.
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../include/symgpu.h"
#include "mp3_entropy.h"  // SYMGPU_HD; packetizer.hpp: VorbisFloor1Setup, VorbisResidueSetup

#include <vector>

namespace symgpu {
namespace vorbise {

using packet::VorbisFloor1Setup;
using packet::VorbisResidueSetup;

SYMGPU_HD uint32_t ilog(uint32_t x) {
    uint32_t n = 0;
    for (; x; x >>= 1) ++n;
    return n;
}
SYMGPU_HD size_t min_sz(size_t a, size_t b) { return a < b ? a : b; }

// The reference's BitReaderRtl, state for state (symphonia-core/src/io/bit.rs:941-1027, :1211-1250, :1305-1370).  In a Vorbis audio
// packet running out of bits is legal and decoding CONTINUES (the next channel's floor, the next sub-map's residue), so which
// bits a failed read leaves behind is observable: the reference keeps a 64-bit cache that it refills 8 bytes at a time, a read
// that fails on the FIRST refill consumes nothing, one that fails on a later refill has already dropped the cache it started
// with.  A simpler reader would differ on truncated packets; this one follows the cache.
struct PacketBits {
    const uint8_t* p;
    size_t n;         // bytes not yet fetched
    uint64_t bits = 0;
    uint32_t left = 0;
    SYMGPU_HD PacketBits(const uint8_t* data, size_t len) : p(data), n(len) {}
    SYMGPU_HD bool fetch() {  // fetch_bits: replace the cache with the next (up to) 8 bytes
        const size_t k = n < 8 ? n : 8;
        if (k == 0) return false;
        uint64_t v = 0;
        for (size_t i = 0; i < k; ++i) v |= uint64_t(p[i]) << (8 * i);
        p += k, n -= k, bits = v, left = uint32_t(8 * k);
        return true;
    }
    SYMGPU_HD void top_up() {  // fetch_bits_partial: fill the free whole bytes of the cache
        size_t k = (64 - left) >> 3;
        if (k > n) k = n;
        for (size_t i = 0; i < k; ++i) bits |= uint64_t(p[i]) << left, left += 8;
        p += k, n -= k;
    }
    SYMGPU_HD void consume(uint32_t w) { left -= w, bits = w < 64 ? bits >> w : 0; }
    SYMGPU_HD bool read(uint32_t width, uint32_t& out) {  // read_bits_leq32
        uint64_t acc = bits;
        uint32_t needed = width;
        while (needed > left) {
            needed -= left;
            if (!fetch()) return false;
            acc |= bits << (width - needed);
        }
        consume(needed);
        out = uint32_t(acc & (width >= 32 ? 0xffffffffull : ((1ull << width) - 1)));
        return true;
    }
    SYMGPU_HD bool read_bool(bool& out) {
        if (left < 1 && !fetch()) return false;
        out = bits & 1;
        consume(1);
        return true;
    }
};

// ---- the setup in flat form ---------------------------------------------------------------------------------------------
// A codebook: offsets into the setup's three pools.  lut[1024]: the next ten stream bits (first bit = bit 0) -> (value + 1) << 6
// | length, 0 = a longer code; child: the binary trie, child[2 * node + bit] = node index, ~value for a leaf, 0 = no such code
// (at least one node per book); vq: [entries][dims] when has_vq.
struct Book {
    uint32_t lut, child, vq;
    uint32_t max_len;
    uint16_t dims;
    uint8_t has_vq, reserved;
};
struct Mapping {  // at most one coupling step, (magnitude 0, angle 1)
    uint8_t n_submaps, coupled, multiplex[2];
    uint8_t submap_floor[16], submap_residue[16];
};
struct Mode {
    uint8_t long_block, mapping;
};
struct Setup {
    const Book* books;
    const uint32_t* lut;
    const int32_t* child;
    const float* vq;
    const VorbisFloor1Setup* floors;
    const VorbisResidueSetup* residues;
    const Mapping* mappings;
    const Mode* modes;
    uint32_t n_modes;
    uint8_t bs0_exp, bs1_exp, channels;
};
// Where a setup's sections lie in a byte blob (16-byte aligned offsets), as the device decoder receives it.
struct SetupHead {
    uint64_t books, lut, child, vq, floors, residues, mappings, modes;
    uint32_t n_modes;
    uint32_t class_cap;  // the most partition classes any residue of this setup needs in one packet
    uint8_t bs0_exp, bs1_exp, channels, reserved;
    uint32_t sample_rate;
};
SYMGPU_HD Setup view_of(const uint8_t* blob, const SetupHead& h) {
    Setup s;
    s.books = reinterpret_cast<const Book*>(blob + h.books);
    s.lut = reinterpret_cast<const uint32_t*>(blob + h.lut);
    s.child = reinterpret_cast<const int32_t*>(blob + h.child);
    s.vq = reinterpret_cast<const float*>(blob + h.vq);
    s.floors = reinterpret_cast<const VorbisFloor1Setup*>(blob + h.floors);
    s.residues = reinterpret_cast<const VorbisResidueSetup*>(blob + h.residues);
    s.mappings = reinterpret_cast<const Mapping*>(blob + h.mappings);
    s.modes = reinterpret_cast<const Mode*>(blob + h.modes);
    s.n_modes = h.n_modes, s.bs0_exp = h.bs0_exp, s.bs1_exp = h.bs1_exp, s.channels = h.channels;
    return s;
}

// The partition-class vector: `size` entries in use (it only grows, never cleared), room for `cap`.
struct ClassBuf {
    uint8_t* p;
    size_t size, cap;
};

// One codeword, first stream bit = root of the tree (codebook.rs:366-369 "BitOrder::Reverse"; bit.rs:1211-1250): the cache is
// topped up, the code is matched against it padded with zeros, and must then fit in what the cache really holds -- else the
// packet has ended and nothing is consumed.
SYMGPU_HD bool read_code(const Setup& S, const Book& b, PacketBits& bs, uint32_t& value) {
    if (bs.left < b.max_len) bs.top_up();
    const uint32_t e = S.lut[b.lut + uint32_t(bs.bits & 1023)];  // codes of up to ten bits: one look-up (the cache holds zeros above `left`)
    if (e) {
        const uint32_t len = e & 63;
        if (len > bs.left) return false;
        bs.consume(len);
        return value = (e >> 6) - 1, true;
    }
    const int32_t* child = S.child + b.child;
    int32_t node = 0;
    for (uint32_t depth = 0; depth < 64; ++depth) {
        const uint32_t bit = uint32_t(bs.bits >> depth) & 1;
        const int32_t next = child[size_t(2 * node) + bit];
        if (next < 0) {
            if (depth + 1 > bs.left) return false;
            bs.consume(depth + 1);
            return value = uint32_t(~next), true;
        }
        if (next == 0) return false;  // cannot happen in a fully specified tree
        node = next;
    }
    return false;
}

// floor.rs:655-722.  Returns false when the floor is unused (flag clear, or the packet ended inside it).
SYMGPU_HD bool read_floor1(const Setup& S, const VorbisFloor1Setup& f, PacketBits& bs, uint16_t* y) {
    bool used;
    if (!bs.read_bool(used) || !used) return false;
    const uint32_t range = f.multiplier == 1 ? 256u : f.multiplier == 2 ? 128u : f.multiplier == 3 ? 86u : 64u;
    const uint32_t bits = ilog(range - 1);
    uint32_t v;
    if (!bs.read(bits, v)) return false;
    y[0] = uint16_t(v);
    if (!bs.read(bits, v)) return false;
    y[1] = uint16_t(v);
    int offset = 2;
    for (int p = 0; p < f.partitions; ++p) {
        const auto& cl = f.classes[f.partition_class[p]];
        const uint32_t cbits = cl.subclass_bits, csub = (1u << cbits) - 1;
        uint32_t cval = 0;
        if (cbits && !read_code(S, S.books[cl.mainbook], bs, cval)) return false;
        for (int d = 0; d < cl.dimensions; ++d) {
            const uint32_t sub = cval & csub;
            cval >>= cbits;
            v = 0;
            if (cl.subbook_used & (1u << sub))
                if (!read_code(S, S.books[cl.subbooks[sub]], bs, v)) return false;
            y[offset + d] = uint16_t(v);
        }
        offset += cl.dimensions;
    }
    return true;
}

// residue.rs:451-477
SYMGPU_HD void decode_classes(uint32_t val, unsigned per_word, uint32_t classifications, uint8_t* out, size_t n_out) {
    unsigned skip = 0;
    if (per_word > n_out) {
        skip = unsigned(per_word - n_out);
        for (unsigned k = 0; k < skip; ++k) val /= classifications;
    }
    for (size_t k = per_word - skip; k-- > 0;) out[k] = uint8_t(val % classifications), val /= classifications;
}

// Element j of a residue vector laid over `lanes` channel rows: row j mod lanes, line j / lanes (type 2's interleaving, residue.rs:
// 177-218; one lane for types 0 / 1).  Every element receives its additions in the same order as through a separate vector.
SYMGPU_HD float& element(float* const* rows, unsigned lanes, size_t j) { return lanes == 1 ? rows[0][j] : rows[j & 1][j >> 1]; }

// One partition: residue.rs:479-543, over elements [start, start + n).  false: the packet ended (legal: decoding stops), `bad`
// set: malformed setup.
SYMGPU_HD bool read_partition(const Setup& S, const Book& book, PacketBits& bs, float* const* rows, unsigned lanes, size_t start, size_t n, bool format0,
                              bool& bad) {
    if (!book.has_vq) return bad = true, false;  // "vorbis: not a vq codebook"
    const size_t dim = book.dims;
    if (format0) {
        const size_t step = n / dim;
        for (size_t i = 0; i < step; ++i) {
            uint32_t e;
            if (!read_code(S, book, bs, e)) return false;
            const float* v = S.vq + book.vq + size_t(e) * dim;
            for (size_t k = 0, o = i; k < dim && o < n; ++k, o += step) element(rows, lanes, start + o) += v[k];
        }
    } else {
        for (size_t o = 0; o + dim <= n; o += dim) {
            uint32_t e;
            if (!read_code(S, book, bs, e)) return false;
            const float* v = S.vq + book.vq + size_t(e) * dim;
            for (size_t k = 0; k < dim; ++k) element(rows, lanes, start + o + k) += v[k];
        }
    }
    return true;
}

// residue.rs:142-449 for the channels in `chans` (1 or 2 of them).  0 ok, 1 decode error.
SYMGPU_HD int read_residue(const Setup& S, const VorbisResidueSetup& r, PacketBits& bs, unsigned bs_exp, const int* chans, int n_chans,
                           const uint8_t* do_not_decode, float* residue, uint32_t slot, ClassBuf& cls) {
    const Book& class_book = S.books[r.classbook];
    const size_t n2 = (size_t(1) << bs_exp) >> 1;
    const size_t full = r.type == 2 ? n2 * size_t(n_chans) : n2;
    const size_t begin = min_sz(r.begin, full), end = min_sz(r.end, full);
    const size_t part_size = r.partition_size, per_word = class_book.dims, parts = (end - begin) / part_size;
    bool any = false;
    for (int c = 0; c < n_chans; ++c) any |= !do_not_decode[chans[c]];
    // the channels' rows (already zeroed by the caller); type 2 adds straight into them through its interleaving
    float* rows[2] = {residue + size_t(chans[0]) * slot, residue + size_t(chans[n_chans - 1]) * slot};
    // the partition classes live in a vector that only ever grows and is never cleared (residue.rs:434-441): what a class word
    // writes is bounded by the vector's END, not by this packet's partition count, so a class word of the last group can spill
    // into the next channel's entries and stale entries of earlier packets stay behind -- reproduced, because later passes read them
    {
        const size_t class_slots = r.type == 2 ? parts : parts * size_t(n_chans);
        if (cls.size < class_slots) {
            if (class_slots > cls.cap) return 1;  // (the caller sizes the buffer for every residue of the setup)
            for (size_t i = cls.size; i < class_slots; ++i) cls.p[i] = 0;
            cls.size = class_slots;
        }
    }
    if (any) {
        bool bad = false, ended = false;
        for (unsigned pass = 0; pass <= r.max_pass && !ended; ++pass)
            for (size_t first = 0; first < parts && !ended; first += per_word) {
                if (pass == 0)
                    for (int c = 0; c < (r.type == 2 ? 1 : n_chans) && !ended; ++c) {
                        if (r.type != 2 && do_not_decode[chans[c]]) continue;
                        uint32_t code;
                        if (!read_code(S, class_book, bs, code)) {
                            ended = true;
                            break;
                        }
                        const size_t base = first + size_t(c) * parts;
                        decode_classes(code, unsigned(per_word), r.classifications, cls.p + base, cls.size - base);
                    }
                const size_t last = min_sz(parts, first + per_word);
                for (size_t part = first; part < last && !ended; ++part)
                    for (int c = 0; c < (r.type == 2 ? 1 : n_chans) && !ended; ++c) {
                        if (r.type != 2 && do_not_decode[chans[c]]) continue;
                        const uint8_t k = cls.p[part + parts * size_t(c)];
                        if (!(r.used[k] & (1u << pass))) continue;
                        const size_t start = begin + part_size * part;
                        const bool ok = r.type == 2 ? read_partition(S, S.books[r.books[k][pass]], bs, rows, unsigned(n_chans), start, part_size, false, bad)
                                                    : read_partition(S, S.books[r.books[k][pass]], bs, rows + c, 1, start, part_size, r.type == 0, bad);
                        if (!ok) ended = true;
                    }
            }
        if (bad) return 1;
    }
    return 0;
}

// One audio packet (lib.rs:145-248): SYMGPU_OK decoded, SYMGPU_ERR_DECODE where the reference errors (the caller drops the
// packet), SYMGPU_ERR_LIMIT when a floor index would not fit the unit's 16 bits.  unit / floor_y [2][65] / residue [2][slot] are
// written (slot >= blocksize_1 / 2, checked by the caller); unit->prev_block_flag is `prev_block_flag`, or the packet's own flag
// when it is negative.  `cls`: the partition-class vector, see read_residue.  residue_zeroed: the caller has zeroed the residue
// rows already (the device clears all packets' rows with one coalesced memset instead of one thread per packet).
SYMGPU_HD symgpu_status decode_packet(const Setup& S, const uint8_t* packet, size_t n, uint32_t slot, uint32_t floor_base, int prev_block_flag,
                                      ClassBuf& cls, symgpu_vorbis_unit* unit, uint16_t* floor_y, float* residue, bool residue_zeroed = false) {
    PacketBits bs(packet, n);
    bool flag;
    if (!bs.read_bool(flag) || flag) return SYMGPU_ERR_DECODE;  // lib.rs:151-154
    const uint32_t n_modes = S.n_modes;
    uint32_t mode_number;
    if (!bs.read(ilog(n_modes - 1), mode_number) || mode_number >= n_modes) return SYMGPU_ERR_DECODE;
    const bool long_block = S.modes[mode_number].long_block;
    const Mapping& mapping = S.mappings[S.modes[mode_number].mapping];
    if (long_block) {  // previous / next window flags: read, not used (lib.rs:168-173)
        if (!bs.read_bool(flag) || !bs.read_bool(flag)) return SYMGPU_ERR_DECODE;
    }
    const unsigned bs_exp = long_block ? S.bs1_exp : S.bs0_exp;
    const int n_ch = S.channels;
    *unit = symgpu_vorbis_unit{};
    for (int i = 0; i < 2 * 65; ++i) floor_y[i] = 0;
    if (!residue_zeroed)
        for (size_t i = 0; i < 2 * size_t(slot); ++i) residue[i] = 0.0f;
    unit->block_flag = long_block;
    unit->prev_block_flag = uint8_t(prev_block_flag < 0 ? long_block : prev_block_flag);
    unit->floor[0] = unit->floor[1] = 0xffff, unit->do_not_decode[0] = unit->do_not_decode[1] = 1;
    // floors, one per channel (lib.rs:184-207).  A packet that ends inside a floor leaves that floor unused and everything
    // behind it unread -- which the reader reports by failing every later read, exactly the reference's behaviour.
    for (int ch = 0; ch < n_ch; ++ch) {
        const uint8_t floor_idx = mapping.submap_floor[mapping.multiplex[ch]];
        if (uint64_t(floor_base) + floor_idx >= 0xffffu) return SYMGPU_ERR_LIMIT;  // unit->floor is 16 bits, 0xffff = unused
        const bool used = read_floor1(S, S.floors[floor_idx], bs, floor_y + ch * 65);
        unit->do_not_decode[ch] = !used;
        unit->floor[ch] = used ? uint16_t(floor_base + floor_idx) : uint16_t(0xffff);
        if (!used)
            for (int i = 0; i < 65; ++i) floor_y[ch * 65 + i] = 0;
    }
    // non-zero vector propagate (lib.rs:213-225)
    if (mapping.coupled && unit->do_not_decode[0] != unit->do_not_decode[1]) unit->do_not_decode[0] = unit->do_not_decode[1] = 0;
    // residues, per sub-map (lib.rs:229-248)
    for (int sm = 0; sm < mapping.n_submaps; ++sm) {
        int chans[2], n_chans = 0;
        for (int ch = 0; ch < n_ch; ++ch)
            if (mapping.multiplex[ch] == sm) chans[n_chans++] = ch;
        const VorbisResidueSetup& r = S.residues[mapping.submap_residue[sm]];
        if (n_chans == 0) continue;  // (the reference still runs the residue over no channels: nothing is read for types 0 / 1;
                                     //  type 2 divides by the channel count: a malformed setup, refuse it)
        // the partitions must lie inside the vector they are added to
        const size_t n2 = (size_t(1) << bs_exp) >> 1, full = r.type == 2 ? n2 * size_t(n_chans) : n2;
        const size_t begin = min_sz(r.begin, full), end = min_sz(r.end, full);
        if (S.books[r.classbook].dims == 0 || begin + ((end - begin) / r.partition_size) * size_t(r.partition_size) > full) return SYMGPU_ERR_DECODE;
        if (read_residue(S, r, bs, bs_exp, chans, n_chans, unit->do_not_decode, residue, slot, cls)) return SYMGPU_ERR_DECODE;
    }
    return SYMGPU_OK;
}

// Host only (vorbis_frontend.cpp): a front-end's setup appended to `blob` in the flat form (sections 16-byte aligned), and where
// its sections lie.
void setup_export(const symgpu_vorbis_fe* fe, std::vector<uint8_t>& blob, SetupHead& head);

}  // namespace vorbise
}  // namespace symgpu
