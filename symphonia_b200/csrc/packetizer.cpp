// C entry points of the packetisers (include/symgpu.h "Packetisers"): thin adapters from the index builders of
// include/symgpu/packetizer.hpp to flat, caller-owned tables.  Host only; no context, no device.
#include <cstring>
#include <vector>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"
#include "caf_records.h"
#include "flac_records.h"
#include "mpa_records.h"

using namespace symgpu::packet;

static symgpu_status to_status(Status s) {
    switch (s) {
        case Status::Ok: return SYMGPU_OK;
        case Status::Unsupported: return SYMGPU_ERR_UNSUPPORTED;
        default: return SYMGPU_ERR_DECODE;
    }
}

extern "C" symgpu_status symgpu_mpa_index(const uint8_t* data, size_t n, int seekable, symgpu_mpa_track* track,
                                          symgpu_mpa_packet* packets, size_t cap, size_t* n_out) {
    if ((!data && n) || !track || !n_out || (cap && !packets)) return SYMGPU_ERR_ARG;
    MpaIndexer ix(data, n);
    if (ix.open(seekable != 0) != Status::Ok) return *n_out = 0, SYMGPU_ERR_DECODE;
    *track = symgpu_detail::mpa_track_record(ix.track());
    size_t count = 0;
    MpaPacket p;
    while (ix.next(p) == Status::Ok) {
        if (count < cap) packets[count] = symgpu_detail::mpa_packet_record(p, data + p.offset);
        ++count;
    }
    *n_out = count;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_adts_index(const uint8_t* data, size_t n, symgpu_adts_packet* packets, size_t cap, size_t* n_out,
                                           symgpu_status* stop) {
    if ((!data && n) || !n_out || !stop || (cap && !packets)) return SYMGPU_ERR_ARG;
    AdtsIndexer ix(data, n);
    AdtsPacket p;
    size_t count = 0;
    Status s;
    while ((s = ix.next(p)) == Status::Ok) {
        if (count < cap) {
            symgpu_adts_packet& o = packets[count];
            o = symgpu_adts_packet{};
            o.offset = p.offset, o.size = p.size, o.sample_rate = p.sample_rate, o.pts = p.pts, o.channels = p.channels, o.profile = p.profile;
        }
        ++count;
    }
    *n_out = count;
    *stop = s == Status::EndOfStream ? (ix.truncated() ? SYMGPU_ERR_LIMIT : SYMGPU_OK) : to_status(s);
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_ogg_index(const uint8_t* data, size_t n, symgpu_ogg_packet* packets, size_t cap_packets,
                                          size_t* n_packets, symgpu_piece* pieces, size_t cap_pieces, size_t* n_pieces) {
    if ((!data && n) || !n_packets || !n_pieces || (cap_packets && !packets) || (cap_pieces && !pieces)) return SYMGPU_ERR_ARG;
    OggIndex ix;
    const Status s = OggIndex::build(data, n, ix, false);
    size_t np = 0, nq = 0;
    for (const auto& kv : ix.streams) {
        const OggLogicalStream& ls = kv.second;
        const size_t piece_base = nq;
        size_t used = 0;  // pieces of completed packets (an open packet's pieces trail the list and are not reported)
        for (const OggPacket& p : ls.packets()) {
            if (np < cap_packets) {
                symgpu_ogg_packet& o = packets[np];
                o = symgpu_ogg_packet{};
                o.serial = kv.first, o.page_sequence = p.page_sequence, o.page_absgp = p.page_absgp, o.len = p.len;
                o.first_piece = uint32_t(piece_base + p.first_piece), o.n_pieces = p.n_pieces, o.last_on_page = p.last_on_page;
            }
            ++np;
            used = size_t(p.first_piece) + p.n_pieces;
        }
        for (size_t k = 0; k < used; ++k, ++nq)
            if (nq < cap_pieces) pieces[nq] = symgpu_piece{ls.pieces()[k].offset, ls.pieces()[k].len, 0};
    }
    *n_packets = np, *n_pieces = nq;
    return to_status(s);
}

extern "C" symgpu_status symgpu_vorbis_ident_parse(const uint8_t* packet, size_t n, symgpu_vorbis_ident* ident) {
    if (!packet || !ident || n < 30) return SYMGPU_ERR_ARG;
    VorbisIdent id;
    const Status s = vorbis_read_ident(packet, n, id);
    if (s != Status::Ok) return to_status(s);
    *ident = symgpu_vorbis_ident{id.sample_rate, id.n_channels, id.bs0_exp, id.bs1_exp, 0};
    return SYMGPU_OK;
}

static bool ident_ok(const symgpu_vorbis_ident* i) {
    return i && i->channels && i->bs0_exp >= 6 && i->bs1_exp <= 13 && i->bs0_exp <= i->bs1_exp;
}

extern "C" symgpu_status symgpu_vorbis_setup_modes(const uint8_t* packet, size_t n, const symgpu_vorbis_ident* ident, uint32_t* n_modes,
                                                   uint64_t* long_block_mask) {
    if (!packet || !n_modes || !long_block_mask || !ident_ok(ident)) return SYMGPU_ERR_ARG;
    VorbisIdent id{ident->channels, ident->sample_rate, ident->bs0_exp, ident->bs1_exp};
    uint8_t modes = 0;
    const Status s = vorbis_read_setup_modes(packet, n, id, modes, *long_block_mask);
    if (s != Status::Ok) return SYMGPU_ERR_DECODE;
    *n_modes = modes;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_setup_parse(const uint8_t* packet, size_t n, const symgpu_vorbis_ident* ident, symgpu_vorbis_setup_info* info,
                                                   symgpu_vorbis_floor1* floors) {
    if (!packet || !info || !floors || !ident_ok(ident)) return SYMGPU_ERR_ARG;
    const VorbisIdent id{ident->channels, ident->sample_rate, ident->bs0_exp, ident->bs1_exp};
    VorbisSetup st;
    if (vorbis_read_setup(packet, n, id, st) != Status::Ok) return SYMGPU_ERR_DECODE;
    *info = symgpu_vorbis_setup_info{};
    info->n_codebooks = st.n_codebooks, info->n_floors = uint32_t(st.floor_type.size()), info->n_residues = uint32_t(st.residues.size());
    info->n_mappings = uint32_t(st.mappings.size()), info->n_modes = uint32_t(st.modes.size());
    for (size_t i = 0; i < st.modes.size(); ++i) {
        if (st.modes[i].first) info->long_block_mask |= uint64_t(1) << i;
        info->mode_mapping[i] = st.modes[i].second;
    }
    for (size_t i = 0; i < st.floor_type.size(); ++i) {
        info->floor_type[i] = st.floor_type[i];
        symgpu_vorbis_floor1& o = floors[i];
        std::memset(&o, 0, sizeof o);
        if (st.floor_type[i] != 1) continue;
        const VorbisFloor1Setup& f = st.floor1[i];
        o.multiplier = f.multiplier, o.n_posts = f.n_posts;
        std::memcpy(o.x_list, f.x_list, sizeof o.x_list), std::memcpy(o.low, f.low, 65), std::memcpy(o.high, f.high, 65), std::memcpy(o.sort_order, f.sort_order, 65);
    }
    return SYMGPU_OK;
}
static_assert(sizeof(symgpu_vorbis_setup_info) == 160, "record sizes are ABI");

extern "C" symgpu_status symgpu_ogg_gather(const uint8_t* data, size_t n, const symgpu_ogg_packet* packets, size_t n_packets, const symgpu_piece* pieces,
                                           size_t n_pieces, uint8_t* out, size_t cap, symgpu_piece* table, size_t* used) {
    if ((!data && n) || (n_packets && (!packets || !pieces || !table)) || !used || (cap && !out)) return SYMGPU_ERR_ARG;
    size_t at = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        const symgpu_ogg_packet& pk = packets[i];
        if (size_t(pk.first_piece) + pk.n_pieces > n_pieces) return SYMGPU_ERR_ARG;
        const size_t start = at;
        for (uint32_t k = 0; k < pk.n_pieces; ++k) {
            const symgpu_piece& pc = pieces[pk.first_piece + k];
            if (pc.offset > n || pc.len > n - pc.offset) return SYMGPU_ERR_ARG;
            if (pc.len > cap - at) return SYMGPU_ERR_LIMIT;
            std::memcpy(out + at, data + pc.offset, pc.len);
            at += pc.len;
        }
        table[i] = symgpu_piece{start, uint32_t(at - start), 0};
    }
    *used = at;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_ogg_page_end_trims(const uint32_t* page_sequence, const uint64_t* page_absgp, const uint32_t* dur,
                                                   const uint32_t* discard, size_t n, uint32_t* trim_end) {
    if (n && (!page_sequence || !page_absgp || !dur || !discard || !trim_end)) return SYMGPU_ERR_ARG;
    ogg_page_end_trims(page_sequence, page_absgp, dur, discard, n, trim_end);
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_packet_durations(const symgpu_vorbis_ident* ident, uint32_t n_modes, uint64_t long_block_mask,
                                                        const uint16_t* heads, const uint8_t* head_len, size_t n_packets, uint8_t* prev_exp,
                                                        uint32_t* dur, uint32_t* discard) {
    if (!ident_ok(ident) || n_modes == 0 || n_modes > 64 || !prev_exp || (n_packets && (!heads || !head_len || !dur || !discard)))
        return SYMGPU_ERR_ARG;
    const bool have_prev = *prev_exp != 0;
    if (have_prev && (*prev_exp < 6 || *prev_exp > 13)) return SYMGPU_ERR_ARG;
    const VorbisIdent id{ident->channels, ident->sample_rate, ident->bs0_exp, ident->bs1_exp};
    // the timer has no way to be seeded; replay the previous block through a one-mode timer of that size instead
    VorbisPacketTimer timer(id, uint8_t(n_modes), long_block_mask);
    if (have_prev) {
        VorbisIdent seed = id;
        seed.bs0_exp = seed.bs1_exp = *prev_exp;
        timer = VorbisPacketTimer(seed, 1, 0);
        const uint8_t zero = 0;
        uint64_t a, b;
        timer.next(&zero, 1, a, b);
        timer.rebind(id, uint8_t(n_modes), long_block_mask);
    }
    for (size_t i = 0; i < n_packets; ++i) {
        const uint8_t bytes[2] = {uint8_t(heads[i] & 0xff), uint8_t(heads[i] >> 8)};
        uint64_t a, b;
        timer.next(bytes, head_len[i] > 2 ? 2 : head_len[i], a, b);
        dur[i] = uint32_t(a), discard[i] = uint32_t(b);
    }
    *prev_exp = timer.prev_exp();
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_flac_index(const uint8_t* data, size_t n, symgpu_flac_stream_info* info, symgpu_flac_packet* packets, size_t cap,
                                           size_t* n_out) {
    if ((!data && n) || !info || !n_out || (cap && !packets)) return SYMGPU_ERR_ARG;
    FlacIndexer ix(data, n);
    const Status s = ix.open();
    if (s != Status::Ok) return *n_out = 0, s == Status::Unsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE;
    *info = symgpu_detail::flac_info_record(ix.info(), ix.first_frame_pos());
    size_t count = 0;
    FlacPacket p;
    while (ix.next(p) == Status::Ok) {
        if (count < cap) packets[count] = symgpu_detail::flac_packet_record(p);
        ++count;
    }
    *n_out = count;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_ogg_flac_packets(const uint8_t* blob, size_t n, const symgpu_piece* table, size_t n_packets,
                                                 symgpu_flac_stream_info* info, uint8_t* audio, uint32_t* slot) {
    if ((!blob && n) || !info || (n_packets && (!table || !audio || !slot))) return SYMGPU_ERR_ARG;
    for (size_t k = 0; k < n_packets; ++k)
        if (table[k].offset > n || table[k].len > n - table[k].offset) return SYMGPU_ERR_ARG;
    if (n_packets == 0) return SYMGPU_ERR_UNSUPPORTED;
    FlacStreamInfo si{};
    const Status s = ogg_flac_ident(blob + table[0].offset, table[0].len, si);
    if (s != Status::Ok) return to_status(s);
    *info = symgpu_detail::flac_info_record(si, 0);
    for (size_t k = 0; k < n_packets; ++k) {
        audio[k] = ogg_flac_is_audio(table[k].len, table[k].len ? blob[table[k].offset] : 0);
        slot[k] = audio[k] ? ogg_flac_packet_block(blob, table + k, 1) : 0;
    }
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_caf_index(const uint8_t* data, size_t n, symgpu_caf_info* info, symgpu_caf_packet* packets, size_t cap, size_t* n_out) {
    if ((!data && n) || !info || !n_out || (cap && !packets)) return SYMGPU_ERR_ARG;
    CafIndexer ix(data, n);
    const Status s = ix.open();
    *info = symgpu_detail::caf_info_record(ix.alac(), s);
    *n_out = 0;
    if (s != Status::Ok) return to_status(s);
    size_t count = 0;
    ix.packets([&](const CafPacket& p) {
        if (count < cap) packets[count] = symgpu_caf_packet{p.offset, p.size, p.frames};
        ++count;
    });
    info->n_packets = count;
    *n_out = count;
    return SYMGPU_OK;
}

static_assert(sizeof(symgpu_caf_info) == 96 && sizeof(symgpu_caf_packet) == 16, "record sizes are ABI");
static_assert(sizeof(symgpu_ogg_flac_file) == 88 && sizeof(symgpu_ogg_flac_packet_rank) == 32, "record sizes are ABI");
static_assert(sizeof(symgpu_flac_stream_info) == 56 && sizeof(symgpu_flac_packet) == 24, "record sizes are ABI");
static_assert(sizeof(symgpu_mpa_track) == 48 && sizeof(symgpu_mpa_packet) == 48 && sizeof(symgpu_adts_packet) == 32, "record sizes are ABI");
static_assert(sizeof(symgpu_piece) == 16 && sizeof(symgpu_ogg_packet) == 40 && sizeof(symgpu_vorbis_ident) == 8, "record sizes are ABI");

// ---- floor-1 setups: what the synthesis kernel relies on (host only; used by symgpu_vorbis_floors_set and by the Vorbis
// front-end when a stream is opened) ---------------------------------------------------------------------------------------
// A setup is what Floor1Setup holds after the reference's own checks (floor.rs:300-420): distinct x positions, sort_order a
// permutation by ascending x that starts at x = 0, and for every post >= 2 the nearest lower / higher neighbours among the
// EARLIER posts.  The kernel divides by x differences and sweeps the posts by dependency level, so none of this may be taken
// on trust.  x <= 2^15: rangebits up to 15 are legal (floor.rs:519-536); the kernel's seeded division stays exact (numerator
// < 2^23, divisor < 2^15).  levels (may be null): per setup 72 bytes = level[65] (level[i] = 1 + max(level[low[i]], level[high[i]]),
// level[0] = level[1] = 0), the largest level, 6 zero bytes -- struct FloorAux of codec_kernels.h.
extern "C" symgpu_status symgpu_vorbis_floors_levels(const symgpu_vorbis_floor1* floors, uint32_t n_floors, uint8_t* levels) {
    if (!floors || n_floors == 0) return SYMGPU_ERR_ARG;
    for (uint32_t i = 0; i < n_floors; ++i) {
        const symgpu_vorbis_floor1& f = floors[i];
        if (f.multiplier < 1 || f.multiplier > 4 || f.n_posts < 2 || f.n_posts > 65) return SYMGPU_ERR_ARG;
        bool seen[65] = {false};
        for (int k = 0; k < f.n_posts; ++k) {
            if (f.sort_order[k] >= f.n_posts || seen[f.sort_order[k]] || f.x_list[k] > 32768) return SYMGPU_ERR_ARG;
            seen[f.sort_order[k]] = true;
            if (k && f.x_list[f.sort_order[k]] <= f.x_list[f.sort_order[k - 1]]) return SYMGPU_ERR_ARG;
        }
        if (f.x_list[f.sort_order[0]] != 0) return SYMGPU_ERR_ARG;
        uint8_t level[72] = {0};
        for (int k = 2; k < f.n_posts; ++k) {
            const int lo = f.low[k], hi = f.high[k];
            if (lo >= k || hi >= k || !(f.x_list[lo] < f.x_list[k] && f.x_list[k] < f.x_list[hi])) return SYMGPU_ERR_ARG;
            level[k] = (uint8_t)(1 + (level[lo] > level[hi] ? level[lo] : level[hi]));
            if (level[k] > level[65]) level[65] = level[k];
        }
        if (levels) std::memcpy(levels + (size_t)i * 72, level, 72);
    }
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_floors_check(const symgpu_vorbis_floor1* floors, uint32_t n_floors) {
    return symgpu_vorbis_floors_levels(floors, n_floors, nullptr);
}
