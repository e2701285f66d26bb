// Vorbis entropy front-end (include/symgpu.h "Vorbis entropy front-end", SURVEY §8f N1): codebooks, floor-1 packet
// decode, residue decode and the packet-level bookkeeping of VorbisDecoder::decode_inner up to -- not including --
// inverse coupling (symphonia-codec-vorbis/src/{codebook,floor,residue,lib}.rs).  Output: what symgpu_vorbis_synth_*
// reads.  The per-packet rules are those of vorbis_entropy.h (shared with the device decoder); this file builds the setup
// (codebooks, canonical codes, VQ tables) in their flat form and runs them packet after packet.
//
// Floating point, bit-exact by construction: a VQ table value is `m * delta + min (+ last)` in f32 in that order, a
// residue element the running f32 sum of the vectors laid over it in pass order -- the same single IEEE operations in
// the same order as the reference (the Makefile compiles host code with -ffp-contract=off).  float32_unpack follows the
// reference down to its use of powi: 2^e is built by repeated squaring in f32 (what llvm.powi lowers to), so that
// exponents outside f32's range give the same 0 / inf the Rust gives, not ldexp's denormals.
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <thread>
#include <vector>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"
#include "vorbis_entropy.h"

namespace {

using namespace symgpu::packet;

float powi2(int b) {  // compiler-rt __powisf2(2.0f, b)
    const bool recip = b < 0;
    float a = 2.0f, r = 1.0f;
    for (;;) {
        if (b & 1) r *= a;
        b /= 2;
        if (b == 0) break;
        a *= a;
    }
    return recip ? 1.0f / r : r;
}
float float32_unpack(uint32_t x) {  // codebook.rs:16-27
    const float value = float(x & 0x1fffff) * powi2(int((x & 0x7fe00000) >> 21) - 788);
    return (x & 0x80000000u) ? -value : value;
}

struct Codebook {  // as read_codebook builds it; appended to the setup's pools (vorbise::Book)
    uint16_t dims = 0;
    bool has_vq = false;
    std::vector<float> vq;           // [entries][dims]
    std::vector<int32_t> child;      // binary trie: child[2 * node + bit] = node index, or ~value for a leaf, or 0 = no such code
    uint32_t max_len = 0;
    uint32_t lut[1024] = {};         // next ten stream bits (first bit = bit 0) -> (value + 1) << 6 | length, 0 = a longer code
};

// Canonical codeword assignment (Vorbis I 3.2.1): each entry, in order, takes the lowest-valued free leaf of its length.
// Free sub-trees are kept as (prefix, depth); the tree must end up exactly full.  codebook.rs:112-210.
bool assign_codewords(const std::vector<uint8_t>& lens, std::vector<uint32_t>& words) {
    struct Free {
        uint32_t prefix;
        uint8_t depth;
    };
    std::vector<Free> free_nodes{{0, 0}};
    words.clear();
    for (uint8_t len : lens) {
        if (len == 0) continue;  // unused entries carry no codeword (the reference skips them and pushes nothing)
        int best = -1;
        uint64_t best_value = ~0ull;
        for (size_t k = 0; k < free_nodes.size(); ++k) {
            if (free_nodes[k].depth > len) continue;
            const uint64_t v = uint64_t(free_nodes[k].prefix) << (len - free_nodes[k].depth);  // its left-most leaf at this length
            if (v < best_value) best_value = v, best = int(k);
        }
        if (best < 0) return false;  // over-specified
        const Free f = free_nodes[size_t(best)];
        free_nodes.erase(free_nodes.begin() + best);
        for (uint8_t d = uint8_t(f.depth + 1); d <= len; ++d)  // going down left, every right sibling becomes free
            free_nodes.push_back(Free{uint32_t(((uint64_t(f.prefix) << (d - f.depth)) | 1)), d});
        words.push_back(uint32_t(best_value));
    }
    return free_nodes.empty();  // anything left: under-specified
}

// codebook.rs:214-360.  0 ok, 1 decode error.
int read_codebook(BitReaderRtl& bs, Codebook& cb) {
    if (bs.read(24) != 0x564342 || !bs.ok()) return 1;
    const uint32_t dims = bs.read(16), entries = bs.read(24);
    if (!bs.ok() || dims == 0 || dims > 32 || entries > 128 * 1024) return 1;
    cb.dims = uint16_t(dims);
    std::vector<uint8_t> lens;
    std::vector<uint32_t> values;
    if (!bs.read_bool()) {
        if (bs.read_bool()) {  // sparse
            for (uint32_t e = 0; e < entries && bs.ok(); ++e)
                if (bs.read_bool()) lens.push_back(uint8_t(bs.read(5) + 1)), values.push_back(e);
        } else {
            for (uint32_t e = 0; e < entries && bs.ok(); ++e) lens.push_back(uint8_t(bs.read(5) + 1)), values.push_back(e);
        }
    } else {
        uint32_t cur = 0, len = bs.read(5) + 1;
        for (;;) {
            const uint32_t num = bs.read(entries > cur ? vorbis_ilog(entries - cur) : 0);
            if (!bs.ok() || cur + num > entries) return 1;
            if (len > 32) return 1;  // (the reference would index past its 33-entry table)
            lens.insert(lens.end(), num, uint8_t(len));
            ++len, cur += num;
            if (cur == entries) break;
        }
        for (uint32_t e = 0; e < cur; ++e) values.push_back(e);
    }
    if (!bs.ok()) return 1;
    if (lens.size() == 1 && lens[0] == 1) lens.push_back(1), values.push_back(values[0]);  // single-entry book: both 1-bit codes (errata 20150226)
    const uint32_t lookup = bs.read(4);
    if (!bs.ok() || lookup > 2) return 1;
    if (lookup) {
        const float min_value = float32_unpack(bs.read(32)), delta = float32_unpack(bs.read(32));
        const uint32_t value_bits = bs.read(4) + 1;
        const bool sequence = bs.read_bool();
        if (!bs.ok()) return 1;
        uint32_t n_values;
        if (lookup == 1) {  // greatest v with v^dims <= entries (the reference computes it in f32 and asserts this bound)
            uint32_t v = 0;
            for (;;) {
                uint64_t pw = 1;
                bool over = false;
                for (uint32_t k = 0; k < dims && !over; ++k) pw *= uint64_t(v) + 1, over = pw > entries;
                if (over) break;
                ++v;
            }
            n_values = v;
        } else {
            n_values = entries * dims;
        }
        std::vector<uint16_t> mult(n_values);
        for (uint32_t k = 0; k < n_values; ++k) mult[k] = uint16_t(bs.read(value_bits));
        if (!bs.ok()) return 1;
        cb.has_vq = true;
        cb.vq.assign(size_t(entries) * dims, 0.0f);
        for (uint32_t e = 0; e < entries; ++e) {
            float last = 0.0f;
            uint32_t divisor = 1;
            for (uint32_t d = 0; d < dims; ++d) {
                const size_t at = lookup == 1 ? size_t((e / divisor) % n_values) : size_t(e) * dims + d;
                const float v = float(mult[at]) * delta + min_value + last;
                cb.vq[size_t(e) * dims + d] = v;
                if (sequence) last = v;
                divisor *= n_values;  // u32 wrap-around included, as in the reference
            }
        }
    }
    std::vector<uint32_t> words;
    if (!assign_codewords(lens, words)) return 1;
    cb.child.assign(2, 0);
    cb.max_len = lens.empty() ? 0 : *std::max_element(lens.begin(), lens.end());
    size_t w = 0;
    for (size_t k = 0; k < lens.size(); ++k) {
        if (lens[k] == 0) continue;
        int32_t node = 0;
        for (int b = lens[k] - 1; b >= 0; --b) {
            const uint32_t bit = (words[w] >> b) & 1;
            int32_t& slot = cb.child[size_t(2 * node) + bit];
            if (b == 0) {
                slot = ~int32_t(values[k]);
            } else {
                if (slot == 0) {
                    const int32_t fresh = int32_t(cb.child.size() / 2);
                    cb.child.push_back(0), cb.child.push_back(0);
                    cb.child[size_t(2 * node) + bit] = fresh;  // (push_back may have moved the storage: index again)
                    node = fresh;
                } else {
                    node = slot;
                }
            }
        }
        if (lens[k] <= 10) {
            uint32_t first = 0;  // the codeword in stream order: bit i of the index = the i-th bit read
            for (int i = 0; i < lens[k]; ++i) first |= ((words[w] >> (lens[k] - 1 - i)) & 1u) << i;
            for (uint32_t rest = 0; rest < (1u << (10 - lens[k])); ++rest) cb.lut[first | (rest << lens[k])] = (uint32_t(values[k]) + 1) << 6 | lens[k];
        }
        ++w;
    }
    return 0;
}

}  // namespace

namespace ve = symgpu::vorbise;

struct symgpu_vorbis_fe {
    VorbisIdent ident{};
    VorbisSetup setup;
    // the setup in the flat form of vorbis_entropy.h
    std::vector<ve::Book> books;
    std::vector<uint32_t> lut;
    std::vector<int32_t> child;
    std::vector<float> vq;
    std::vector<ve::Mapping> mappings;
    std::vector<ve::Mode> modes;
    uint32_t class_cap = 0;
    ve::Setup view{};
    int prev_block_flag = -1;
    std::vector<uint8_t> part_classes;  // persistent across packets, see read_residue
    ve::ClassBuf classes{};
};

namespace {

void append_book(symgpu_vorbis_fe& fe, const Codebook& cb) {
    ve::Book b{};
    b.lut = uint32_t(fe.lut.size()), b.child = uint32_t(fe.child.size()), b.vq = uint32_t(fe.vq.size());
    b.max_len = cb.max_len, b.dims = cb.dims, b.has_vq = cb.has_vq;
    fe.lut.insert(fe.lut.end(), cb.lut, cb.lut + 1024);
    fe.child.insert(fe.child.end(), cb.child.begin(), cb.child.end());
    fe.vq.insert(fe.vq.end(), cb.vq.begin(), cb.vq.end());
    fe.books.push_back(b);
}

// Pools, mappings and modes in place: the pointers of fe.view, and the class vector sized for the setup's largest residue.
void finish_setup(symgpu_vorbis_fe& fe) {
    for (const auto& m : fe.setup.mappings) {
        ve::Mapping o{};
        o.n_submaps = m.n_submaps, o.coupled = uint8_t(m.couplings.empty() ? 0 : 1);
        for (size_t c = 0; c < m.multiplex.size() && c < 2; ++c) o.multiplex[c] = m.multiplex[c];
        std::memcpy(o.submap_floor, m.submap_floor, 16), std::memcpy(o.submap_residue, m.submap_residue, 16);
        fe.mappings.push_back(o);
    }
    for (const auto& md : fe.setup.modes) fe.modes.push_back(ve::Mode{uint8_t(md.first), md.second});
    const size_t n2 = (size_t(1) << fe.ident.bs1_exp) >> 1, ch = fe.ident.n_channels;
    for (const VorbisResidueSetup& r : fe.setup.residues) {  // a short block's partitions are never more than a long block's
        const size_t full = r.type == 2 ? n2 * ch : n2;
        const size_t begin = std::min<size_t>(r.begin, full), end = std::min<size_t>(r.end, full);
        const size_t parts = r.partition_size ? (end - begin) / r.partition_size : 0;
        fe.class_cap = std::max<uint32_t>(fe.class_cap, uint32_t(r.type == 2 ? parts : parts * ch));
    }
    fe.part_classes.assign(std::max<uint32_t>(fe.class_cap, 1), 0);
    fe.classes = ve::ClassBuf{fe.part_classes.data(), 0, fe.class_cap};
    ve::Setup& v = fe.view;
    v.books = fe.books.data(), v.lut = fe.lut.data(), v.child = fe.child.data(), v.vq = fe.vq.data();
    v.floors = fe.setup.floor1.data(), v.residues = fe.setup.residues.data(), v.mappings = fe.mappings.data(), v.modes = fe.modes.data();
    v.n_modes = uint32_t(fe.setup.modes.size()), v.bs0_exp = fe.ident.bs0_exp, v.bs1_exp = fe.ident.bs1_exp, v.channels = fe.ident.n_channels;
}

template <class T>
uint64_t put(std::vector<uint8_t>& blob, const T* p, size_t n) {
    const uint64_t at = (blob.size() + 15) & ~uint64_t(15);
    blob.resize(size_t(at) + n * sizeof(T));
    if (n) std::memcpy(blob.data() + at, p, n * sizeof(T));
    return at;
}

}  // namespace

void symgpu::vorbise::setup_export(const symgpu_vorbis_fe* fe, std::vector<uint8_t>& blob, SetupHead& h) {
    h = SetupHead{};
    h.books = put(blob, fe->books.data(), fe->books.size());
    h.lut = put(blob, fe->lut.data(), fe->lut.size());
    h.child = put(blob, fe->child.data(), fe->child.size());
    h.vq = put(blob, fe->vq.data(), fe->vq.size());
    h.floors = put(blob, fe->setup.floor1.data(), fe->setup.floor1.size());
    h.residues = put(blob, fe->setup.residues.data(), fe->setup.residues.size());
    h.mappings = put(blob, fe->mappings.data(), fe->mappings.size());
    h.modes = put(blob, fe->modes.data(), fe->modes.size());
    h.n_modes = uint32_t(fe->modes.size()), h.class_cap = fe->class_cap;
    h.bs0_exp = fe->ident.bs0_exp, h.bs1_exp = fe->ident.bs1_exp, h.channels = fe->ident.n_channels, h.sample_rate = fe->ident.sample_rate;
}

extern "C" symgpu_status symgpu_vorbis_fe_create(const uint8_t* ident, size_t n_ident, const uint8_t* setup, size_t n_setup, symgpu_vorbis_fe** out) {
    if (!ident || !setup || !out) return SYMGPU_ERR_ARG;
    std::unique_ptr<symgpu_vorbis_fe> fe(new (std::nothrow) symgpu_vorbis_fe());
    if (!fe) return SYMGPU_ERR_LIMIT;
    const Status si = vorbis_read_ident(ident, n_ident, fe->ident);
    if (si != Status::Ok) return si == Status::Unsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE;
    if (vorbis_read_setup(setup, n_setup, fe->ident, fe->setup) != Status::Ok) return SYMGPU_ERR_DECODE;
    // the codebooks once more, this time built (the walk above only checked their syntax)
    BitReaderRtl bs(setup + 7, n_setup - 7);
    const uint32_t n_books = bs.read(8) + 1;
    for (uint32_t k = 0; k < n_books; ++k) {
        Codebook cb;
        if (read_codebook(bs, cb)) return SYMGPU_ERR_DECODE;
        append_book(*fe, cb);
    }
    // residue partitions must fit the blocks they are laid over (the reference would panic slicing past the vector)
    // -- checked per packet; here: what the synthesis kernel cannot take
    if (fe->ident.n_channels > 2) return SYMGPU_ERR_UNSUPPORTED;
    for (uint8_t t : fe->setup.floor_type)
        if (t != 1) return SYMGPU_ERR_UNSUPPORTED;
    for (const auto& m : fe->setup.mappings) {
        if (m.couplings.size() > 1) return SYMGPU_ERR_UNSUPPORTED;
        if (m.couplings.size() == 1 && !(m.couplings[0].first == 0 && m.couplings[0].second == 1)) return SYMGPU_ERR_UNSUPPORTED;
    }
    // what symgpu_vorbis_floors_set will insist on at launch time is refused here, per stream (a setup whose read X values
    // repeat an implied end point passes the reference's parser but would divide by zero in its render_line)
    {
        std::vector<symgpu_vorbis_floor1> fl(fe->setup.floor1.size());
        for (size_t i = 0; i < fl.size(); ++i) {
            const VorbisFloor1Setup& f = fe->setup.floor1[i];
            std::memset(&fl[i], 0, sizeof fl[i]);
            fl[i].multiplier = f.multiplier, fl[i].n_posts = f.n_posts;
            std::memcpy(fl[i].x_list, f.x_list, sizeof fl[i].x_list), std::memcpy(fl[i].low, f.low, 65), std::memcpy(fl[i].high, f.high, 65),
                std::memcpy(fl[i].sort_order, f.sort_order, 65);
        }
        if (!fl.empty() && symgpu_vorbis_floors_check(fl.data(), uint32_t(fl.size())) != SYMGPU_OK) return SYMGPU_ERR_UNSUPPORTED;
    }
    // one coupling flag per stream record: every mode's mapping must agree
    for (size_t k = 1; k < fe->setup.modes.size(); ++k)
        if (fe->setup.mappings[fe->setup.modes[k].second].couplings.size() != fe->setup.mappings[fe->setup.modes[0].second].couplings.size())
            return SYMGPU_ERR_UNSUPPORTED;
    finish_setup(*fe);
    *out = fe.release();
    return SYMGPU_OK;
}
extern "C" void symgpu_vorbis_fe_destroy(symgpu_vorbis_fe* fe) { delete fe; }
extern "C" void symgpu_vorbis_fe_reset(symgpu_vorbis_fe* fe) {
    if (fe) fe->prev_block_flag = -1;
}

extern "C" symgpu_status symgpu_vorbis_fe_config(const symgpu_vorbis_fe* fe, symgpu_vorbis_stream* stream, symgpu_vorbis_floor1* floors, uint32_t* n_floors) {
    if (!fe || !stream || !floors || !n_floors) return SYMGPU_ERR_ARG;
    *stream = symgpu_vorbis_stream{fe->ident.bs0_exp, fe->ident.bs1_exp, fe->ident.n_channels,
                                   uint8_t(fe->setup.mappings[fe->setup.modes[0].second].couplings.empty() ? 0 : 1)};
    *n_floors = uint32_t(fe->setup.floor1.size());
    for (size_t i = 0; i < fe->setup.floor1.size(); ++i) {
        const VorbisFloor1Setup& f = fe->setup.floor1[i];
        symgpu_vorbis_floor1& o = floors[i];
        std::memset(&o, 0, sizeof o);
        o.multiplier = f.multiplier, o.n_posts = f.n_posts;
        std::memcpy(o.x_list, f.x_list, sizeof o.x_list), std::memcpy(o.low, f.low, 65), std::memcpy(o.high, f.high, 65), std::memcpy(o.sort_order, f.sort_order, 65);
    }
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_fe_decode(symgpu_vorbis_fe* fe, const uint8_t* packet, size_t n, uint32_t slot, uint32_t floor_base,
                                                 symgpu_vorbis_unit* unit, uint16_t* floor_y, float* residue) {
    if (!fe || (!packet && n) || !unit || !floor_y || !residue) return SYMGPU_ERR_ARG;
    if (slot < ((1u << fe->ident.bs1_exp) >> 1)) return SYMGPU_ERR_ARG;
    const symgpu_status st = ve::decode_packet(fe->view, packet, n, slot, floor_base, fe->prev_block_flag, fe->classes, unit, floor_y, residue);
    if (st != SYMGPU_OK) return st;
    fe->prev_block_flag = unit->block_flag;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_vorbis_fe_decode_packets(symgpu_vorbis_fe* fe, const uint8_t* data, size_t n, const symgpu_piece* packets, size_t n_packets,
                                                         uint32_t slot, uint32_t floor_base, symgpu_vorbis_unit* units, uint16_t* floor_y, float* residue,
                                                         uint32_t* packet_of, size_t* n_good) {
    if (!fe || (!data && n) || (n_packets && (!packets || !units || !floor_y || !residue || !packet_of)) || !n_good) return SYMGPU_ERR_ARG;
    if (slot < ((1u << fe->ident.bs1_exp) >> 1)) return SYMGPU_ERR_ARG;
    size_t good = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].len > n - packets[i].offset) continue;
        const symgpu_status st = symgpu_vorbis_fe_decode(fe, data + packets[i].offset, packets[i].len, slot, floor_base, units + good, floor_y + 130 * good,
                                                         residue + 2 * size_t(slot) * good);
        if (st != SYMGPU_OK) continue;  // the caller of the reference drops the packet and goes on
        packet_of[good++] = uint32_t(i);
    }
    *n_good = good;
    return SYMGPU_OK;
}

// A stream's audio packets as independent jobs (DESIGN 10.9): a packet depends on its predecessors only through the previous block
// flag, which is output, not input, of the entropy stage -- the partition-class vector's history never reaches an entry a packet reads
// before writing it, and what a class word writes does not depend on the vector's length beyond the entries it has (the digits kept
// when it is cut are the same most significant ones).  Every thread owns a front-end built from the headers; outputs stay at their
// packet's index (units[i], floor_y[130 i], residue[2 slot i]); accepted[0 .. n_good) lists the packets the reference decodes, in
// order, and the previous block flags are chained over exactly those.
extern "C" symgpu_status symgpu_vorbis_fe_decode_packets_jobs(const uint8_t* ident, size_t n_ident, const uint8_t* setup, size_t n_setup, const uint8_t* data,
                                                              size_t n, const symgpu_piece* packets, size_t n_packets, uint32_t slot, uint32_t floor_base,
                                                              symgpu_vorbis_unit* units, uint16_t* floor_y, float* residue, uint32_t* accepted, size_t* n_good,
                                                              uint32_t n_threads) {
    if (n_good) *n_good = 0;
    if ((!data && n) || (n_packets && (!packets || !units || !floor_y || !residue || !accepted)) || !n_good) return SYMGPU_ERR_ARG;
    n_threads = std::max<uint32_t>(1, std::min<uint32_t>({n_threads, 64u, std::max(1u, std::thread::hardware_concurrency()),
                                                           uint32_t(std::min<size_t>(std::max<size_t>(n_packets, 1), 64))}));
    try { // no C++ exception crosses the ABI (vector / thread creation may throw)
    std::vector<symgpu_vorbis_fe*> fes(n_threads, nullptr);
    symgpu_status st = SYMGPU_OK;
    for (uint32_t t = 0; t < n_threads && st == SYMGPU_OK; ++t) st = symgpu_vorbis_fe_create(ident, n_ident, setup, n_setup, &fes[t]);
    if (st == SYMGPU_OK && slot < ((1u << fes[0]->ident.bs1_exp) >> 1)) st = SYMGPU_ERR_ARG;
    std::vector<uint8_t> ok(n_packets, 0);
    if (st == SYMGPU_OK) {
        std::vector<std::thread> pool;
        for (uint32_t t = 0; t < n_threads; ++t)
            pool.emplace_back([&, t] {
                for (size_t i = t; i < n_packets; i += n_threads) {
                    if (packets[i].offset > n || packets[i].len > n - packets[i].offset) continue;
                    ok[i] = symgpu_vorbis_fe_decode(fes[t], data + packets[i].offset, packets[i].len, slot, floor_base, units + i, floor_y + 130 * i,
                                                    residue + 2 * size_t(slot) * i) == SYMGPU_OK;
                }
            });
        for (auto& th : pool) th.join();
        size_t good = 0;
        int prev = -1;
        for (size_t i = 0; i < n_packets; ++i) {
            if (!ok[i]) {
                std::memset(units + i, 0, sizeof *units);
                continue;
            }
            units[i].prev_block_flag = uint8_t(prev < 0 ? units[i].block_flag : prev);
            prev = units[i].block_flag;
            accepted[good++] = uint32_t(i);
        }
        *n_good = good;
    }
    for (symgpu_vorbis_fe* fe : fes) symgpu_vorbis_fe_destroy(fe);
    return st;
    } catch (...) {
        *n_good = 0;
        return SYMGPU_ERR_LIMIT;
    }
}
