// MP3 entropy front-end (include/symgpu.h "MP3 entropy front-end", SURVEY §8f N1): the serial, per-stream half of
// the Layer III decoder -- side information, bit reservoir, scale factors, Huffman-coded spectrum -- producing the
// batch format the synthesis kernels consume.  CPU only.
//
// Same results as the reference's reader (symphonia-bundle-mp3/src/layer3/{mod,bitstream,requantize}.rs), different
// construction: the Huffman tables are two-level direct-lookup tables built once from the standard's (code, length)
// lists (mp3_huffman_data.inc), the bit reader is a 64-bit big-endian window that reads zeros past the end of the
// data and reports over-reads by position, and the spectrum is written as int16 sign * x -- the POW43 lookup that the
// reference folds into this loop (requantize.rs:128, :144) runs on the device.
#include <algorithm>
#include <cstring>
#include <new>
#include <thread>
#include <vector>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"
#include "mp3_entropy.h"
#include "tables.h"

namespace {

#include "mp3_huffman_data.inc"

using symgpu::packet::MpaHeader;

// ---------------------------------------------------------------------------------------------- Huffman tables
// Two-level direct lookup: the first kFirstBits bits of the window select either a finished entry or a second-level
// table sized for the longest code under that prefix (entry format: mp3_entropy.h).
constexpr unsigned kFirstBits = 9;

void append_table(std::vector<uint32_t>& lut, uint32_t& base, uint8_t& first_bits, const uint32_t* packed, size_t n, unsigned wrap, bool quad) {
    unsigned max_len = 0;
    for (size_t i = 0; i < n; ++i) max_len = std::max(max_len, packed[i] >> 24);
    const unsigned first = std::min(max_len, kFirstBits);
    base = uint32_t(lut.size()), first_bits = uint8_t(first);
    std::vector<uint32_t> t(size_t(1) << first, 0);
    std::vector<unsigned> deepest(t.size(), 0);  // longest code under each first-level prefix
    for (size_t i = 0; i < n; ++i) {
        const unsigned len = packed[i] >> 24, code = packed[i] & 0x7ffff;
        if (len > first) deepest[code >> (len - first)] = std::max(deepest[code >> (len - first)], len - first);
    }
    for (size_t pfx = 0; pfx < deepest.size(); ++pfx)
        if (deepest[pfx]) {
            t[pfx] = 0x80000000u | uint32_t(t.size()) | (deepest[pfx] << 24);
            t.resize(t.size() + (size_t(1) << deepest[pfx]), 0);
        }
    for (size_t i = 0; i < n; ++i) {
        const unsigned len = packed[i] >> 24, code = packed[i] & 0x7ffff;
        const uint32_t entry = (quad ? unsigned(i) : unsigned(((i / wrap) << 4) | (i % wrap))) | (len << 8);
        if (len <= first) {
            const unsigned pad = first - len;
            for (unsigned k = 0; k < (1u << pad); ++k) t[(code << pad) + k] = entry;
        } else {
            const unsigned rest = len - first, prefix = code >> rest;
            const unsigned sub = (t[prefix] >> 24) & 31, at = t[prefix] & 0xffffff, pad = sub - rest;
            for (unsigned k = 0; k < (1u << pad); ++k) t[at + ((code & ((1u << rest) - 1)) << pad) + k] = entry;
        }
    }
    lut.insert(lut.end(), t.begin(), t.end());
}

struct HostTables {
    std::vector<uint32_t> lut;
    symgpu::mp3e::HuffSet set{};
    HostTables() {
        static const uint8_t linbits[32] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 6, 8, 10, 13, 4, 5, 6, 7, 8, 9, 11, 13};
        std::memcpy(set.linbits, linbits, 32);
#define SYMGPU_BIG(T, W) append_table(lut, set.base[T], set.first_bits[T], kHuff_##T, sizeof(kHuff_##T) / 4, W, false)
        SYMGPU_BIG(1, 2), SYMGPU_BIG(2, 3), SYMGPU_BIG(3, 3), SYMGPU_BIG(5, 4), SYMGPU_BIG(6, 4), SYMGPU_BIG(7, 6), SYMGPU_BIG(8, 6), SYMGPU_BIG(9, 6);
        SYMGPU_BIG(10, 8), SYMGPU_BIG(11, 8), SYMGPU_BIG(12, 8), SYMGPU_BIG(13, 16), SYMGPU_BIG(15, 16), SYMGPU_BIG(16, 16), SYMGPU_BIG(24, 16);
#undef SYMGPU_BIG
        for (int t = 17; t < 24; ++t) set.base[t] = set.base[16], set.first_bits[t] = set.first_bits[16];  // same codes, other linbits
        for (int t = 25; t < 32; ++t) set.base[t] = set.base[24], set.first_bits[t] = set.first_bits[24];
        append_table(lut, set.base[32], set.first_bits[32], kHuff_quadA, 16, 16, true);
        append_table(lut, set.base[33], set.first_bits[33], kHuff_quadB, 16, 16, true);
        set.lut = lut.data();
    }
};
const HostTables& host_tables() {
    static const HostTables t;
    return t;
}

// ---------------------------------------------------------------------------------------------- packet prologue
using symgpu::mp3e::FrameSide;
using symgpu::mp3e::GcJob;

// decoder.rs:84-131: synchronise inside the packet, parse, insist that the packet is exactly one frame of the stream's
// signal specification (fixed by the first packet whose header passes) and of Layer III, skip the CRC; then the side
// information (mp3_entropy.h, the code the device runs).  s.state says how far the packet got.
struct Spec {
    bool have = false;
    uint32_t rate = 0;
    int channels = 0;
};
symgpu_status open_frame(Spec& spec, const uint8_t* frame, size_t n, FrameSide& s) {
    using namespace symgpu::mp3e;
    s = FrameSide{};
    MpaHeader h{};
    size_t q = 0;
    const int hs = read_header(frame, n, h, q);
    if (hs != kDecoded) return hs == kUnsupported ? SYMGPU_ERR_UNSUPPORTED : SYMGPU_ERR_DECODE;
    if (!spec.have) spec.have = true, spec.rate = h.sample_rate, spec.channels = h.n_channels();
    else if (spec.rate != h.sample_rate || spec.channels != h.n_channels()) return SYMGPU_ERR_DECODE;
    uint32_t at = 0, bytes = 0;
    if (!body_of(h, 3, n, q, at, bytes)) return SYMGPU_ERR_DECODE;
    read_frame_side(frame + at, at, bytes, h, symgpu::mp3_long_edges_host(), s);
    return SYMGPU_OK;
}

void frame_info(const FrameSide& s, const symgpu::mp3e::StepOut& o, symgpu_mp3_frame_info* info) {
    static const uint32_t rates[9] = {44100, 48000, 32000, 22050, 24000, 16000, 11025, 12000, 8000};
    *info = symgpu_mp3_frame_info{};
    info->sample_rate = rates[s.sample_rate_idx], info->channels = s.n_ch, info->granules = s.n_gr;
    info->sample_rate_idx = s.sample_rate_idx, info->version = uint8_t(s.mpeg1 ? 0 : s.sample_rate_idx < 6 ? 1 : 2);
    info->underflow_bytes = o.underflow, info->main_data_bytes = o.used;
}

}  // namespace

struct symgpu_mp3_fe {
    uint8_t reservoir[2048];
    size_t len = 0, consumed = 0;
    Spec spec;
    void clear() { len = consumed = 0; }
};

const symgpu::mp3e::LongEdges& symgpu::mp3_long_edges_host() {
    static const mp3e::LongEdges E = [] {
        mp3e::LongEdges e{};
        for (int r = 0; r < 9; ++r)
            for (int k = 0; k < 23; ++k) e.e[r][k] = mp3_tables_host().edges[r][kKindLong][k];
        return e;
    }();
    return E;
}

const symgpu::mp3e::HuffSet& symgpu::mp3_huffset_host(size_t* words) {
    if (words) *words = host_tables().lut.size();
    return host_tables().set;
}

extern "C" symgpu_status symgpu_mp3_fe_create(symgpu_mp3_fe** out) {
    if (!out) return SYMGPU_ERR_ARG;
    host_tables();
    *out = new (std::nothrow) symgpu_mp3_fe();
    return *out ? SYMGPU_OK : SYMGPU_ERR_LIMIT;
}
extern "C" void symgpu_mp3_fe_destroy(symgpu_mp3_fe* fe) { delete fe; }
extern "C" void symgpu_mp3_fe_reset(symgpu_mp3_fe* fe) {
    if (fe) fe->clear(), fe->spec = Spec{};
}

extern "C" symgpu_status symgpu_mp3_fe_decode(symgpu_mp3_fe* fe, const uint8_t* frame, size_t n, symgpu_mp3_gc* units, int16_t* quant,
                                              symgpu_mp3_frame_info* info) {
    using namespace symgpu::mp3e;
    if (!fe || (!frame && n) || !units || !quant) return SYMGPU_ERR_ARG;
    FrameSide s;
    {
        const symgpu_status hs = open_frame(fe->spec, frame, n, s);
        if (hs != SYMGPU_OK) return hs;
    }
    // the reservoir step of the plan (mp3_entropy.h), then its jobs run in order against the reservoir's bytes
    Reservoir r{uint32_t(fe->len), uint32_t(fe->consumed), fe->len};
    GcJob jobs[4];
    StepOut o{};
    if (reservoir_step(r, s, 0, 0, jobs, o) != kStepDecoded) return fe->len = r.len, fe->consumed = r.consumed, SYMGPU_ERR_DECODE;
    std::memmove(fe->reservoir, fe->reservoir + fe->len - o.reuse, o.reuse);  // BitResevoir::fill (mod.rs:42-95)
    std::memcpy(fe->reservoir + o.reuse, frame + s.body_at + s.side_len, o.slot);
    fe->len = r.len, fe->consumed = r.consumed;
    const HuffSet& hs = host_tables().set;
    int failed = 0;
    for (int k = 0; k < 4; ++k) {
        jobs[k].seg_begin = 0;
        failed |= decode_gc_job(jobs[k], fe->reservoir, hs, units + k, quant + k * 576);
    }
    if (failed) return fe->clear(), SYMGPU_ERR_DECODE;
    if (info) frame_info(s, o, info);
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_mp3_fe_decode_packets(symgpu_mp3_fe* fe, const uint8_t* data, size_t n, const symgpu_mpa_packet* packets,
                                                      size_t n_packets, symgpu_mp3_gc* units, int16_t* quant, uint32_t* frame_of,
                                                      size_t* n_good, symgpu_mp3_frame_info* info) {
    if (!fe || !data || !n_good || (n_packets && (!packets || !units || !quant || !frame_of))) return SYMGPU_ERR_ARG;
    size_t good = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].size > n - packets[i].offset) return SYMGPU_ERR_ARG;
        symgpu_mp3_frame_info fi;
        if (symgpu_mp3_fe_decode(fe, data + packets[i].offset, packets[i].size, units + good * 4, quant + good * 4 * 576, &fi) != SYMGPU_OK) continue;
        if (good == 0 && info) *info = fi;
        frame_of[good++] = uint32_t(i);
    }
    *n_good = good;
    return SYMGPU_OK;
}

// ---------------------------------------------------------------------------------------------- plan + jobs
static_assert(sizeof(symgpu_mp3_gc_job) == sizeof(symgpu::mp3e::GcJob), "the public job record is the GcJob");

extern "C" symgpu_status symgpu_mp3_entropy_plan(const uint8_t* data, size_t n, const symgpu_mpa_packet* packets, size_t n_packets,
                                                 const uint8_t* bad, uint8_t* md, size_t md_cap, size_t* md_len, symgpu_mp3_gc_job* jobs_out,
                                                 uint32_t* frame_of, size_t* n_good, symgpu_mp3_frame_info* info) {
    using namespace symgpu::mp3e;
    if ((!data && n) || (n_packets && !packets) || !md_len || !n_good || (!md && md_cap)) return SYMGPU_ERR_ARG;
    GcJob* jobs = reinterpret_cast<GcJob*>(jobs_out);
    Spec spec;
    Reservoir r{0, 0, 0};  // the reservoir, as byte counts only
    size_t good = 0;
    for (size_t i = 0; i < n_packets; ++i) {
        if (packets[i].offset > n || packets[i].size > n - packets[i].offset) return SYMGPU_ERR_ARG;
        const uint8_t* frame = data + packets[i].offset;
        FrameSide s;
        if (open_frame(spec, frame, packets[i].size, s) != SYMGPU_OK) continue;
        GcJob four[4];
        StepOut o{};
        const int step = reservoir_step(r, s, bad ? bad[i] : 0, uint32_t(good), four, o);
        if (step != kStepDecoded && step != kStepLeftOut) continue;
        if (o.copy_at + o.slot > md_cap) return SYMGPU_ERR_LIMIT;
        if (md) std::memcpy(md + o.copy_at, frame + s.body_at + s.side_len, o.slot);
        if (step == kStepLeftOut) continue;  // refused AFTER its main data was read (stereo.rs:503-505): the reservoir moves on, no audio
        if (jobs) std::memcpy(jobs + good * 4, four, sizeof four);
        if (good == 0 && info) frame_info(s, o, info);
        if (frame_of) frame_of[good] = uint32_t(i);
        ++good;
    }
    *md_len = r.md_at, *n_good = good;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_mp3_entropy_run_cpu(const uint8_t* md, size_t md_len, const symgpu_mp3_gc_job* jobs_in, size_t n_jobs,
                                                    symgpu_mp3_gc* units, int16_t* quant, uint8_t* failed) {
    using namespace symgpu::mp3e;
    if ((n_jobs && (!jobs_in || !units || !quant)) || (!md && md_len)) return SYMGPU_ERR_ARG;
    const GcJob* jobs = reinterpret_cast<const GcJob*>(jobs_in);
    const HuffSet& hs = host_tables().set;
    const uint32_t first = n_jobs ? jobs[0].out_index & ~3u : 0;
    for (size_t k = 0; k < n_jobs; ++k) {
        const GcJob& j = jobs[k];
        if (j.out_index < first || j.seg_begin > md_len || j.seg_len > md_len - j.seg_begin) return SYMGPU_ERR_ARG;
        const uint32_t slot = j.out_index - first;
        if (decode_gc_job(j, md, hs, units + slot, quant + size_t(slot) * 576) && failed) failed[slot >> 2] = 1;
    }
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_mp3_entropy_run_cpu_mt(const uint8_t* md, size_t md_len, const symgpu_mp3_gc_job* jobs, size_t n_jobs,
                                                       symgpu_mp3_gc* units, int16_t* quant, uint8_t* failed, uint32_t n_threads) {
    if (n_jobs % 4) return SYMGPU_ERR_ARG;
    const size_t n_frames = n_jobs / 4;
    if (n_threads == 0) n_threads = std::max(1u, std::thread::hardware_concurrency());
    n_threads = uint32_t(std::min<size_t>(n_threads, std::max<size_t>(n_frames, 1)));
    if (n_threads <= 1) return symgpu_mp3_entropy_run_cpu(md, md_len, jobs, n_jobs, units, quant, failed);
    host_tables();  // built before the threads start
    std::vector<symgpu_status> status(n_threads, SYMGPU_OK);
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < n_threads; ++t)
        pool.emplace_back([&, t] {
            const size_t a = n_frames * t / n_threads, b = n_frames * (t + 1) / n_threads;  // whole frames: a job's slot is relative to its range's first frame
            status[t] = symgpu_mp3_entropy_run_cpu(md, md_len, jobs + a * 4, (b - a) * 4, units + a * 4, quant + a * 4 * 576, failed ? failed + a : nullptr);
        });
    for (auto& th : pool) th.join();
    for (symgpu_status s : status)
        if (s != SYMGPU_OK) return s;
    return SYMGPU_OK;
}

extern "C" symgpu_status symgpu_mp3_entropy_decode_cpu(const uint8_t* data, size_t n, const symgpu_mpa_packet* packets, size_t n_packets,
                                                       symgpu_mp3_gc* units, int16_t* quant, uint32_t* frame_of, size_t* n_good,
                                                       symgpu_mp3_frame_info* info, uint32_t* n_rounds) {
    if ((!data && n) || !n_good || (n_packets && (!packets || !units || !quant || !frame_of))) return SYMGPU_ERR_ARG;
    size_t total = 0;
    for (size_t i = 0; i < n_packets; ++i) total += packets[i].size;
    std::vector<uint8_t> md(total + 8), bad(n_packets, 0), failed;
    std::vector<symgpu_mp3_gc_job> jobs(n_packets * 4);
    uint32_t rounds = 0;
    for (;;) {
        ++rounds;
        size_t md_len = 0, good = 0;
        const symgpu_status s = symgpu_mp3_entropy_plan(data, n, packets, n_packets, bad.data(), md.data(), md.size(), &md_len, jobs.data(), frame_of, &good, info);
        if (s != SYMGPU_OK) return s;
        failed.assign(good, 0);
        const symgpu_status r = symgpu_mp3_entropy_run_cpu(md.data(), md_len, jobs.data(), good * 4, units, quant, failed.data());
        if (r != SYMGPU_OK) return r;
        // only the FIRST failure is certain: frames behind it were planned with a reservoir the reference would have emptied
        size_t first_bad = good;
        for (size_t f = 0; f < good; ++f)
            if (failed[f]) {
                first_bad = f;
                break;
            }
        if (first_bad == good) {
            *n_good = good;
            break;
        }
        bad[frame_of[first_bad]] = 1;
    }
    if (n_rounds) *n_rounds = rounds;
    return SYMGPU_OK;
}
