// The Vorbis job build of symgpu_vorbis_heads_dev / symgpu_vorbis_jobs_dev (symphonia_b200/csrc/vorbis_jobs_kernel.cu) run on
// the CPU through the same functions of include/symgpu/packetizer.hpp the kernels call, with the kernels' scans done as loops
// over a table of jobs in which each stream is a segment.  Input on stdin, one request per line:
//   vorbis <data> <packets> <pieces>  (a file's bytes and its symgpu_ogg_packet / symgpu_piece records)
//                                     -> "H n_stream setup ident_len setup_len", "A index len" per audio packet, then
//                                        "J discard trim_end" per audio packet when the headers parse, else "X"
//   trims <streams> (<n> (seq absgp dur discard)*n)*   -> the trim_end values, stream after stream
//   durs <bs0> <bs1> <n_modes> <mask> <streams> (<n> (head head_len)*n)*   -> "dur discard" per packet, stream after stream
#include <cstdio>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/symgpu.h"
#include "../../include/symgpu/packetizer.hpp"

using namespace symgpu::packet;

namespace {

std::vector<uint8_t> slurp(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

// A job table: each job's stream is [first, first + count).
struct Jobs {
    std::vector<uint32_t> first, count, seq;
    std::vector<uint64_t> absgp;
    std::vector<uint8_t> exp;
    void add_stream(size_t n) {
        const uint32_t at = uint32_t(first.size());
        for (size_t k = 0; k < n; ++k) first.push_back(at), count.push_back(uint32_t(n));
    }
};

// vorbis_job_scan_kernel's previous-exponent scan (exclusive max of "job + 1 where the exponent is non-zero") and the time rule.
void times(const Jobs& t, std::vector<uint32_t>& dur, std::vector<uint32_t>& disc) {
    const size_t n = t.first.size();
    dur.assign(n, 0), disc.assign(n, 0);
    uint32_t latest = 0;  // the scan's carry: job + 1 of the latest job with a block before the current one
    for (size_t j = 0; j < n; ++j) {
        const uint8_t prev_exp = latest && latest - 1 >= t.first[j] ? t.exp[latest - 1] : 0;
        uint64_t d, c;
        vorbis_packet_time(prev_exp, t.exp[j], d, c);
        dur[j] = uint32_t(d), disc[j] = uint32_t(c);
        if (t.exp[j]) latest = uint32_t(j + 1);
    }
}

// vorbis_job_scan_kernel's runs and prefix sums, then vorbis_job_trim_kernel for every job.
std::vector<uint32_t> trims(const Jobs& t, const std::vector<uint32_t>& dur, const std::vector<uint32_t>& disc) {
    const size_t n = t.first.size();
    std::vector<uint32_t> run(n), run_head, out(n);
    std::vector<int64_t> dur_sum(n), disc_sum(n);
    int64_t sd = 0, sc = 0;
    for (size_t j = 0; j < n; ++j) {
        if (j == t.first[j] || t.seq[j] != t.seq[j - 1]) run_head.push_back(uint32_t(j));
        run[j] = uint32_t(run_head.size() - 1);
        dur_sum[j] = sd += dur[j], disc_sum[j] = sc += disc[j];
    }
    for (size_t j = 0; j < n; ++j) {
        const uint32_t first = t.first[j], last = first + t.count[j], r = run[j], h = run_head[r];
        const uint32_t next_head = r + 1 < run_head.size() ? run_head[r + 1] : uint32_t(n);
        const int64_t dur_before = h ? dur_sum[h - 1] : 0, disc_before = h ? disc_sum[h - 1] : 0;
        const int64_t tot = dur_sum[next_head - 1] - dur_before, dc = disc_sum[next_head - 1] - disc_before, end = int64_t(t.absgp[h]);
        const bool have_prev = h > first;
        const uint32_t ph = have_prev ? run_head[r - 1] : h;
        const int64_t start = ogg_run_start(have_prev, t.seq[ph], int64_t(t.absgp[ph]), t.seq[h], h == first && next_head == last, tot, dc, end);
        out[j] = ogg_packet_end_trim(start + (dur_sum[j] - dur_before), end, dur[j], disc[j]);
    }
    return out;
}

void vorbis(const std::vector<uint8_t>& d, const std::vector<uint8_t>& pk_bytes, const std::vector<uint8_t>& pc_bytes) {
    std::vector<symgpu_ogg_packet> pk(pk_bytes.size() / sizeof(symgpu_ogg_packet));
    std::vector<symgpu_piece> pc(pc_bytes.size() / sizeof(symgpu_piece));
    if (!pk.empty()) std::memcpy(pk.data(), pk_bytes.data(), pk_bytes.size());
    if (!pc.empty()) std::memcpy(pc.data(), pc_bytes.data(), pc_bytes.size());
    const VorbisStreamHeads h = vorbis_stream_heads(d.data(), pk.data(), uint32_t(pk.size()), pc.data());
    const bool have_setup = h.setup < h.n_stream;
    std::printf("H %u %u %llu %llu\n", h.n_stream, h.setup, pk.empty() ? 0ull : (unsigned long long)pk[0].len,
                have_setup ? (unsigned long long)pk[h.setup].len : 0ull);
    std::vector<uint32_t> audio;
    for (uint32_t k = 0; k < pk.size(); ++k)
        if (vorbis_is_audio(d.data(), pk.data(), pc.data(), h, k)) audio.push_back(k), std::printf("A %u %llu\n", k, (unsigned long long)pk[k].len);
    VorbisIdent id{};
    uint8_t n_modes = 0;
    uint64_t mask = 0;
    auto header = [&](uint32_t k) {
        std::vector<uint8_t> b(pk[k].len);
        ogg_packet_head(d.data(), pc.data() + pk[k].first_piece, pk[k].n_pieces, b.data(), uint32_t(b.size()));
        return b;
    };
    if (!have_setup || vorbis_read_ident(header(0).data(), pk[0].len, id) != Status::Ok ||
        vorbis_read_setup_modes(header(h.setup).data(), pk[h.setup].len, id, n_modes, mask) != Status::Ok) {
        std::printf("X\n");
        return;
    }
    Jobs t;
    t.add_stream(audio.size());
    for (uint32_t k : audio) {
        uint8_t head[2] = {0, 0};
        const uint32_t got = ogg_packet_head(d.data(), pc.data() + pk[k].first_piece, pk[k].n_pieces, head, 2);
        t.exp.push_back(vorbis_packet_exp(head, got, n_modes, mask, id.bs0_exp, id.bs1_exp));
        t.seq.push_back(pk[k].page_sequence), t.absgp.push_back(pk[k].page_absgp);
    }
    std::vector<uint32_t> dur, disc;
    times(t, dur, disc);
    const std::vector<uint32_t> trim = trims(t, dur, disc);
    for (size_t j = 0; j < audio.size(); ++j) std::printf("J %u %u\n", disc[j], trim[j]);
}

}  // namespace

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string mode;
        in >> mode;
        if (mode == "vorbis") {
            std::string a, b, c;
            in >> a >> b >> c;
            vorbis(slurp(a), slurp(b), slurp(c));
        } else if (mode == "trims") {
            size_t streams;
            in >> streams;
            Jobs t;
            std::vector<uint32_t> dur, disc;
            for (size_t s = 0; s < streams; ++s) {
                size_t n;
                in >> n;
                t.add_stream(n);
                for (size_t i = 0; i < n; ++i) {
                    uint32_t sq, du, di;
                    uint64_t gp;
                    in >> sq >> gp >> du >> di;
                    t.seq.push_back(sq), t.absgp.push_back(gp), dur.push_back(du), disc.push_back(di);
                }
            }
            for (uint32_t v : trims(t, dur, disc)) std::printf("%u\n", v);
        } else if (mode == "durs") {
            unsigned bs0, bs1, n_modes;
            unsigned long long mask;
            size_t streams;
            in >> bs0 >> bs1 >> n_modes >> mask >> streams;
            Jobs t;
            for (size_t s = 0; s < streams; ++s) {
                size_t n;
                in >> n;
                t.add_stream(n);
                for (size_t i = 0; i < n; ++i) {
                    unsigned head, head_len;
                    in >> head >> head_len;
                    const uint8_t b[2] = {uint8_t(head & 0xff), uint8_t(head >> 8)};
                    t.exp.push_back(vorbis_packet_exp(b, head_len, uint8_t(n_modes), mask, uint8_t(bs0), uint8_t(bs1)));
                }
            }
            std::vector<uint32_t> dur, disc;
            times(t, dur, disc);
            for (size_t j = 0; j < dur.size(); ++j) std::printf("%u %u\n", dur[j], disc[j]);
        }
        std::printf("end\n");
        std::fflush(stdout);
    }
    return 0;
}
