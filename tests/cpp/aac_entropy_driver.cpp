// Host driver of the shared AAC-LC packet rules (symphonia_b200/csrc/aac_entropy.h), for tests/test_aac_entropy_shared.py.
// Built with -ffp-contract=off and -DSYMGPU_MP3E_DEVICE_WINDOW (the bit window the device composes from byte loads), and in a
// second build with AddressSanitizer + UndefinedBehaviorSanitizer.
//
//   aac_entropy_driver IN SEED
// IN: u32 n_files; per file u32 sample_rate, u32 channels, u32 n_packets, per packet u32 len, len bytes.
// Runs every file twice:
//   1. symgpu_aac_fe_decode packet by packet, in order, one front-end per file (the library);
//   2. the device's schedule (aac_decode_kernel.cu) on the CPU: pass A -- decode_job from a fresh state -- over every packet of
//      every file in an order shuffled with SEED, into coefficient buffers that start at zero; walk_step over each file's
//      records in order; pass B -- decode_job again, from the walk's generator states -- for the decoded packets that drew
//      noise; the pulse step with the scale factors the walk named and pulse_apply.
// Each packet lives in a buffer of exactly its length.  Per packet the status, and for a decoded one its units (with the
// walk's prev_window_shape), the TNS records each unit names and the coefficient bits, must be equal.  Prints
// "decoded refused unsupported redecoded pulses stale" counts; exit status 1 and a message at the first difference.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include "../../symphonia_b200/csrc/aac_entropy.h"

namespace {

namespace ae = symgpu::aace;

struct Job {
    std::vector<uint8_t> bytes;  // exactly the packet
    uint32_t file = 0;
    std::unique_ptr<ae::JobState> state{new ae::JobState()};
    symgpu_aac_unit units[2];
    symgpu_aac_tns tns[16];
    std::vector<float> coeffs = std::vector<float>(2048, 0.0f);
    ae::PulseLines pulse[2];
    float scales0[128] = {};
    ae::WalkOut walk{};
};

struct File {
    uint32_t rate, channels, rate_idx, first, n;
};

uint32_t u32_at(const std::vector<uint8_t>& in, size_t& at) {
    uint32_t v;
    std::memcpy(&v, in.data() + at, 4);
    at += 4;
    return v;
}

uint8_t status_of(int st) { return st == SYMGPU_OK ? SYMGPU_AAC_JOB_DECODED : st == SYMGPU_ERR_UNSUPPORTED ? SYMGPU_AAC_JOB_UNSUPPORTED : SYMGPU_AAC_JOB_REFUSED; }

void decode(Job& j, const File& f, const uint32_t start[2], bool pass_a) {
    ae::JobOut o{j.units, j.tns, j.coeffs.data(), j.pulse, j.scales0};
    ae::decode_job(j.bytes.data(), j.bytes.size(), symgpu::aac_tables_host(), f.rate_idx, f.channels, start, pass_a, *j.state, o);
}

int fail(const char* what, uint32_t file, uint32_t packet) {
    std::printf("MISMATCH %s: file %u packet %u\n", what, file, packet);
    return 1;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    std::vector<uint8_t> in;
    {
        FILE* fp = std::fopen(argv[1], "rb");
        if (!fp) return 2;
        uint8_t buf[65536];
        for (size_t n; (n = std::fread(buf, 1, sizeof buf, fp)) > 0;) in.insert(in.end(), buf, buf + n);
        std::fclose(fp);
    }
    size_t at = 0;
    const uint32_t n_files = u32_at(in, at);
    std::vector<File> files;
    std::vector<Job> jobs;
    for (uint32_t i = 0; i < n_files; ++i) {
        File f;
        f.rate = u32_at(in, at), f.channels = u32_at(in, at), f.n = u32_at(in, at);
        f.rate_idx = symgpu::aac_rate_index(f.rate), f.first = uint32_t(jobs.size());
        for (uint32_t k = 0; k < f.n; ++k) {
            const uint32_t len = u32_at(in, at);
            jobs.emplace_back();
            jobs.back().bytes.assign(in.begin() + long(at), in.begin() + long(at + len));
            jobs.back().file = i;
            at += len;
        }
        files.push_back(f);
    }
    // pass A, shuffled
    std::vector<uint32_t> order(jobs.size());
    for (uint32_t k = 0; k < order.size(); ++k) order[k] = k;
    std::shuffle(order.begin(), order.end(), std::mt19937(uint32_t(std::atoi(argv[2]))));
    const uint32_t seeds[2] = {ae::kLcgSeed, ae::kLcgSeed};
    for (uint32_t k : order) decode(jobs[k], files[jobs[k].file], seeds, true);
    // the walk, one file after the other
    for (const File& f : files) {
        ae::WalkState w;
        ae::walk_begin(w);
        for (uint32_t k = f.first; k < f.first + f.n; ++k) jobs[k].walk = ae::walk_step(w, jobs[k].state->rec, k, jobs[k].pulse);
    }
    // pass B, shuffled
    long redecoded = 0, pulses = 0, stale = 0;
    for (uint32_t k : order) {
        Job& j = jobs[k];
        if (j.walk.status != SYMGPU_OK || (j.state->rec.draws[0] == 0 && j.state->rec.draws[1] == 0)) continue;
        decode(j, files[j.file], j.walk.lcg_start, false);
        ++redecoded;
    }
    // the pulse step
    for (uint32_t k = 0; k < jobs.size(); ++k) {
        Job& j = jobs[k];
        if (j.walk.status != SYMGPU_OK) continue;
        for (uint32_t c = 0; c < files[j.file].channels; ++c) {
            const ae::PulseLines& p = j.pulse[c];
            if (!p.n) continue;
            float value[4], scale[4];
            for (uint32_t i = 0; i < p.n; ++i) {
                const uint32_t src = j.walk.scale_src[c][i];
                value[i] = j.coeffs[1024 * c + p.line[i]];
                scale[i] = src == ae::kNoJob ? 0.0f : jobs[src].scales0[64 * c + p.band[i]];
                stale += src != k;
            }
            ae::pulse_apply(p, scale, value);
            for (uint32_t i = 0; i < p.n; ++i) j.coeffs[1024 * c + p.line[i]] = value[i];
            ++pulses;
        }
    }
    // against the library, packet by packet
    long count[3] = {0, 0, 0};
    for (uint32_t fi = 0; fi < n_files; ++fi) {
        const File& f = files[fi];
        symgpu_aac_fe* fe = nullptr;
        if (symgpu_aac_fe_create(f.rate, f.channels, &fe) != SYMGPU_OK) return fail("create", fi, 0);
        for (uint32_t i = 0; i < f.n; ++i) {
            Job& j = jobs[f.first + i];
            symgpu_aac_unit units[2];
            symgpu_aac_tns tns[16];
            uint32_t n_tns = 0;
            std::vector<float> coeffs(2048);
            const int st = symgpu_aac_fe_decode(fe, j.bytes.data(), j.bytes.size(), 0, units, tns, &n_tns, coeffs.data());
            const uint8_t want = status_of(st), got = status_of(j.walk.status);
            ++count[want];
            if (want != got) return fail("status", fi, i);
            if (st != SYMGPU_OK) continue;
            for (uint32_t c = 0; c < 2; ++c) {
                symgpu_aac_unit u{};
                if (c < f.channels) u = j.units[c], u.prev_window_shape = uint8_t(j.walk.prev_shape >> c & 1);
                const symgpu_aac_unit& r = units[c];
                if (u.window_sequence != r.window_sequence || u.window_shape != r.window_shape || u.prev_window_shape != r.prev_window_shape ||
                    u.n_tns != r.n_tns || u.reserved[0] != r.reserved[0] || u.reserved[1] != r.reserved[1])
                    return fail("unit", fi, i);
                for (uint32_t t = 0; t < r.n_tns; ++t)
                    if (std::memcmp(&j.tns[8 * c + t], &tns[r.tns_first + t], sizeof(symgpu_aac_tns))) return fail("tns", fi, i);
                for (uint32_t l = 0; l < 1024; ++l) {
                    const float g = c < f.channels ? j.coeffs[1024 * c + l] : 0.0f;
                    if (std::memcmp(&g, &coeffs[1024 * c + l], 4)) return fail("coefficients", fi, i);
                }
            }
        }
        symgpu_aac_fe_destroy(fe);
    }
    std::printf("%ld %ld %ld %ld %ld %ld\n", count[0], count[1], count[2], redecoded, pulses, stale);
    return 0;
}
