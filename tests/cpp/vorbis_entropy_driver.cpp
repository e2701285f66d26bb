// Host driver of the shared Vorbis packet rules (symphonia_b200/csrc/vorbis_entropy.h), for tests/test_vorbis_entropy_shared.py.
// Built with -ffp-contract=off, and in a second build with AddressSanitizer + UndefinedBehaviorSanitizer.
//
//   vorbis_entropy_driver IN SEED
// IN: u32 n_files; per file u32 ident_len, ident, u32 setup_len, setup, u32 n_packets, per packet u32 len, len bytes.
// Runs every file twice:
//   1. symgpu_vorbis_fe_decode_packets over the file's packets in order (the library's serial front-end);
//   2. the device's schedule (vorbis_decode_kernel.cu) on the CPU: the setup in flat form (setup_export), every packet of every
//      file decoded by decode_packet in an order shuffled with SEED, each with a fresh partition-class buffer of exactly the
//      setup's class_cap bytes and its packet in a buffer of exactly its length; then the previous block flags chained over each
//      file's decoded packets in stream order.
// The decoded packets must be the same, and for each its unit, floor_y and residue bits.  Prints "decoded refused" counts; exit
// status 1 and a message at the first difference.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../symphonia_b200/csrc/vorbis_entropy.h"

namespace {

namespace ve = symgpu::vorbise;

struct File {
    std::vector<uint8_t> ident, setup;
    std::vector<std::vector<uint8_t>> packets;
};

struct Job {
    uint32_t file, packet;
    symgpu_status st = SYMGPU_ERR_DECODE;
    symgpu_vorbis_unit unit{};
    std::vector<uint16_t> floor_y;
    std::vector<float> residue;
};

uint32_t u32_at(const std::vector<uint8_t>& in, size_t& at) {
    uint32_t v;
    std::memcpy(&v, in.data() + at, 4);
    at += 4;
    return v;
}
std::vector<uint8_t> bytes_at(const std::vector<uint8_t>& in, size_t& at) {
    const uint32_t n = u32_at(in, at);
    std::vector<uint8_t> v(in.begin() + long(at), in.begin() + long(at + n));
    at += n;
    return v;
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
        FILE* f = std::fopen(argv[1], "rb");
        if (!f) return 2;
        int c;
        while ((c = std::fgetc(f)) != EOF) in.push_back(uint8_t(c));
        std::fclose(f);
    }
    size_t at = 0;
    std::vector<File> files(u32_at(in, at));
    for (File& f : files) {
        f.ident = bytes_at(in, at), f.setup = bytes_at(in, at);
        f.packets.resize(u32_at(in, at));
        for (auto& p : f.packets) p = bytes_at(in, at);
    }
    // the device's schedule: flat setups, jobs in a shuffled order
    std::vector<std::vector<uint8_t>> blobs(files.size());
    std::vector<ve::SetupHead> heads(files.size());
    std::vector<uint32_t> slots(files.size());
    std::vector<Job> jobs;
    for (uint32_t f = 0; f < files.size(); ++f) {
        symgpu_vorbis_fe* fe = nullptr;
        if (symgpu_vorbis_fe_create(files[f].ident.data(), files[f].ident.size(), files[f].setup.data(), files[f].setup.size(), &fe) != SYMGPU_OK)
            return fail("setup refused", f, 0);
        ve::setup_export(fe, blobs[f], heads[f]);
        symgpu_vorbis_fe_destroy(fe);
        slots[f] = (1u << heads[f].bs1_exp) >> 1;
        for (uint32_t p = 0; p < files[f].packets.size(); ++p) jobs.push_back(Job{f, p});
    }
    std::vector<size_t> order(jobs.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::shuffle(order.begin(), order.end(), std::mt19937(uint32_t(std::atoi(argv[2]))));
    for (size_t i : order) {
        Job& j = jobs[i];
        const ve::SetupHead& h = heads[j.file];
        const ve::Setup S = ve::view_of(blobs[j.file].data(), h);
        const std::vector<uint8_t> packet(files[j.file].packets[j.packet]);  // exactly the packet
        std::vector<uint8_t> classes(h.class_cap);                           // fresh, exactly the setup's size
        ve::ClassBuf cls{classes.data(), 0, h.class_cap};
        j.floor_y.assign(130, 0xdead), j.residue.assign(2 * size_t(slots[j.file]), -1.0f);
        j.st = ve::decode_packet(S, packet.data(), packet.size(), slots[j.file], 0, -1, cls, &j.unit, j.floor_y.data(), j.residue.data());
    }
    uint32_t decoded = 0, refused = 0;
    size_t first_job = 0;
    for (uint32_t f = 0; f < files.size(); ++f) {
        const File& F = files[f];
        const size_t n = F.packets.size();
        // the serial front-end over the same packets, back to back
        std::vector<uint8_t> data;
        std::vector<symgpu_piece> pieces(n);
        for (size_t p = 0; p < n; ++p) {
            pieces[p] = symgpu_piece{data.size(), uint32_t(F.packets[p].size()), 0};
            data.insert(data.end(), F.packets[p].begin(), F.packets[p].end());
        }
        symgpu_vorbis_fe* fe = nullptr;
        if (symgpu_vorbis_fe_create(F.ident.data(), F.ident.size(), F.setup.data(), F.setup.size(), &fe) != SYMGPU_OK) return fail("setup refused", f, 0);
        const uint32_t slot = slots[f];
        std::vector<symgpu_vorbis_unit> units(n);
        std::vector<uint16_t> fy(130 * n);
        std::vector<float> res(2 * size_t(slot) * n);
        std::vector<uint32_t> packet_of(n);
        size_t good = 0;
        const symgpu_status st = symgpu_vorbis_fe_decode_packets(fe, data.data(), data.size(), pieces.data(), n, slot, 0, units.data(), fy.data(), res.data(),
                                                                 packet_of.data(), &good);
        symgpu_vorbis_fe_destroy(fe);
        if (st != SYMGPU_OK) return fail("decode_packets", f, 0);
        // previous block flags chained over the decoded packets, in stream order
        int prev = -1;
        size_t g = 0;
        for (uint32_t p = 0; p < n; ++p) {
            Job& j = jobs[first_job + p];
            const bool ok = j.st == SYMGPU_OK;
            const bool want = g < good && packet_of[g] == p;
            if (ok != want) return fail("status", f, p);
            if (!ok) {
                ++refused;
                continue;
            }
            j.unit.prev_block_flag = uint8_t(prev < 0 ? j.unit.block_flag : prev);
            prev = j.unit.block_flag;
            if (std::memcmp(&j.unit, &units[g], sizeof j.unit)) return fail("unit", f, p);
            if (std::memcmp(j.floor_y.data(), fy.data() + 130 * g, 130 * sizeof(uint16_t))) return fail("floor_y", f, p);
            if (std::memcmp(j.residue.data(), res.data() + 2 * size_t(slot) * g, 2 * size_t(slot) * sizeof(float))) return fail("residue", f, p);
            ++g, ++decoded;
        }
        first_job += n;
    }
    std::printf("%u %u\n", decoded, refused);
    return 0;
}
