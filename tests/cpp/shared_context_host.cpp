// Many decoders of every codec on ONE context (include/symgpu/decoder.hpp), the server shape: one decoder thread per file, every
// decoder made by the registry, every decode() one packet.  The files are read as decoder_host's `file` modes read them, and each
// file's PCM is written as those modes write it, so the two can be compared byte for byte.
//   shared_context_host files KIND:IN ...        GPU tier: every decoder on ONE context; PCM of each file to IN.pcm, batch statistics
//                                                per codec (KIND 1 | 2 | 3 | mpa | aac | vorbis)
//   shared_context_host files-apart KIND:IN ...  the same with a context per thread (no launch shared), for comparison
//   shared_context_host open vorbis N IN         GPU tier: Vorbis decoders on a context of N slots until the registry refuses one
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../../include/symgpu/decoder.hpp"
#include "../../include/symgpu/packetizer.hpp"

using namespace symgpu_host;

// One input file, indexed and cut into the packets a demuxer would hand to decode(), with its codec parameters.
struct Job {
    AudioCodecParameters params;
    std::vector<uint8_t> bytes;
    std::vector<std::vector<uint8_t>> owned;  // Ogg: packets gathered from their pages
    std::vector<Packet> packets;
    uint32_t delay = 0, padding = 0;          // MPEG audio: the tag's gapless values
};

static std::vector<uint8_t> read_file(const char* path) {
    std::ifstream in(path, std::ios::binary);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

// MPEG audio: layer 0 takes the layer of the first frame.
static int load_mpa(int layer, const char* path, Job& job) {
    job.bytes = read_file(path);
    symgpu::packet::MpaTrack track;
    std::vector<symgpu::packet::MpaPacket> packets;
    if (symgpu::packet::MpaIndexer::index(job.bytes.data(), job.bytes.size(), track, packets) != symgpu::packet::Status::Ok) return 5;
    if (layer == 0) layer = track.first.layer;
    job.params.codec = layer == 1 ? CODEC_ID_MP1 : layer == 2 ? CODEC_ID_MP2 : CODEC_ID_MP3;
    job.params.sample_rate = track.first.sample_rate;
    job.params.channels = (uint32_t)track.first.n_channels();
    job.delay = track.delay, job.padding = track.padding;
    for (const auto& pk : packets) {
        Packet p;
        p.data = job.bytes.data() + pk.offset, p.len = pk.size, p.pts = (uint64_t)pk.pts, p.dur = pk.dur;
        p.trim_start = pk.trim_start, p.trim_end = (uint32_t)std::min<uint64_t>(pk.trim_end, pk.dur);
        job.packets.push_back(p);
    }
    return 0;
}

static int load_adts(const char* path, Job& job) {
    job.bytes = read_file(path);
    size_t count = 0;
    symgpu_status stop;
    if (symgpu_adts_index(job.bytes.data(), job.bytes.size(), nullptr, 0, &count, &stop) != SYMGPU_OK || count == 0) return 5;
    std::vector<symgpu_adts_packet> packets(count);
    symgpu_adts_index(job.bytes.data(), job.bytes.size(), packets.data(), count, &count, &stop);
    job.params.codec = CODEC_ID_AAC, job.params.sample_rate = packets[0].sample_rate, job.params.channels = packets[0].channels;
    for (const auto& pk : packets) {
        Packet p;
        p.data = job.bytes.data() + pk.offset, p.len = pk.size, p.pts = (uint64_t)pk.pts, p.dur = 1024;
        job.packets.push_back(p);
    }
    return 0;
}

// Pages -> packets -> mapping (durations, discards, end trims against the page granule positions).
static int load_ogg_vorbis(const char* path, Job& job) {
    using namespace symgpu::packet;
    job.bytes = read_file(path);
    OggIndex ix;
    OggIndex::build(job.bytes.data(), job.bytes.size(), ix, false);
    if (ix.streams.empty()) return 5;
    auto& stream = ix.streams.begin()->second;
    OggVorbisMapper mapper;
    std::vector<uint32_t> seq, dur, discard;
    std::vector<uint64_t> absgp;
    bool first = true;
    for (const OggPacket& pk : stream.packets()) {
        std::vector<uint8_t> b(pk.len);
        stream.gather(job.bytes.data(), pk, b.data());
        if (first) {
            first = false;
            if (!mapper.detect(b.data(), b.size())) return 6;
            continue;
        }
        const auto m = mapper.map(b.data(), b.size());
        if (m.kind != OggVorbisMapper::Kind::Audio || !mapper.ready()) continue;
        seq.push_back(pk.page_sequence), absgp.push_back(pk.page_absgp), dur.push_back((uint32_t)m.dur), discard.push_back((uint32_t)m.discard);
        job.owned.push_back(std::move(b));
    }
    std::vector<uint32_t> trim_end(job.owned.size());
    symgpu_ogg_page_end_trims(seq.data(), absgp.data(), dur.data(), discard.data(), job.owned.size(), trim_end.data());
    job.params.codec = CODEC_ID_VORBIS, job.params.sample_rate = mapper.ident().sample_rate, job.params.channels = mapper.ident().n_channels;
    job.params.extra_data = mapper.extra_data();
    for (size_t k = 0; k < job.owned.size(); ++k) {
        Packet p;
        p.data = job.owned[k].data(), p.len = job.owned[k].size(), p.dur = dur[k], p.trim_start = discard[k], p.trim_end = trim_end[k];
        job.packets.push_back(p);
    }
    return 0;
}

static int load_job(const std::string& kind, const char* path, Job& job) {
    if (kind == "aac") return load_adts(path, job);
    if (kind == "vorbis") return load_ogg_vorbis(path, job);
    return load_mpa(kind == "mpa" ? 0 : std::atoi(kind.c_str()), path, job);
}

// A decoder from the registry, then decode() per packet; the planes of every decoded packet go to `out` one after the other.  A
// refused packet yields no audio and the stream goes on (what a player does).
struct Decoded {
    size_t good = 0, samples = 0;
};
static int decode_job(const CodecRegistry& reg, const Job& job, std::vector<char>& out, Decoded& d, const std::function<void()>& ready = {}) {
    auto dec = reg.make_audio_decoder(job.params, AudioDecoderOptions{});  // gapless: the packets' trims are applied
    if (ready) ready();
    if (!dec.ok()) {
        std::fprintf(stderr, "%s\n", dec.error.message);
        return 3;
    }
    for (const Packet& p : job.packets) {
        auto res = dec.value->decode(p);
        if (!res.ok()) continue;
        ++d.good, d.samples += res.value.frames;
        for (size_t ch = 0; ch < res.value.n_planes; ++ch) {
            const char* b = reinterpret_cast<const char*>(res.value.planes[ch]);
            out.insert(out.end(), b, b + res.value.frames * sizeof(float));
        }
    }
    return 0;
}

// Many files, one decoder thread per file, every decoder from one registry on ONE context (the server shape): each thread decodes
// its file packet by packet and its PCM goes to IN.pcm as in the single-file mode.  With `apart`, every thread builds a context and
// a registry of its own instead (one decoder per context: no launch is shared).  The timed window starts when every decoder is
// open and ends when the last thread has decoded its last packet.
static int run_files(bool apart, const std::vector<std::pair<std::string, std::string>>& files) {
    const size_t n = files.size();
    std::vector<Job> jobs(n);
    for (size_t i = 0; i < n; ++i)
        if (int rc = load_job(files[i].first, files[i].second.c_str(), jobs[i])) {
            std::fprintf(stderr, "cannot index %s\n", files[i].second.c_str());
            return rc;
        }
    std::shared_ptr<GpuContext> shared;
    CodecRegistry shared_reg;
    if (!apart) {
        auto gpu = GpuContext::create(0, (uint32_t)n);
        if (!gpu.ok()) {
            std::fprintf(stderr, "%s\n", gpu.error.message);
            return 2;
        }
        shared = gpu.value;
        register_gpu_decoders(shared_reg, shared);
    }
    std::vector<std::vector<char>> pcm(n);
    std::vector<Decoded> done(n);
    std::vector<int> rc(n, 0);
    std::mutex m;
    std::condition_variable cv;
    size_t opened = 0;
    std::chrono::steady_clock::time_point t0;
    auto ready = [&] {  // every decoder is open before the first packet is decoded
        std::unique_lock<std::mutex> lk(m);
        if (++opened == n) {
            t0 = std::chrono::steady_clock::now();
            cv.notify_all();
        }
        cv.wait(lk, [&] { return opened == n; });
    };
    std::vector<std::thread> threads;
    for (size_t i = 0; i < n; ++i)
        threads.emplace_back([&, i] {
            if (!apart) {
                rc[i] = decode_job(shared_reg, jobs[i], pcm[i], done[i], ready);
                return;
            }
            auto gpu = GpuContext::create(0, 2);
            if (!gpu.ok()) {
                rc[i] = 2;
                ready();
                return;
            }
            CodecRegistry reg;
            register_gpu_decoders(reg, gpu.value);
            rc[i] = decode_job(reg, jobs[i], pcm[i], done[i], ready);
        });
    for (auto& t : threads) t.join();
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    size_t packets = 0, good = 0;
    int failed = 0;
    for (size_t i = 0; i < n; ++i) {
        std::ofstream(files[i].second + ".pcm", std::ios::binary).write(pcm[i].data(), (std::streamsize)pcm[i].size());
        packets += jobs[i].packets.size(), good += done[i].good;
        failed += rc[i] != 0;
    }
    std::printf("files %zu packets %zu decoded %zu seconds %.4f packets_per_s %.0f failed %d\n", n, packets, good, sec, (double)packets / sec, failed);
    if (shared) {
        static const char* names[] = {"mp3", "mp1", "mp2", "aac", "vorbis"};
        for (int c = SYMGPU_CODEC_MP3; c <= SYMGPU_CODEC_VORBIS; ++c) {
            uint64_t batches = 0, frames = 0;
            symgpu_async_stats(shared->raw(), c, &batches, &frames);
            if (frames)
                std::printf("codec %s batches %llu frames %llu frames_per_batch %.2f\n", names[c], (unsigned long long)batches,
                            (unsigned long long)frames, (double)frames / (double)batches);
        }
    }
    return failed ? 4 : 0;
}

// Opens Vorbis decoders for one Ogg file on a context of N slots until the registry refuses one: prints how many opened and why
// the next one was refused.
static int run_open_vorbis(int n_slots, const char* in_path) {
    Job job;
    if (int rc = load_ogg_vorbis(in_path, job)) return rc;
    auto gpu = GpuContext::create(0, (uint32_t)n_slots);
    if (!gpu.ok()) {
        std::fprintf(stderr, "%s\n", gpu.error.message);
        return 2;
    }
    CodecRegistry reg;
    register_gpu_decoders(reg, gpu.value);
    std::vector<std::unique_ptr<AudioDecoder>> open;
    Error refused;
    for (;;) {
        auto dec = reg.make_audio_decoder(job.params, AudioDecoderOptions{});
        if (!dec.ok()) {
            refused = dec.error;
            break;
        }
        open.push_back(std::move(dec.value));
    }
    std::printf("opened %zu refused %s\n", open.size(), refused.kind == ErrorKind::LimitError ? "LimitError" : refused.message);
    // every open decoder still decodes its packets
    int bad = 0;
    for (auto& d : open)
        for (size_t k = 0; k < std::min<size_t>(job.packets.size(), 2); ++k) bad += !d->decode(job.packets[k]).ok();
    std::printf("decode failures %d\n", bad);
    return bad ? 4 : 0;
}

int main(int argc, char** argv) {
    if (argc >= 5 && std::string(argv[1]) == "open" && std::string(argv[2]) == "vorbis") return run_open_vorbis(std::atoi(argv[3]), argv[4]);
    if (argc >= 3 && (std::string(argv[1]) == "files" || std::string(argv[1]) == "files-apart")) {
        std::vector<std::pair<std::string, std::string>> files;  // KIND:PATH
        for (int i = 2; i < argc; ++i) {
            const std::string a = argv[i];
            const size_t colon = a.find(':');
            if (colon == std::string::npos) return 64;
            files.emplace_back(a.substr(0, colon), a.substr(colon + 1));
        }
        return run_files(std::string(argv[1]) == "files-apart", files);
    }
    std::fprintf(stderr, "usage: shared_context_host files[-apart] KIND:IN... (KIND 1|2|3|mpa|aac|vorbis; PCM to IN.pcm) | open vorbis N IN\n");
    return 64;
}
