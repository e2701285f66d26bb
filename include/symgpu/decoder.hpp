// C++ host-side mirror of the reference's decoder plug-in interface, on top of the C ABI (symgpu.h).
//
// The reference is Rust; its toolchain is not available in this environment (see INTEGRATION.md for
// the Rust adapter a maintainer would add).  This header restates the SAME interface in C++17 with
// the same names, argument meaning and error behaviour, so a C++ host can drop the GPU synthesis
// path in behind a registry exactly as a Rust host would:
//
//   AudioDecoder            symphonia-core/src/codecs/audio.rs:251-298   (reset / codec_params / decode /
//                                                                          finalize / last_decoded)
//   AudioDecoderOptions     symphonia-core/src/codecs/audio.rs:210-227   (gapless = true, verify = false)
//   CodecRegistry, Tier     symphonia-core/src/codecs/registry.rs:176-341, symphonia-core/src/common.rs:54-62
//                           (lookup order preferred -> standard -> fallback)
//   Error                   symphonia-core/src/errors.rs:43-57
//   Packet                  symphonia-core/src/packet.rs:146-170 (PacketRef)
//
// A packet handed to GpuMpaDecoder is what the reference's MpaReader emits: one whole MPEG audio frame, header word
// first (Layers I, II and III; the entropy front-ends of SURVEY.md §8f N1 run on the CPU inside decode(), the
// synthesis on the GPU).  For tests and for hosts with their own bit reader it also accepts the *parsed* Layer III
// frame -- the state the reference has at layer3/mod.rs:421 -- as bytes: symgpu_mp3_gc[2][2] (256 B) followed by
// f32 spectra [2][2][576]; the two cannot be confused, a real frame is at most 2881 bytes.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../symgpu.h"

namespace symgpu_host {

enum class ErrorKind { None, IoError, DecodeError, SeekError, Unsupported, LimitError, ResetRequired };
struct Error {
    ErrorKind kind = ErrorKind::None;
    const char* message = ""; // static storage, like the reference's &'static str
    explicit operator bool() const { return kind != ErrorKind::None; }
};
template <typename T>
struct Result {
    T value{};
    Error error{};
    bool ok() const { return !error; }
};

inline Error map_status(symgpu_status st) { // INTEGRATION.md §3
    switch (st) {
        case SYMGPU_OK: return {};
        case SYMGPU_ERR_DECODE: return {ErrorKind::DecodeError, symgpu_strerror(st)};
        case SYMGPU_ERR_UNSUPPORTED: return {ErrorKind::Unsupported, symgpu_strerror(st)};
        case SYMGPU_ERR_LIMIT: return {ErrorKind::LimitError, symgpu_strerror(st)};
        case SYMGPU_ERR_RESET: return {ErrorKind::ResetRequired, symgpu_strerror(st)};
        default: return {ErrorKind::IoError, symgpu_strerror(st)};
    }
}

// Codec ids, symphonia-core/src/codecs/audio.rs:404-418.
constexpr uint32_t CODEC_ID_VORBIS = 0x1000, CODEC_ID_MP1 = 0x1004, CODEC_ID_MP2 = 0x1005, CODEC_ID_MP3 = 0x1006, CODEC_ID_AAC = 0x1007;

struct AudioCodecParameters {
    uint32_t codec = 0;
    uint32_t sample_rate = 0;
    uint32_t channels = 0;
    std::vector<uint8_t> extra_data;
};
struct AudioDecoderOptions {
    bool gapless = true;
    bool verify = false;
};
struct FinalizeResult {
    bool has_verify = false, verify_ok = false;
};
struct Packet { // PacketRef
    uint32_t track_id = 0;
    uint64_t pts = 0, dur = 0;
    uint32_t trim_start = 0, trim_end = 0;
    const uint8_t* data = nullptr;
    size_t len = 0;
};
// Borrow of the decoder-owned planar f32 buffer, valid until the next call on the decoder
// (GenericAudioBufferRef over AudioBuffer<f32>, symphonia-core/src/audio/buf.rs:68-73).
struct AudioBufferRef {
    const float* planes[2] = {nullptr, nullptr};
    size_t n_planes = 0;
    size_t frames = 0;
};

class AudioDecoder {
  public:
    virtual ~AudioDecoder() = default;
    virtual void reset() = 0;
    virtual const AudioCodecParameters& codec_params() const = 0;
    virtual Result<AudioBufferRef> decode(const Packet& packet) = 0;
    virtual FinalizeResult finalize() { return {}; }
    virtual AudioBufferRef last_decoded() const = 0;
};

enum class Tier { Preferred, Standard, Fallback };
using AudioDecoderFactory =
    std::function<Result<std::unique_ptr<AudioDecoder>>(const AudioCodecParameters&, const AudioDecoderOptions&)>;

class CodecRegistry {
  public:
    void register_audio_decoder_at_tier(Tier tier, uint32_t codec, AudioDecoderFactory factory) {
        slots_[codec][(int)tier] = std::move(factory);
    }
    // registry.rs:330-341: preferred, then standard, then fallback.
    Result<std::unique_ptr<AudioDecoder>> make_audio_decoder(const AudioCodecParameters& p, const AudioDecoderOptions& o) const {
        auto it = slots_.find(p.codec);
        if (it != slots_.end())
            for (int t = 0; t < 3; ++t)
                if (it->second[t]) return it->second[t](p, o);
        return {nullptr, {ErrorKind::Unsupported, "core (codec): unsupported codec"}};
    }

  private:
    std::map<uint32_t, AudioDecoderFactory[3]> slots_;
};

// A context shared by GPU decoders (one CUDA stream).  Stream-state slots are handed out from a free list under a mutex; every
// decoder of the registry takes one, whatever its codec (a Vorbis decoder too: its slot holds the stream's configuration and
// floor setups).  Every decoder of the registry may run on any thread: decode() goes through the thread-safe submit / wait pair
// of its codec, which gathers the packets of all threads into shared launches, and reset() through the thread-safe slot resets.
class GpuContext {
  public:
    // max_streams: decoders open at once.  Vorbis decoders can use the first min(max_streams, SYMGPU_VORBIS_MAX_SLOTS) slots.
    static Result<std::shared_ptr<GpuContext>> create(int device, uint32_t max_streams) {
        symgpu_ctx* c = nullptr;
        symgpu_status st = symgpu_ctx_create(device, &c);
        if (st != SYMGPU_OK) return {nullptr, map_status(st)};
        std::shared_ptr<GpuContext> g(new GpuContext(c, max_streams, device));
        st = symgpu_mp3_streams_alloc(c, max_streams);
        if (st == SYMGPU_OK) st = symgpu_aac_streams_alloc(c, max_streams);
        if (st == SYMGPU_OK) st = symgpu_vorbis_streams_alloc(c, std::min<uint32_t>(max_streams, SYMGPU_VORBIS_MAX_SLOTS));
        if (st != SYMGPU_OK) return {nullptr, map_status(st)};
        return {g, {}};
    }
    ~GpuContext() { symgpu_ctx_destroy(ctx_); }
    symgpu_ctx* raw() const { return ctx_; }
    int device() const { return device_; }
    int acquire_stream() {
        std::lock_guard<std::mutex> g(m_);
        if (free_.empty()) return -1;
        const int s = free_.back();
        free_.pop_back();
        return s;
    }
    void release_stream(int s) {
        std::lock_guard<std::mutex> g(m_);
        free_.push_back(s);
    }

  private:
    GpuContext(symgpu_ctx* c, uint32_t n, int device) : ctx_(c), device_(device) {
        for (int i = (int)n - 1; i >= 0; --i) free_.push_back(i);
    }
    symgpu_ctx* ctx_;
    int device_;
    std::mutex m_;
    std::vector<int> free_;
};

// MPEG audio decoder (Layers I-III by codec id) whose synthesis stage runs on the GPU (mirrors MpaDecoder,
// symphonia-bundle-mp3/src/decoder.rs:66-197).  See the packet format note at the top of this file.
class GpuMpaDecoder final : public AudioDecoder {
  public:
    static constexpr size_t kPacketBytes = 4 * sizeof(symgpu_mp3_gc) + SYMGPU_MP3_FRAME_FLOATS * sizeof(float);

    static Result<std::unique_ptr<AudioDecoder>> try_new(std::shared_ptr<GpuContext> gpu, const AudioCodecParameters& p,
                                                         const AudioDecoderOptions& o) {
        if (p.codec != CODEC_ID_MP3 && p.codec != CODEC_ID_MP2 && p.codec != CODEC_ID_MP1)
            return {nullptr, {ErrorKind::Unsupported, "mpa: invalid codec type"}};
        const int slot = gpu->acquire_stream();
        if (slot < 0) return {nullptr, {ErrorKind::LimitError, "symgpu: no free stream slot"}};
        symgpu_mp3_fe* fe = nullptr;
        if (p.codec == CODEC_ID_MP3 && symgpu_mp3_fe_create(&fe) != SYMGPU_OK) {
            gpu->release_stream(slot);
            return {nullptr, {ErrorKind::LimitError, "symgpu: out of memory"}};
        }
        return {std::unique_ptr<AudioDecoder>(new GpuMpaDecoder(std::move(gpu), p, o, (uint32_t)slot, fe)), {}};
    }
    ~GpuMpaDecoder() override {
        symgpu_mp3_stream_reset(gpu_->raw(), stream_);
        gpu_->release_stream((int)stream_);
        symgpu_mp3_fe_destroy(fe_);
    }
    void reset() override { // decoder.rs:152-155: the whole decoder state starts over
        symgpu_mp3_stream_reset(gpu_->raw(), stream_);
        symgpu_mp3_fe_reset(fe_);
        have_spec_ = false;
        frames_ = 0;
    }
    const AudioCodecParameters& codec_params() const override { return params_; }
    Result<AudioBufferRef> decode(const Packet& packet) override {
        frames_ = 0; // buf.clear(): on any error the buffer stays empty (codecs/audio.rs:278)
        if (packet.len != kPacketBytes) return decode_frame(packet);
        if (params_.codec != CODEC_ID_MP3) return {{}, {ErrorKind::DecodeError, "mpa: invalid mpeg audio layer"}};
        symgpu_mp3_gc units[4];
        std::memcpy(units, packet.data, sizeof units);
        const float* spectra = reinterpret_cast<const float*>(packet.data + sizeof units);
        const bool mpeg1 = units[0].flags & SYMGPU_MP3_F_MPEG1;
        const bool mono = units[1].flags & SYMGPU_MP3_F_MUTE;
        const bool joint = units[0].flags & (SYMGPU_MP3_F_MID_SIDE | SYMGPU_MP3_F_INTENSITY);
        // stereo.rs:503-505: a parse-level validity check that stays on the host side of the ABI
        for (int gr = 0; gr < (mpeg1 ? 2 : 1) && joint && !mono; ++gr)
            if (units[2 * gr].block_type != units[2 * gr + 1].block_type ||
                ((units[2 * gr].flags ^ units[2 * gr + 1].flags) & SYMGPU_MP3_F_MIXED))
                return {{}, {ErrorKind::DecodeError, "mpa: stereo channel pair block_type mismatch"}};
        symgpu_mp3_run run{};
        run.stream = stream_;
        run.first_frame = 0;
        run.n_frames = 1;
        run.granules_per_frame = mpeg1 ? 2 : 1;
        run.channels = mono ? 1 : 2;
        // thread-safe, batched with the packets other decoders of this context have in flight
        symgpu_ticket ticket;
        symgpu_status st = symgpu_mp3_submit(gpu_->raw(), stream_, units, spectra, run.granules_per_frame, run.channels, &ticket);
        if (st == SYMGPU_OK) st = symgpu_mp3_wait(gpu_->raw(), ticket, pcm_.data());
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        return finish(packet, mpeg1 ? 1152 : 576, mono ? 1 : 2);
    }
    AudioBufferRef last_decoded() const override {
        AudioBufferRef r;
        r.n_planes = planes_;
        r.frames = frames_;
        r.planes[0] = pcm_.data() + first_;
        r.planes[1] = pcm_.data() + 1152 + first_;
        return r;
    }

  private:
    GpuMpaDecoder(std::shared_ptr<GpuContext> gpu, AudioCodecParameters p, AudioDecoderOptions o, uint32_t stream, symgpu_mp3_fe* fe)
        : gpu_(std::move(gpu)), params_(std::move(p)), opts_(o), stream_(stream), fe_(fe), pcm_(SYMGPU_MP3_FRAME_FLOATS, 0.0f),
          planes_(params_.channels ? params_.channels : 2) {}

    // A real frame: entropy front-end on the CPU (MpaDecoder::decode_inner up to the synthesis call), synthesis on the GPU.
    Result<AudioBufferRef> decode_frame(const Packet& packet) {
        symgpu_mp3_frame_info info{};
        symgpu_status st;
        size_t frames;
        if (params_.codec == CODEC_ID_MP3) {
            symgpu_mp3_gc units[4];
            st = symgpu_mp3_fe_decode(fe_, packet.data, packet.len, units, quant_, &info);
            if (st != SYMGPU_OK) return {{}, map_status(st)};
            const bool joint = units[0].flags & (SYMGPU_MP3_F_MID_SIDE | SYMGPU_MP3_F_INTENSITY);
            for (int gr = 0; gr < info.granules && joint && info.channels == 2; ++gr)  // stereo.rs:503-505
                if (units[2 * gr].block_type != units[2 * gr + 1].block_type ||
                    (units[2 * gr].block_type == SYMGPU_MP3_SHORT && ((units[2 * gr].flags ^ units[2 * gr + 1].flags) & SYMGPU_MP3_F_MIXED)))
                    return {{}, {ErrorKind::DecodeError, "mpa: stereo channel pair block_type mismatch"}};
            symgpu_mp3_run run{};
            run.stream = stream_, run.n_frames = 1, run.granules_per_frame = info.granules, run.channels = info.channels;
            symgpu_ticket ticket;
            st = symgpu_mp3_submit_quantized(gpu_->raw(), stream_, units, quant_, run.granules_per_frame, run.channels, &ticket);
            if (st == SYMGPU_OK) st = symgpu_mp3_wait(gpu_->raw(), ticket, pcm_.data());
            frames = info.granules == 2 ? 1152 : 576;
        } else {
            const int layer = params_.codec == CODEC_ID_MP1 ? 1 : 2, n_slots = layer == 1 ? 12 : 36;
            st = symgpu_mpa12_fe_decode(packet.data, packet.len, layer, sub_, &info);
            if (st != SYMGPU_OK) return {{}, map_status(st)};
            // decoder.rs:96-108: the signal specification is fixed by the first frame
            if (!have_spec_) have_spec_ = true, spec_rate_ = info.sample_rate, spec_channels_ = info.channels;
            else if (spec_rate_ != info.sample_rate || spec_channels_ != info.channels)
                return {{}, {ErrorKind::DecodeError, "mpa: invalid audio buffer signal spec for packet"}};
            symgpu_ticket ticket;  // batched with the Layer I / II packets other decoders of this context have in flight
            st = symgpu_mpa12_submit(gpu_->raw(), stream_, sub_, (uint32_t)n_slots, info.channels, &ticket);
            if (st == SYMGPU_OK) st = symgpu_mpa12_wait(gpu_->raw(), ticket, pcm_.data());
            frames = 32 * (size_t)n_slots;
        }
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        return finish(packet, frames, info.channels);
    }
    Result<AudioBufferRef> finish(const Packet& packet, size_t frames, size_t planes) {
        frames_ = frames, planes_ = planes;
        // gapless trimming (decoder.rs:130-132)
        size_t begin = 0, end = frames_;
        if (opts_.gapless) {
            begin = std::min<size_t>(packet.trim_start, frames_);
            end = frames_ - std::min<size_t>(packet.trim_end, frames_ - begin);
        }
        first_ = begin;
        frames_ = end - begin;
        return {last_decoded(), {}};
    }

    std::shared_ptr<GpuContext> gpu_;
    AudioCodecParameters params_;
    AudioDecoderOptions opts_;
    uint32_t stream_;
    symgpu_mp3_fe* fe_;
    std::vector<float> pcm_;
    int16_t quant_[4 * 576];
    float sub_[2 * 32 * 36];
    size_t frames_ = 0, first_ = 0, planes_ = 2;
    bool have_spec_ = false;
    uint32_t spec_rate_ = 0, spec_channels_ = 0;
};

// AAC-LC decoder whose filterbank runs on the GPU (mirrors AacDecoder, symphonia-codec-aac/src/aac/mod.rs:42-304).  A packet is
// one raw_data_block, what the reference's AdtsReader and IsoMp4Reader emit.  Without extra data the stream parameters are the
// codec parameters' (the ADTS case, mod.rs:64-78); with extra data they come from the AudioSpecificConfig, read and judged as the
// reference does (symgpu_aac_fe_create_asc: AAC-LC, no SBR, at most two channels, 1024-sample frames).
class GpuAacDecoder final : public AudioDecoder {
  public:
    static Result<std::unique_ptr<AudioDecoder>> try_new(std::shared_ptr<GpuContext> gpu, const AudioCodecParameters& p,
                                                         const AudioDecoderOptions&) {
        if (p.codec != CODEC_ID_AAC) return {nullptr, {ErrorKind::Unsupported, "aac: invalid codec"}};
        AudioCodecParameters params = p;
        symgpu_aac_fe* fe = nullptr;
        if (!p.extra_data.empty()) {  // AudioSpecificConfig (mod.rs:59-62, :101-108)
            symgpu_aac_asc asc;
            const symgpu_status st = symgpu_aac_fe_create_asc(p.extra_data.data(), p.extra_data.size(), &fe, &asc);
            if (st != SYMGPU_OK) return {nullptr, map_status(st)};
            params.sample_rate = asc.sample_rate, params.channels = asc.channels;
        }
        if (params.sample_rate == 0) return {nullptr, {ErrorKind::Unsupported, "aac: sample rate is required"}};
        if (params.channels == 0) return {nullptr, {ErrorKind::Unsupported, "aac: channels or channel layout is required"}};
        if (params.channels > 2) return {nullptr, {ErrorKind::Unsupported, "aac: aac too complex"}};
        const int slot = gpu->acquire_stream();
        if (slot < 0) {
            symgpu_aac_fe_destroy(fe);
            return {nullptr, {ErrorKind::LimitError, "symgpu: no free stream slot"}};
        }
        if (!fe) {
            const symgpu_status st = symgpu_aac_fe_create(params.sample_rate, params.channels, &fe);
            if (st != SYMGPU_OK) {
                gpu->release_stream(slot);
                return {nullptr, map_status(st)};
            }
        }
        symgpu_aac_stream_reset(gpu->raw(), (uint32_t)slot);
        return {std::unique_ptr<AudioDecoder>(new GpuAacDecoder(std::move(gpu), std::move(params), (uint32_t)slot, fe)), {}};
    }
    ~GpuAacDecoder() override {
        gpu_->release_stream((int)stream_);
        symgpu_aac_fe_destroy(fe_);
    }
    void reset() override {  // mod.rs:259-263: every pair's window history and delay lines
        symgpu_aac_stream_reset(gpu_->raw(), stream_);
        symgpu_aac_fe_reset(fe_);
        frames_ = 0;
    }
    const AudioCodecParameters& codec_params() const override { return params_; }
    Result<AudioBufferRef> decode(const Packet& packet) override {
        frames_ = 0;  // buf.clear() on any error (mod.rs:274-277)
        symgpu_aac_unit units[2];
        uint32_t n_tns = 0;
        symgpu_status st = symgpu_aac_fe_decode(fe_, packet.data, packet.len, 0, units, tns_, &n_tns, coeffs_.data());
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        symgpu_ticket ticket;  // batched with the AAC packets other decoders of this context have in flight
        st = symgpu_aac_submit(gpu_->raw(), stream_, units, n_tns ? tns_ : nullptr, n_tns, coeffs_.data(), (uint8_t)params_.channels, &ticket);
        if (st == SYMGPU_OK) st = symgpu_aac_wait(gpu_->raw(), ticket, pcm_.data());
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        frames_ = 1024;  // the reference's AAC decoder trims nothing (mod.rs:231-255)
        return {last_decoded(), {}};
    }
    AudioBufferRef last_decoded() const override {
        AudioBufferRef r;
        r.n_planes = params_.channels;
        r.frames = frames_;
        r.planes[0] = pcm_.data();
        r.planes[1] = pcm_.data() + 1024;
        return r;
    }

  private:
    GpuAacDecoder(std::shared_ptr<GpuContext> gpu, AudioCodecParameters p, uint32_t stream, symgpu_aac_fe* fe)
        : gpu_(std::move(gpu)), params_(std::move(p)), stream_(stream), fe_(fe), coeffs_(2048, 0.0f), pcm_(2048, 0.0f) {}
    std::shared_ptr<GpuContext> gpu_;
    AudioCodecParameters params_;
    uint32_t stream_;
    symgpu_aac_fe* fe_;
    symgpu_aac_tns tns_[16];
    std::vector<float> coeffs_, pcm_;
    size_t frames_ = 0;
};

// Vorbis decoder whose floor synthesis, inverse coupling, IMDCT and overlap-add run on the GPU (mirrors VorbisDecoder,
// symphonia-codec-vorbis/src/lib.rs:48-420).  Extra data = the identification packet followed by the setup packet, as the Ogg
// mapping hands them over (mappings/vorbis.rs:196-214).  The decoder takes a stream slot of the shared context and configures it
// with the stream's block sizes and floor setups; its packets are batched with those of every other decoder of the context.
class GpuVorbisDecoder final : public AudioDecoder {
  public:
    static Result<std::unique_ptr<AudioDecoder>> try_new(std::shared_ptr<GpuContext> gpu, const AudioCodecParameters& p,
                                                         const AudioDecoderOptions& o) {
        if (p.codec != CODEC_ID_VORBIS) return {nullptr, {ErrorKind::Unsupported, "vorbis: invalid codec type"}};
        if (p.extra_data.size() <= 30) return {nullptr, {ErrorKind::Unsupported, "vorbis: missing extra data"}};
        symgpu_vorbis_fe* fe = nullptr;
        symgpu_status st = symgpu_vorbis_fe_create(p.extra_data.data(), 30, p.extra_data.data() + 30, p.extra_data.size() - 30, &fe);
        if (st != SYMGPU_OK) return {nullptr, map_status(st)};
        symgpu_vorbis_stream config{};
        std::vector<symgpu_vorbis_floor1> floors(SYMGPU_VORBIS_SLOT_FLOORS);
        uint32_t n_floors = 0;
        symgpu_vorbis_fe_config(fe, &config, floors.data(), &n_floors);
        const int slot = gpu->acquire_stream();
        if (slot < 0) {
            symgpu_vorbis_fe_destroy(fe);
            return {nullptr, {ErrorKind::LimitError, "symgpu: no free stream slot"}};
        }
        uint32_t floor_base = 0;
        st = symgpu_vorbis_stream_configure(gpu->raw(), (uint32_t)slot, &config, floors.data(), n_floors, &floor_base);
        if (st != SYMGPU_OK) {
            gpu->release_stream(slot);
            symgpu_vorbis_fe_destroy(fe);
            return {nullptr, map_status(st)};
        }
        AudioCodecParameters params = p;
        params.channels = config.channels;
        return {std::unique_ptr<AudioDecoder>(new GpuVorbisDecoder(std::move(gpu), std::move(params), o, fe, config, (uint32_t)slot, floor_base)), {}};
    }
    ~GpuVorbisDecoder() override {
        gpu_->release_stream((int)stream_);
        symgpu_vorbis_fe_destroy(fe_);
    }
    void reset() override {  // lib.rs:336-338 -> dsp.rs:26-32: overlap cleared, no previous block
        symgpu_vorbis_stream_reset(gpu_->raw(), stream_);
        symgpu_vorbis_fe_reset(fe_);
        have_prev_ = false;
        frames_ = 0;
    }
    const AudioCodecParameters& codec_params() const override { return params_; }
    Result<AudioBufferRef> decode(const Packet& packet) override {
        frames_ = first_ = 0;
        symgpu_vorbis_unit unit;
        symgpu_status st = symgpu_vorbis_fe_decode(fe_, packet.data, packet.len, slot_, floor_base_, &unit, floor_y_, residue_.data());
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        symgpu_ticket ticket;  // batched with the Vorbis packets other decoders of this context have in flight
        st = symgpu_vorbis_submit(gpu_->raw(), stream_, &unit, floor_y_, residue_.data(), slot_, &ticket);
        if (st == SYMGPU_OK) st = symgpu_vorbis_wait(gpu_->raw(), ticket, pcm_.data());
        if (st != SYMGPU_OK) return {{}, map_status(st)};
        const size_t prev_n = size_t(1) << (unit.prev_block_flag ? config_.bs1_exp : config_.bs0_exp);
        const size_t n = size_t(1) << (unit.block_flag ? config_.bs1_exp : config_.bs0_exp);
        frames_ = (prev_n + n) / 4;
        if (opts_.gapless) {  // lib.rs:316-326
            if (!have_prev_) {
                frames_ = 0;  // the first packet after a reset is silenced
            } else {
                first_ = std::min<size_t>(packet.trim_start, frames_);
                frames_ -= first_;
                frames_ -= std::min<size_t>(packet.trim_end, frames_);
            }
        }
        have_prev_ = true;
        return {last_decoded(), {}};
    }
    AudioBufferRef last_decoded() const override {
        AudioBufferRef r;
        r.n_planes = params_.channels;
        r.frames = frames_;
        r.planes[0] = pcm_.data() + first_;
        r.planes[1] = pcm_.data() + slot_ + first_;
        return r;
    }

  private:
    GpuVorbisDecoder(std::shared_ptr<GpuContext> gpu, AudioCodecParameters p, AudioDecoderOptions o, symgpu_vorbis_fe* fe,
                     symgpu_vorbis_stream config, uint32_t stream, uint32_t floor_base)
        : gpu_(std::move(gpu)), params_(std::move(p)), opts_(o), fe_(fe), config_(config), stream_(stream), floor_base_(floor_base),
          slot_((1u << config.bs1_exp) >> 1), residue_(2 * size_t(slot_), 0.0f), pcm_(2 * size_t(slot_), 0.0f) {}
    std::shared_ptr<GpuContext> gpu_;
    AudioCodecParameters params_;
    AudioDecoderOptions opts_;
    symgpu_vorbis_fe* fe_;
    symgpu_vorbis_stream config_;
    uint32_t stream_, floor_base_;
    uint32_t slot_;  // floats per channel of the residue / PCM buffers: blocksize_1 / 2
    uint16_t floor_y_[2 * 65];
    std::vector<float> residue_, pcm_;
    size_t frames_ = 0, first_ = 0;
    bool have_prev_ = false;
};

// What an application does next to symphonia::default::register_enabled_codecs (symphonia/src/lib.rs:234-255).
inline void register_gpu_decoders(CodecRegistry& registry, std::shared_ptr<GpuContext> gpu) {
    for (uint32_t codec : {CODEC_ID_MP1, CODEC_ID_MP2, CODEC_ID_MP3})
        registry.register_audio_decoder_at_tier(Tier::Preferred, codec, [gpu](const AudioCodecParameters& p, const AudioDecoderOptions& o) {
            return GpuMpaDecoder::try_new(gpu, p, o);
        });
    registry.register_audio_decoder_at_tier(Tier::Preferred, CODEC_ID_AAC, [gpu](const AudioCodecParameters& p, const AudioDecoderOptions& o) {
        return GpuAacDecoder::try_new(gpu, p, o);
    });
    registry.register_audio_decoder_at_tier(Tier::Preferred, CODEC_ID_VORBIS, [gpu](const AudioCodecParameters& p, const AudioDecoderOptions& o) {
        return GpuVorbisDecoder::try_new(gpu, p, o);
    });
}

} // namespace symgpu_host
