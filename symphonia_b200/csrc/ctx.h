// Internal context definition shared by symgpu.cpp (MP3 + context) and symgpu_codecs.cpp (AAC, Vorbis).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/symgpu.h"
#include "codec_kernels.h"
#include "mp3_kernel.h"
#include "tables.h"

struct symgpu_async;                           // symgpu_async.cpp: batches gathered from many submitting threads
symgpu_async* symgpu_async_create();
void symgpu_async_destroy(symgpu_async*);

struct symgpu_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    char cuda_err[256] = {0};
    uint64_t launches = 0;
    symgpu_async* async = nullptr; // one submission queue per codec
    // Held by every batch leader of every codec around its host-entry-point call, and by the stream-slot calls decoders make
    // while other threads decode (resets, Vorbis slot configuration): they share d_stage, the plan / chunk caches and the stream.
    std::mutex launch_m;
    int numa_node = -1; // node the creating thread was bound to (-1: platform does not say, -2: binding switched off)
    // Layer III kernel choice (SYMGPU_MP3_KERNEL): 0 auto (by plan shape: long runs -> first generation,
    // short runs -> second generation), 1 always the first generation, 2 always the second
    int mp3_kernel_mode = 0;
    // tables
    symgpu::Mp3Tables* d_mp3_tab = nullptr;
    // MP3 streams
    symgpu::Mp3StreamState* d_mp3_states = nullptr; // [n][2]
    uint32_t* d_mp3_gen = nullptr;           // [n] + 1 word: retired-CTA counter
    uint32_t n_mp3_streams = 0;
    // tile list (host staging is pinned; cached while the caller repeats the same runs)
    symgpu::Mp3Tile* d_tiles = nullptr;
    symgpu::Mp3Tile* h_tiles = nullptr;
    size_t tiles_cap = 0;
    std::vector<symgpu_mp3_run> cached_runs;
    uint32_t cached_frames = 0;
    int cached_tiles = 0, cached_hdr = 0, cached_ctas = 0;
    bool cached_multi = false;
    bool cached_v2 = false;
    // launch plans of the host entry point's copy pipeline (one per slice), kept while the caller repeats the same runs: a
    // server that decodes the same streams step after step plans once.  Invalidated by anything that rewrites d_tiles.
    struct SlicePlan { uint32_t r0, r1, f0, f1; int t0, hdr, n_tiles, n_ctas; bool multi, v2; };
    std::vector<SlicePlan> slice_plans;
    std::vector<symgpu_mp3_run> slice_runs;
    uint32_t slice_frames = 0;
    int slice_key_slices = 0, slice_key_mode = -1;
    bool slice_plans_valid = false;
    // staging for the host entry points
    void* d_stage = nullptr;
    size_t stage_cap = 0;
    // copy pipeline of the host entry points: H2D on copy_in, kernels on `stream`, D2H on copy_out
    static constexpr int kMaxSlices = 32;
    // pinned (device-mapped) host buffers handed straight to the kernels: 0 never (default), 1 output only (PCM stores cross
    // PCIe from the kernel, no D2H copy), 2 input too (TMA reads across PCIe).  SM stores to host memory
    // are slower than the copy engines, so the staged pipeline is the default.  SYMGPU_ZERO_COPY
    int zero_copy = 0;
    bool zero_copy_small = true; // host batches below the pipeline threshold with mapped buffers: one launch on the caller's memory
    int h2d_ahead = 2; // slices whose H2D copy is queued before the host's descriptor check and planning (SYMGPU_H2D_AHEAD)
    int n_slices = 8; // slices of a host batch in the copy pipeline (SYMGPU_SLICES overrides, for tuning)
    cudaStream_t copy_in = nullptr, copy_out = nullptr;
    cudaStream_t copy_in2 = nullptr, copy_out2 = nullptr; // odd slices (SYMGPU_COPY_STREAMS=2): the next copy is already queued on
                                                          // another engine when one ends, so the link does not idle between slices
    int copy_streams = 1; // 2: copies of one direction on two streams can delay each other
    cudaEvent_t ev_in[kMaxSlices] = {}, ev_k[kMaxSlices] = {};
    cudaEvent_t ev_units = nullptr;
    // ---- AAC / Vorbis ----
    symgpu::CodecTables* d_codec_tab = nullptr;
    void* d_aac_fe_tab = nullptr;    // symgpu::aace::Tables: the AAC packet rules' tables (symgpu_aac_decode_*), on first use
    symgpu::CodecChunk* d_chunks = nullptr;
    symgpu::CodecChunk* h_chunks = nullptr;
    size_t chunks_cap = 0;
    // the chunk list on the device is reused while the caller repeats the same runs (tag + raw run bytes)
    std::vector<unsigned char> chunk_key;
    int cached_chunks = 0;
    int cached_groups = 0; // AAC: CTA passes (groups of chunks) of the cached list
    float* d_aac_states = nullptr;   // [n][2 gen][2 ch][1024]
    uint32_t* d_aac_gen = nullptr;   // [n] + retired-CTA counter
    uint32_t n_aac_streams = 0;
    float* d_aac_scratch = nullptr;  // TNS output, same shape as the batch spectra
    size_t aac_scratch_cap = 0;
    uint32_t* d_aac_tns_idx = nullptr; // [2][cap]: filter indices sorted by order, owner of each filter
    size_t aac_tns_idx_cap = 0;
    symgpu_vorbis_stream* d_vorbis_streams = nullptr;
    std::vector<symgpu_vorbis_stream> h_vorbis_streams;
    symgpu_vorbis_floor1* d_vorbis_floors = nullptr;
    symgpu::FloorAux* d_vorbis_floor_aux = nullptr;
    uint32_t n_vorbis_floors = 0;
    float* d_vorbis_states = nullptr; // [n][2 gen][kVorbisStateFloats]
    uint32_t* d_vorbis_gen = nullptr;
    uint32_t n_vorbis_streams = 0;
    // multichannel Vorbis (symgpu_vorbis_mc_*): the caller's stream records; every one is registered as 4 stereo pseudo-streams
    symgpu_vorbis_stream_mc* d_vorbis_mc_streams = nullptr;
    std::vector<symgpu_vorbis_stream_mc> h_vorbis_mc_streams;
    uint32_t n_vorbis_mc_streams = 0;
    void* d_vorbis_mc_scratch = nullptr; // per-pair unit records + stream of every packet
    size_t vorbis_mc_scratch_cap = 0;
    uint32_t vorbis_cfg_epoch = 0;   // bumped by streams_set: chunk sizes depend on the stream block sizes
    // slots of symgpu_vorbis_streams_alloc: floor setups configured per slot (empty when the streams came from streams_set);
    // a slot is configured when its record's bs1_exp is non-zero
    std::vector<uint8_t> vorbis_slot_floors;
    std::atomic<uint32_t> vorbis_row{0}; // largest blocksize_1 / 2 among the configured slots: the row of a submission batch
};

namespace symgpu_detail {

inline symgpu_status cuda_fail(symgpu_ctx* ctx, cudaError_t e, const char* where) {
    if (ctx) std::snprintf(ctx->cuda_err, sizeof ctx->cuda_err, "%s: %s", where, cudaGetErrorString(e));
    return SYMGPU_ERR_CUDA;
}

#define CU(ctx, call)                                                   \
    do {                                                                \
        cudaError_t e_ = (call);                                        \
        if (e_ != cudaSuccess) return cuda_fail((ctx), e_, #call);      \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};


// Grows the scratch/staging buffer of a context (synchronises the stream first).
inline symgpu_status ensure_stage(symgpu_ctx* ctx, size_t need) {
    if (need <= ctx->stage_cap) return SYMGPU_OK;
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaStreamSynchronize");
    if (ctx->d_stage) cudaFree(ctx->d_stage);
    ctx->d_stage = nullptr;
    ctx->stage_cap = 0;
    e = cudaMalloc(&ctx->d_stage, need);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaMalloc(stage)");
    ctx->stage_cap = need;
    return SYMGPU_OK;
}

// ensure_stage for a call that has already written the first `keep` bytes of the buffer: a larger buffer starts with a copy of them.
inline symgpu_status ensure_stage_keep(symgpu_ctx* ctx, size_t need, size_t keep) {
    if (need <= ctx->stage_cap) return SYMGPU_OK;
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaStreamSynchronize");
    void* grown = nullptr;
    e = cudaMalloc(&grown, need);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaMalloc(stage)");
    if (keep) e = cudaMemcpy(grown, ctx->d_stage, keep, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) {
        cudaFree(grown);
        return cuda_fail(ctx, e, "cudaMemcpy(stage)");
    }
    cudaFree(ctx->d_stage);
    ctx->d_stage = grown;
    ctx->stage_cap = need;
    return SYMGPU_OK;
}

} // namespace symgpu_detail
